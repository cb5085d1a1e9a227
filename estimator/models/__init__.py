from .builder import build_model  # noqa: F401
from .baseline_pretrain import BaselinePretrain  # noqa: F401
from .patchfusion import PatchFusion  # noqa: F401
