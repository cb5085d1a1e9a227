"""Import-path shim: `from estimator.models.patchfusion import PatchFusion` and
`from estimator.models.baseline_pretrain import BaselinePretrain` resolve to the H100 implementations (reference
`estimator/models/patchfusion.py:55`, `baseline_pretrain.py:43`), and `from estimator.datasets import build_dataset`
to the evaluation datasets.  Only inference and evaluation are provided; the reference's trainers are out of scope."""
