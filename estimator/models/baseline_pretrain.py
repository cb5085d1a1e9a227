"""Drop-in for the reference module of the same path: `BaselinePretrain` registered under the same name."""
from estimator.registry import MODELS
from patchfusion_b200.baseline import BaselinePretrain as _BaselinePretrain

BaselinePretrain = MODELS.register_module(name='BaselinePretrain')(_BaselinePretrain)
