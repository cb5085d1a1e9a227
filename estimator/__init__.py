"""Import-path shim: `from estimator.models.patchfusion import PatchFusion` and
`from estimator.models.baseline_pretrain import BaselinePretrain` resolve to the H100 implementations (reference
`estimator/models/patchfusion.py:55`, `baseline_pretrain.py:43`).  Only the inference models are provided; the
reference's trainers, datasets and tools are out of scope."""
