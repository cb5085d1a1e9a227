"""Import-path shim: `from estimator.datasets import build_dataset, UnrealStereo4kDataset, ImageDataset` resolves to
the evaluation datasets of patchfusion_b200/datasets.py, registered in `DATASETS` under the reference's names
(`estimator/datasets/__init__.py`, `builder.py:5-7`)."""
from estimator.registry import DATASETS
from patchfusion_b200 import datasets as _ds

UnrealStereo4kDataset = DATASETS.register_module(name='UnrealStereo4kDataset')(_ds.UnrealStereo4kDataset)
ImageDataset = DATASETS.register_module(name='ImageDataset')(_ds.ImageDataset)


def build_dataset(cfg):
    return DATASETS.build(cfg)


__all__ = ['build_dataset', 'UnrealStereo4kDataset', 'ImageDataset']
