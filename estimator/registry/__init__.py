"""Minimal `MODELS` / `DATASETS` registries with the reference's call surface (`estimator/registry/registry.py:7-8`,
`estimator/models/builder.py:6-8`, `estimator/datasets/builder.py:5-7`):
`MODELS.build(dict(type='PatchFusion', config=...))`, `DATASETS.build(dict(type='UnrealStereo4kDataset', ...))`."""


class _Registry:
    def __init__(self, name):
        self.name, self._mods = name, {}

    def register_module(self, name=None):
        def deco(cls):
            self._mods[name or cls.__name__] = cls
            return cls
        return deco

    def get(self, k):
        return self._mods.get(k)

    def build(self, cfg):
        cfg = dict(cfg)
        typ = cfg.pop('type')
        if typ not in self._mods:
            raise KeyError('%s is not in the %s registry (registered: %s)' % (typ, self.name, ', '.join(sorted(self._mods))))
        return self._mods[typ](**cfg)


MODELS = _Registry('model')
DATASETS = _Registry('dataset')
