"""Model construction entry point with the reference's name (`build_model`).  Only the inference model types are
registered in this build (PatchFusion, BaselinePretrain); anything else is reported with the list of what exists."""
from estimator import registry


def build_model(cfg):
    if not isinstance(cfg, dict) or 'type' not in cfg:
        raise TypeError("build_model expects a dict with a 'type' key, got %r" % (type(cfg).__name__,))
    known = sorted(registry.MODELS._mods)
    if cfg['type'] not in known:
        raise KeyError("model type %r is not available here (registered: %s)" % (cfg['type'], ', '.join(known)))
    kwargs = {k: v for k, v in cfg.items() if k != 'type'}
    return registry.MODELS.get(cfg['type'])(**kwargs)
