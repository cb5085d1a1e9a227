"""Reference-format Python config files (`configs/patchfusion_depthanything/*.py`) without mmengine.

`load_config(path)` executes the file, resolves its `_base_` list relative to the file and merges the bases in order,
then the file itself: a child key overrides, nested dicts merge recursively, lists and every other value replace.
`--cfg-options a.b=v` strings go through `parse_options` / `merge_options` with mmengine's `DictAction` value parsing.
The result is an `AttrDict` (attribute access, as the reference's code reads `cfg.val_dataloader.dataset`)."""
import copy
import os
import pprint
import runpy
import types

from .model import AttrDict


def _merge(base, child):
    out = copy.deepcopy(base)
    for k, v in child.items():
        if isinstance(v, dict) and isinstance(out.get(k), dict) and not v.get('_delete_', False):
            out[k] = _merge(out[k], v)
        else:
            out[k] = copy.deepcopy({a: b for a, b in v.items() if a != '_delete_'} if isinstance(v, dict) else v)
    return out


def _file_dict(path):
    path = os.path.abspath(path)
    ns = runpy.run_path(path)
    bases = ns.get('_base_', [])
    if isinstance(bases, str):
        bases = [bases]
    merged = {}
    for b in bases:
        merged = _merge(merged, _file_dict(os.path.join(os.path.dirname(path), b)))
    own = {k: v for k, v in ns.items()
           if not k.startswith('__') and k != '_base_' and not isinstance(v, types.ModuleType)
           and not callable(v)}
    return _merge(merged, own)


def load_config(path):
    """Config dict of a reference-format config file, `_base_` chains resolved."""
    return AttrDict(_file_dict(path))


def _plain(v):
    if isinstance(v, dict):
        return {k: _plain(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return type(v)(_plain(x) for x in v)
    return v


def save_config(cfg, path):
    """Write cfg (a load_config dict, `_base_` already merged) as a self-contained config file that load_config reads
    back equal: one `key = <literal>` per top-level key.  ValueError for a value without such a literal."""
    cfg = _plain(dict(cfg))
    text = ''.join('%s = %s\n' % (k, pprint.pformat(v, width=120, sort_dicts=False)) for k, v in cfg.items())
    with open(path, 'w') as f:
        f.write(text)
    try:
        back = _plain(dict(load_config(path)))
    except Exception as e:
        raise ValueError('save_config: %s does not load back (%r)' % (path, e))
    if back != cfg:
        raise ValueError('save_config: %s loads back as a different config' % path)


def _parse_int_float_bool(v):
    try:
        return int(v)
    except ValueError:
        pass
    try:
        return float(v)
    except ValueError:
        pass
    if v.lower() in ('true', 'false'):
        return v.lower() == 'true'
    if v == 'None':
        return None
    return v


def _find_next_comma(s):
    """Index of the first comma of s outside brackets (mmengine DictAction.find_next_comma)."""
    depth = 0
    for i, c in enumerate(s):
        if c in '([':
            depth += 1
        elif c in ')]':
            depth -= 1
        elif c == ',' and depth == 0:
            return i
    if depth != 0:
        raise ValueError('imbalanced brackets in %r' % s)
    return len(s)


def parse_value(val):
    """mmengine `DictAction._parse_iterable`: 'a' -> str, '1' -> int, '1.5' -> float, 'true' -> bool, 'None' -> None,
    'a,b' / '[a,b]' -> list, '(a,b)' -> tuple, nested brackets allowed."""
    val = val.strip('\'"').replace(' ', '')
    is_tuple = False
    if val.startswith('(') and val.endswith(')'):
        is_tuple, val = True, val[1:-1]
    elif val.startswith('[') and val.endswith(']'):
        val = val[1:-1]
    elif ',' not in val:
        return _parse_int_float_bool(val)
    values = []
    while len(val) > 0:
        i = _find_next_comma(val)
        values.append(parse_value(val[:i]))
        val = val[i + 1:]
    return tuple(values) if is_tuple else values


def parse_options(items):
    """['a.b=1', 'c=[x,y]'] -> {'a.b': 1, 'c': ['x', 'y']} (DictAction.__call__)."""
    out = {}
    for kv in items or []:
        key, val = kv.split('=', 1)
        out[key] = parse_value(val)
    return out


def merge_options(cfg, options):
    """Config.merge_from_dict: every dotted key replaces one value, creating the nested dicts on its way."""
    for dotted, v in options.items():
        d = cfg
        keys = dotted.split('.')
        for k in keys[:-1]:
            if not isinstance(d.get(k), dict):
                d[k] = AttrDict()
            d = d[k]
        d[keys[-1]] = AttrDict(v) if isinstance(v, dict) else v
    return cfg
