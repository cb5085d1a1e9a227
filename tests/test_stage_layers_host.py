"""The expected-layer lists of tests/stage_layers_ref.py against the state dicts of vits / vitb / vitl (CPU): every conv
or linear weight belongs to exactly one bf16 layer of a stage call or to the short list of modules inference never
runs, and each layer's sources, N and fused tail match its weights' shapes."""
import collections

import pytest

import stage_layers_ref as sl

CALLS = ('coarse', 'fine', 'g2l', 'fusion')


def _cfg(enc):
    from patchfusion_b200.configs import depth_anything_patchfusion
    return depth_anything_patchfusion(enc, image_raw_shape=[1080, 1920], patch_split_num=[2, 2])


def _shapes(enc):
    """{key: shape} of the state dict: vits drawn by synthetic_state_dict, vitb / vitl from its layout (the same keys
    and shapes without allocating a ViT-L)"""
    from patchfusion_b200.params import state_layout, synthetic_state_dict
    cfg = _cfg(enc)
    if enc == 'vits':
        return {k: tuple(v.shape) for k, v in synthetic_state_dict(cfg, seed=0).items()}
    return {k: shape for k, (shape, _, _) in state_layout(cfg).items()}


@pytest.mark.parametrize('enc', ['vits', 'vitb', 'vitl'])
def test_layer_lists_cover_the_state_dict(enc):
    cfg = _cfg(enc)
    shapes = _shapes(enc)
    weights = [k[:-len('.weight')] for k, s in shapes.items() if k.endswith('.weight') and len(s) >= 2]
    used = collections.Counter(m for c in CALLS for spec in sl.layer_specs(cfg, c) for m in spec['mods'])
    used.update(sl.never_run(cfg))
    twice = sorted(m for m, n in used.items() if n > 1)
    missing = sorted(set(weights) - set(used))
    unknown = sorted(set(used) - set(weights))
    assert not twice, 'modules used twice: %s' % twice[:8]
    assert not missing, 'weights no layer computes: %s' % missing[:8]
    assert not unknown, 'layers naming modules the state dict lacks: %s' % unknown[:8]
    for c in CALLS:
        ks = [spec['key'] for spec in sl.layer_specs(cfg, c)]
        assert len(ks) == len(set(ks)), c


@pytest.mark.parametrize('enc', ['vits', 'vitb', 'vitl'])
def test_layer_shapes_match_the_weights(enc):
    cfg = _cfg(enc)
    shapes = _shapes(enc)
    for c in CALLS:
        for spec in sl.layer_specs(cfg, c):
            w = shapes[spec['mods'][0] + '.weight']
            k = spec['k']
            cin = sum(spec['srcs']) + (1 if spec.get('drop_rel') else 0)
            if spec['key'] == 'patch':
                assert (w[0], w[1] * w[2] * w[3]) == (spec['N'], cin), spec['key']
            elif isinstance(k, str) and k.startswith('T'):          # ConvTranspose2d: (in, out, k, k)
                assert (w[0], w[1], w[2]) == (cin, spec['N'], int(k[1:])), spec['key']
            else:
                taps = 3 if k in (3, 's2') else 1
                assert tuple(w) == ((spec['N'], cin) if spec['kind'] == 'linear' else (spec['N'], cin, taps, taps)), \
                    (spec['key'], w)
            if spec['tail'] is not None:
                n2 = shapes[spec['tail'] + '.weight'][0]
                assert spec['n2'] == (n2 // 2 if spec.get('even') else n2) <= 16, spec['key']
            if spec['bn'] is not None:
                assert shapes[spec['bn'] + '.running_var'] == (spec['N'],)
