"""The normed / hybrid bin-centre heads on the CPU: the state-dict layout of each bin_centers_type against the
reference's, oracle/bin_centers_oracle.py against the reference's own layers and models (fixtures of
oracle/make_golden_bin_centers.py), and the fp64 references and kernel emulations of tests/bin_centers_ref.py within
their bounds, with every planted bug landing >= 4x above its bound."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import bin_centers_ref as cr
import bins_ref as br

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
CASE_NAMES = ['normed', 'hybrid1', 'hybrid2', 'mixed']
pytestmark = pytest.mark.timeout(900)


def _gold(name):
    return dict(np.load(os.path.join(GOLD, 'bin_centers_%s.npz' % name)))


@pytest.mark.parametrize('name', CASE_NAMES)
def test_layout_matches_reference(name):
    """the softplus layout with the reference's shapes for this case (its keys, order and dtypes are the same)"""
    from oracle.make_golden_bin_centers import case_config
    from patchfusion_b200.params import state_layout
    ref = json.load(open(os.path.join(GOLD, 'state_dict_layout_vits.json')))
    for k, shape in json.load(open(os.path.join(GOLD, 'bin_centers.json')))['layouts'][name].items():
        ref[k][0] = shape
    L = state_layout(case_config(name))
    assert list(L.keys()) == list(ref.keys())
    assert all(list(shape) == ref[k][0] and str(dt)[6:] == ref[k][1] for k, (shape, dt, _) in L.items())


def test_refusals_stay():
    from patchfusion_b200.configs import depth_anything_patchfusion
    from patchfusion_b200.params import state_layout
    for key, val, exc in (('bin_centers_type', 'nope', ValueError), ('inverse_midas', True, NotImplementedError),
                          ('do_resize', True, NotImplementedError)):
        for b in ('coarse_branch', 'fine_branch'):
            cfg = depth_anything_patchfusion('vits')
            cfg[b][key] = val
            with pytest.raises(exc):
                state_layout(cfg)


def test_model_state_dict_round_trip():
    """load_dict / get_save_dict keep the full 2 nA attractor tensors of a normed head"""
    from oracle.make_golden_bin_centers import case_config
    from patchfusion_b200.model import PatchFusion
    from patchfusion_b200.params import synthetic_state_dict
    cfg = case_config('normed')
    m = PatchFusion(cfg)
    sd = synthetic_state_dict(cfg, seed=1)
    m.load_state_dict(sd, strict=True)
    assert tuple(m.state_dict()['attractors.0._net.2.weight'].shape) == (32, 128, 1, 1)
    m2 = PatchFusion(cfg)
    m2.load_dict(m.get_save_dict())
    assert torch.equal(m2.state_dict()['attractors.3._net.2.weight'], sd['attractors.3._net.2.weight'])


# ------------------------------------------------------------------------------------------------------ oracle
def test_oracle_layers_against_reference():
    from oracle import bin_centers_oracle as bco
    from oracle.make_golden_bin_centers import LAYER_RANGE, N_ATTRACTORS, PAIRS
    g = dict(np.load(os.path.join(GOLD, 'bin_centers_layers.npz')))
    lo, hi = LAYER_RANGE
    close = lambda got, key, scale: np.abs(got.numpy() - g[key]).max() <= 1e-6 * scale     # noqa: E731
    for tag in ('', '_adv'):
        s = torch.tensor(g['seed_s' + tag])
        for normed in (True, False):
            for unit in (False, True):
                key = 'seed%s_%s%s' % (tag, 'normed' if normed else 'unnormed', '_unit' if unit else '')
                got = bco.seed_bins(F.relu(s) if normed else F.softplus(s), lo, hi, normed, unit)
                assert close(got, key, np.abs(g[key]).max()), key
        for kind, typ in PAIRS:
            for nA in N_ATTRACTORS:
                key = 'att%s_%s_%s_%d' % (tag, kind, typ, nA)
                A2 = F.relu(torch.tensor(g['att_A2' + tag])[:, :2 * nA])
                b, c = bco.attractor_update_normed(A2, torch.tensor(g['att_b_prev' + tag]), lo, hi, kind, typ)
                assert close(b, key + '_b', np.abs(g[key + '_b']).max()) and close(c, key + '_centers', hi), key


def _tiles(cfg, img, orc):
    from oracle.make_golden_bin_centers import MODEL
    H, W = MODEL['image_raw_shape']
    h, w = H // 2, W // 2
    raw = [(0, 0), (h // 2, w // 2)]
    P = cfg['patch_process_shape']
    fx, fy = 1 / W * P[1], 1 / H * P[0]
    boxes = torch.tensor([[x, y, x + w, y + h] for (y, x) in raw]).int() * torch.tensor([[fx, fy, fx, fy]])
    return torch.cat([orc.resizer(img[:, :, y:y + h, x:x + w]) for (y, x) in raw]), boxes


@pytest.fixture(scope='module')
def heads():
    """per case: the oracle's coarse depth and taps, and (mixed, hybrid2) the arguments of its fusion head on the
    fixture's two tiles and the fusion depth"""
    from oracle import bin_centers_oracle as bco
    from oracle import pf_oracle as po
    from oracle.make_golden_bin_centers import CASES, case_inputs
    torch.set_num_threads(os.cpu_count())
    out = {}
    for name in CASES:
        cfg, sd, img = case_inputs(name)
        orc = po.Oracle(sd, cfg)
        taps, seen = {}, {}
        with torch.no_grad(), bco.typed_heads(cfg):
            d, f = orc.coarse(orc.resizer(img), taps)
            out[name] = dict(cfg=cfg, coarse=(d, taps))
            if name not in ('mixed', 'hybrid2'):
                continue
            crops, boxes = _tiles(cfg, img, orc)
            fd, ff = po.branch_forward(sd, 'fine_branch.', crops, cfg['fine_branch'])
            rois = [po.roi_crop_zoom(t, boxes, t.shape[-2] / cfg['patch_process_shape'][0]) for t in f]
            g2l = po.g2l_all(sd, f, cfg['guided_fusion'])
            typed = po.metric_head

            def capture(*a):
                seen['args'] = a
                return typed(*a)
            po.metric_head = capture
            try:
                fu = po.fusion_forward(sd, cfg, fd, crops, ff, boxes, po.roi_crop_zoom(d, boxes, 1.0), rois, g2l)
            finally:
                po.metric_head = typed
            out[name].update(args=seen['args'], fusion=fu)
    return out


@pytest.mark.parametrize('name', CASE_NAMES)
def test_oracle_coarse_branch_against_reference(heads, name):
    from oracle.make_golden_bin_centers import CASES, MODEL
    st, cc = MODEL['sample_stride'], MODEL['center_channels']
    g = _gold(name)
    d, taps = heads[name]['coarse']
    assert np.abs(d[..., ::st, ::st].numpy() - g[name + '_coarse_depth']).max() < 1e-5
    c = taps['centers' if CASES[name][0] in ('normed', 'hybrid2') else 'b3'][:, ::cc, ::st, ::st].numpy()
    assert np.abs(c - g[name + '_coarse_centers']).max() < 1e-5 * np.abs(c).max()


# the fusion tolerances of tests/test_gpu_bin_centers.py (max |d - d_ref| / max_depth)
FUSION_TOL = {'mixed': 2e-2, 'hybrid2': 4e-2}


def test_oracle_fusion_head_and_planted_config_bugs(heads):
    """the oracle's fusion depth matches the fixture; a fusion head that takes the fine branch's bin_centers_type or
    the coarse branch's depth range, or a hybrid2 seed b_prev left unnormalised, misses it by >= 4x the tolerance"""
    from oracle import bin_centers_oracle as bco
    from oracle.make_golden_bin_centers import MODEL
    st = MODEL['sample_stride']

    def err(name, depth):
        c = heads[name]
        return np.abs(depth[..., ::st, ::st].numpy() - _gold(name)[name + '_fusion_depth']).max() / c['cfg']['max_depth']
    mixed, hyb = heads['mixed'], heads['hybrid2']
    assert err('mixed', mixed['fusion']) < 1e-5 and err('hybrid2', hyb['fusion']) < 1e-5
    w, x, xb, last, rel, hp = mixed['args'][:6]
    top = (mixed['cfg']['min_depth'], mixed['cfg']['max_depth'])
    real = bco.seed_bins
    with torch.no_grad():
        fine_type = dict(hp, bin_centers_type=mixed['cfg']['fine_branch']['bin_centers_type'])
        bugs = {('mixed', 'fine type'): bco.metric_head(w, x, xb, last, rel, fine_type, None, top),
                ('mixed', 'branch range'): bco.metric_head(w, x, xb, last, rel, hp)}
        bco.seed_bins = lambda S, lo, hi, normed_seed=True, to_unit=False: real(S, lo, hi, normed_seed, False)
        try:
            hyb_top = (hyb['cfg']['min_depth'], hyb['cfg']['max_depth'])
            bugs[('hybrid2', 'seed not normalised')] = bco.metric_head(*hyb['args'][:6], None, hyb_top)
        finally:
            bco.seed_bins = real
    for (name, tag), d in bugs.items():
        e = err(name, d)
        print('%s %s: %.3e (%.1fx the tolerance)' % (name, tag, e, e / FUSION_TOL[name]))
        assert e >= 4 * FUSION_TOL[name], tag


# ------------------------------------------------------------------------------------------------ kernel emulations
@pytest.mark.parametrize('rng', [(1e-3, 80.0), (0.05, 40.0), (0.01, 20.0)])
def test_seed_bins_emulation_and_planted_bugs(rng):
    lo, hi = rng
    S = cr.seed_case(6000, torch.Generator().manual_seed(3))
    for flags in (1, 2, 3):
        ref, scale = cr.seed_bins_fp64(S, lo, hi, flags & 1, flags & 2)
        e = cr.seed_error(cr.seed_bins_emulated(S, lo, hi, flags), ref, scale)
        print('flags %d: emulation %.2f of the bound' % (flags, e / cr.SEED_TOL))
        assert e <= cr.SEED_TOL / 2
        for bug in cr.PLANTED_BUGS['seed']:
            if not (flags & 2 if bug == 'no_unit' else flags & 1):       # the step the bug breaks is not run
                continue
            eb = cr.seed_error(cr.seed_bins_emulated(S, lo, hi, flags, bug), ref, scale)
            print('   %s: %.3g x the bound' % (bug, eb / cr.SEED_TOL))
            assert eb >= 4 * cr.SEED_TOL, (flags, bug)


# the input that makes each attractor bug visible: the odd channels and the 1e-3 change b everywhere, the sort needs
# unsorted centres, the clip centres outside [0, 1]
BUG_ORDERS = {'odd_channels': 'sorted', 'eps_dropped': 'sorted', 'sort_skipped': 'interleaved', 'clip_skipped': 'outside'}


@pytest.mark.parametrize('level', range(3))
def test_attractor_normed_emulation_and_planted_bugs(level):
    hw, HW, nA = br.CHAIN[level]
    gen = torch.Generator().manual_seed(40 + level)
    for order in cr.ORDERS:
        A2, _, b_prev = cr.attractor_normed_case(1, hw, HW, nA, gen, order)
        for flags in range(4):
            kind, typ = br.ATTRACTOR_FLAGS[flags]
            b64, c64, _ = cr.attractor_normed_fp64(A2, nA, b_prev, 1e-3, 80.0, kind, typ)
            errs = lambda bug=None: cr.attractor_errors(                                        # noqa: E731
                *cr.attractor_normed_emulated(A2, nA, b_prev, flags, 1e-3, 80.0, bug), b64, c64, 1e-3, 80.0, hw, nA, kind)
            assert max(errs()) <= 1, (order, flags)
            for bug in [b for b, o in BUG_ORDERS.items() if o == order]:
                print('level %d %s flags %d: %s %.3g x the bound' % (level, order, flags, bug, max(errs(bug))))
                assert max(errs(bug)) >= 4, (bug, flags)
