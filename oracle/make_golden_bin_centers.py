"""Pins oracle/bin_centers_oracle.py (seed_bins, attractor_update_normed, the typed metric_head)
against the reference and writes tests/golden/bin_centers_*.   python -m oracle.make_golden_bin_centers
(needs $PATCHFUSION_REFERENCE)

- Layers: SeedBinRegressor / SeedBinRegressorUnnormed (localbins_layers.py:29-103) with `_net` replaced by its last
  activation (nn.ReLU / nn.Softplus), so the pre-activation is an input, and AttractorLayer (attractor.py:60-136) with
  `_net` replaced by nn.ReLU(), in every (kind, type) pair at nA = 16, 1, B = 2, centres up-sampled 3 x 4 -> 5 x 6.
  Seeded inputs and adversarial ones: all-negative and all-zero seed outputs, one dominant bin; b_prev outside
  [0, 1], reversed, interleaved, tied and all-equal (the sort and the clip decide the output).
- Model: a vits PatchFusion (rh.build_reference) with synthetic_state_dict for each case of CASES at 1080 x 1920,
  2 x 2 tiles: the coarse, fine and fusion heads' final centres and depths on two tiles, and forward(mode='infer',
  m1).  Branch and top-level depth ranges all differ, so a head reading the wrong range shows.
- The reference's state-dict layout for each case: its keys equal tests/golden/state_dict_layout_vits.json's (asserted),
  and the shapes that differ are stored.
"""
import json
import os
import random
import sys

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import bin_centers_oracle as bco  # noqa: E402
from oracle import pf_oracle as po          # noqa: E402
from oracle import ref_harness as rh        # noqa: E402
from oracle.make_golden import sample       # noqa: E402
from patchfusion_b200.configs import depth_anything_patchfusion      # noqa: E402
from patchfusion_b200.params import synthetic_state_dict             # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
B, NBINS, SRC, DST = 2, 64, (3, 4), (5, 6)
N_ATTRACTORS = (16, 1)
PAIRS = (('mean', 'inv'), ('sum', 'inv'), ('mean', 'exp'), ('sum', 'exp'))
LAYER_RANGE = (0.01, 20.0)
# (coarse type, fine type); depth ranges: top-level (fusion head), coarse branch, fine branch
CASES = {'normed': ('normed', 'normed'), 'hybrid1': ('hybrid1', 'hybrid1'), 'hybrid2': ('hybrid2', 'hybrid2'),
         'mixed': ('normed', 'softplus')}
RANGES = dict(top=(0.05, 40.0), coarse=(1e-3, 80.0), fine=(0.01, 60.0))
# hybrid2's fine head: its softplus seed centres are a few metres, so at (0.01, 60) the normalised centres sit near 0
# and the output stays within a few percent of a softplus head's; at (0.01, 2) they spread over [0, 1.5], where the
# attractors and the clip act
CASE_RANGES = {'hybrid2': dict(fine=(0.01, 2.0))}
MODEL = dict(encoder='vits', seed=0, image_raw_shape=(1080, 1920), patch_split_num=(2, 2), process_num=2, input_seed=0,
             sample_stride=4, infer_stride=8, center_channels=16)


def case_config(name):
    ct, ft = CASES[name]
    cfg = depth_anything_patchfusion(MODEL['encoder'], image_raw_shape=MODEL['image_raw_shape'],
                                     patch_split_num=MODEL['patch_split_num'])
    cfg['min_depth'], cfg['max_depth'] = RANGES['top']
    for b, t in (('coarse', ct), ('fine', ft)):
        cfg[b + '_branch']['bin_centers_type'] = t
        cfg[b + '_branch']['min_depth'], cfg[b + '_branch']['max_depth'] = CASE_RANGES.get(name, {}).get(b, RANGES[b])
    return cfg


def case_inputs(name):
    cfg = case_config(name)
    sd = synthetic_state_dict(cfg, seed=MODEL['seed'])
    g = torch.Generator().manual_seed(MODEL['input_seed'])
    img = torch.rand(1, 3, *MODEL['image_raw_shape'], generator=g)
    return cfg, sd, img


# ------------------------------------------------------------------------------------------------ layer level
def layer_inputs():
    g = torch.Generator().manual_seed(1)
    s = torch.randn(B, NBINS, *SRC, generator=g)
    s_adv = torch.randn(B, NBINS, *SRC, generator=g)
    s_adv[0, :, 0, 0] = -1.0                       # every width 1e-3: uniform bins
    s_adv[0, :, 0, 1] = 0.0
    s_adv[0, :, 1, 0] = -1.0
    s_adv[0, 17, 1, 0] = 1e4                       # one bin takes nearly the whole range
    s_adv[1] = s_adv[1].abs() * 1e-3               # widths dominated by the 1e-3
    b_prev = torch.rand(B, NBINS, *SRC, generator=g)
    adv = torch.rand(B, NBINS, *SRC, generator=g) * 1.6 - 0.3                     # outside [0, 1], unsorted
    adv[0, :, 0, 0] = torch.linspace(1.2, -0.2, NBINS)                           # reversed
    adv[0, :, 0, 1] = torch.where(torch.arange(NBINS) % 2 == 0, 0.1, 0.9)        # interleaved, ties
    adv[0, :, 1, 0] = 0.5                                                         # all equal
    adv[1, :, 2, 3] = torch.floor(torch.rand(NBINS, generator=g) * 4) / 3        # four tied levels
    A2 = torch.randn(B, 2 * max(N_ATTRACTORS), *DST, generator=g) * 0.5 + 0.4     # ReLU'd inside the layer
    A2_adv = torch.randn(B, 2 * max(N_ATTRACTORS), *DST, generator=g) * 0.8 + 0.2
    A2_adv[:, 1::2] += 5.0                        # odd channels far from the bins: reading them moves b_new
    return dict(seed_s=s, seed_s_adv=s_adv, att_b_prev=b_prev, att_b_prev_adv=adv, att_A2=A2, att_A2_adv=A2_adv)


def savez(path, arrays):
    """np.savez_compressed with fixed member order and timestamps, so two runs write identical bytes"""
    import io
    import zipfile
    with zipfile.ZipFile(path, 'w', zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[k]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + '.npy', date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(),
                       compress_type=zipfile.ZIP_DEFLATED)


def _err(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def layers(out):
    rh._enter()
    from zoedepth.models.layers.attractor import AttractorLayer
    from zoedepth.models.layers.localbins_layers import SeedBinRegressor, SeedBinRegressorUnnormed
    x = layer_inputs()
    out.update({k: v.numpy() for k, v in x.items()})
    lo, hi = LAYER_RANGE
    with torch.no_grad():
        for tag in ('', '_adv'):
            s = x['seed_s' + tag]
            for normed in (True, False):
                layer = (SeedBinRegressor if normed else SeedBinRegressorUnnormed)(8, NBINS, min_depth=lo, max_depth=hi)
                layer._net = nn.ReLU() if normed else nn.Softplus()
                _, c = layer(s)
                act = F.relu(s) if normed else F.softplus(s)
                for to_unit in (False, True):
                    ref = (c - lo) / (hi - lo) if to_unit else c
                    mine = bco.seed_bins(act, lo, hi, normed, to_unit)
                    e = _err(mine, ref)
                    key = 'seed%s_%s%s' % (tag, 'normed' if normed else 'unnormed', '_unit' if to_unit else '')
                    print('%s: oracle vs reference %.2e' % (key, e))
                    assert e <= 1e-6, key
                    out[key] = ref.numpy()
            for kind, typ in PAIRS:
                for nA in N_ATTRACTORS:
                    layer = AttractorLayer(8, NBINS, nA, min_depth=lo, max_depth=hi, kind=kind, attractor_type=typ)
                    layer._net = nn.ReLU()
                    A2 = x['att_A2' + tag][:, :2 * nA].contiguous()
                    b_ref, c_ref = layer(A2, x['att_b_prev' + tag])
                    b_mine, c_mine = bco.attractor_update_normed(F.relu(A2), x['att_b_prev' + tag], lo, hi, kind, typ)
                    e = max(_err(b_mine, b_ref), _err(c_mine, c_ref))
                    key = 'att%s_%s_%s_%d' % (tag, kind, typ, nA)
                    print('%s: oracle vs reference %.2e' % (key, e))
                    assert e <= 1e-6, key
                    out[key + '_b'], out[key + '_centers'] = b_ref.numpy(), c_ref.numpy()


# ------------------------------------------------------------------------------------------------ model level
class _LastAttractor:
    """forward hook on a head's last attractor: its (b, centres) outputs of the latest call"""

    def __init__(self, module):
        self.out = None
        module.register_forward_hook(self)

    def __call__(self, module, inp, output):
        self.out = output


def _centers(hook, typ, taps, cc):
    """the centres the expectation reads (ZD:217-219): sorted metric for AttractorLayer, b_new otherwise; every cc-th
    channel of the reference's (hook) and the oracle's (taps)"""
    b, c = hook.out
    normed = typ in ('normed', 'hybrid2')
    return (c if normed else b)[:, ::cc], taps['centers' if normed else 'b3'][:, ::cc]


def model_case(name, out):
    st, sc, cc = MODEL['sample_stride'], MODEL['infer_stride'], MODEL['center_channels']
    cfg, sd, img = case_inputs(name)
    ref = rh.build_reference(MODEL['encoder'], cfg)
    print(name, ref.load_state_dict(sd, strict=True))
    ct, ft = CASES[name]
    hooks = dict(coarse=_LastAttractor(ref.coarse_branch.attractors[3]),
                 fine=_LastAttractor(ref.fine_branch.attractors[3]), fusion=_LastAttractor(ref.attractors[3]))
    orc = po.Oracle(sd, cfg)
    lr = ref.resizer(img)
    p = name + '_'

    def keep(key, ref_t, mine, tol, stride):
        e = _err(mine, ref_t)
        print('%s%s: oracle vs reference %.2e (max |ref| %.3g)' % (p, key, e, ref_t.abs().max().item()))
        assert e <= tol, key
        out[p + key] = sample(ref_t, stride)

    with torch.no_grad(), bco.typed_heads(cfg):
        taps = {}
        d_ref, f_ref = ref.coarse_forward(lr)
        d_o, f_o = orc.coarse(lr, taps)
        keep('coarse_depth', d_ref, d_o, 1e-5, st)
        keep('coarse_centers', *_centers(hooks['coarse'], ct, taps, cc), 1e-5, st)
        H, W = MODEL['image_raw_shape']
        h, w = H // 2, W // 2
        raw = [(0, 0), (h // 2, w // 2)]
        P = cfg['patch_process_shape']
        fx, fy = 1 / W * P[1], 1 / H * P[0]
        boxes = torch.tensor([[x, y, x + w, y + h] for (y, x) in raw]).int() * torch.tensor([[fx, fy, fx, fy]])
        bf = torch.cat([torch.arange(2).unsqueeze(1).float(), boxes], 1)
        post = ref.coarse_postprocess_test(bboxs=None, bboxs_feat=bf, coarse_prediction=d_ref, coarse_features=f_ref)
        crops = torch.cat([ref.resizer(img[:, :, y:y + h, x:x + w]) for (y, x) in raw])
        fd_ref, ff_ref = ref.fine_forward(crops)
        taps = {}
        fd_o, ff_o = po.branch_forward(sd, 'fine_branch.', crops, cfg['fine_branch'], taps)
        keep('fine_depth', fd_ref, fd_o, 1e-5, st)
        keep('fine_centers', *_centers(hooks['fine'], ft, taps, cc), 1e-5, st)
        bff = bf.clone()
        bff[:, 0] = 0
        fu_ref, _ = ref.fusion_forward(fd_ref, crops, f_ref, ff_ref, bff, **post)
        rois_o = [po.roi_crop_zoom(f, boxes, f.shape[-2] / P[0]) for f in f_o]
        g2l = po.g2l_all(sd, f_o, cfg['guided_fusion'])
        taps = {}
        fu_o = po.fusion_forward(sd, cfg, fd_o, crops, ff_o, boxes, po.roi_crop_zoom(d_o, boxes, 1.0), rois_o, g2l, taps)
        keep('fusion_depth', fu_ref, fu_o, 1e-3, st)
        keep('fusion_centers', *_centers(hooks['fusion'], ct, taps, cc), 1e-3, st)
        random.seed(0)
        y_ref, _ = ref(mode='infer', image_lr=lr, image_hr=img, cai_mode='m1', process_num=MODEL['process_num'])
        random.seed(0)
        y_o = orc.infer(lr, img, cai_mode='m1', process_num=MODEL['process_num'])
        keep('infer_m1', y_ref, y_o, 1e-3, sc)


def layouts():
    """per case, the reference's state-dict entries whose shape differs from the softplus layout of
    tests/golden/state_dict_layout_vits.json; keys, their order and dtypes are the same (asserted)"""
    base = json.load(open(os.path.join(GOLD, 'state_dict_layout_vits.json')))
    out = {}
    for name in CASES:
        sd = rh.build_reference(MODEL['encoder'], case_config(name)).state_dict()
        assert list(sd) == list(base) and all(str(v.dtype)[6:] == base[k][1] for k, v in sd.items()), name
        out[name] = {k: list(v.shape) for k, v in sd.items() if list(v.shape) != base[k][0]}
    return out


def main():
    """all fixtures; `layers` writes only the layer-level archive and the layouts"""
    torch.set_num_threads(os.cpu_count())
    names = sys.argv[1:] or list(CASES)
    out = {}
    layers(out)
    savez(os.path.join(GOLD, 'bin_centers_layers.npz'), out)
    with open(os.path.join(GOLD, 'bin_centers.json'), 'w') as f:
        json.dump(dict(model=MODEL, ranges=RANGES, case_ranges=CASE_RANGES, cases=CASES, layouts=layouts()), f)
    for name in names if names != ['layers'] else []:
        out = {}
        model_case(name, out)
        savez(os.path.join(GOLD, 'bin_centers_%s.npz' % name), out)
    print('wrote', sorted(f for f in os.listdir(GOLD) if f.startswith('bin_centers')))


if __name__ == '__main__':
    main()
