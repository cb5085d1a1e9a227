"""The stage workspace contract: a stage reads only workspace bytes it wrote in the same call, and writes only below the
end of its last allocation (need - 256 of pf_*_workspace_bytes).

Every intermediate of pf_branch_forward / pf_g2l_forward / pf_fusion_forward is bump-allocated from one caller-owned
workspace that nothing clears (Engine.arena is torch.empty).  The GEMM and conv kernels read each source's channels
[C, pad8(C)) (the e4m3 convs: [C, pad64(C))) and multiply them by zero weights, so a producer that leaves its pad columns
unwritten hands NaN to the output whenever the memory held NaN.  On a zeroed workspace such a read returns exactly the
clean result, which is why the tests here fill the workspace bytewise with

    0xFF  NaN in bf16, fp32 and e4m3: any read that is multiplied, added or accumulated, times a zero weight included;
    0x40  3.0 (bf16), 3.00390625 (fp32), 2.0 (e4m3): reads NaN cannot show (fmaxf drops NaN, so a stale value behind
          a ReLU epilogue or pf_maxpool2 stays invisible with NaN),

and require the same bits as the same call on a zeroed workspace: outputs, every debug tap over its logical columns
(the e4m3 maps over their full padded width, whose pad bytes must be 0), the bytes past the last allocation and those
before the stage's offset untouched.  Then: calibration tables and whole-model forwards (graph replays over every
poisoned arena) unchanged, and a workspace declared too small refused before any launch lands past it."""
import gc
import json
import os
import random
import re

import pytest
import torch

from test_gpu_gemm_exact import _Opt

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
FILLS = {'nan': 0xFF, 'three': 0x40}
SLACK = 64 << 10            # bytes of the arena past `need`
OFF = 768                   # the stage's byte offset in a poisoned arena: [0, OFF) must stay untouched
BOXES = [(0, 0, .5, .5), (.25, .25, .75, .75), (.5, .5, 1, 1), (.02, .01, .58, .51), (0, 0, 1, 1)]
TILE_IMAGE = [2, 0, 1, 1, 2]
STATIC = dict(fusion_precision='fp8_static', vit_precision='fp8_static', dpt_precision='fp8_static')


def _bits(t):
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def _same_bits(tag, got, want):
    assert got.shape == want.shape and got.dtype == want.dtype, (tag, got.shape, want.shape, got.dtype, want.dtype)
    diff = (_bits(got) != _bits(want)).nonzero()
    assert diff.numel() == 0, '%s: %d elements differ from the zeroed-workspace run, first at %s (%s vs %s)' % (
        tag, diff.shape[0], diff[0].tolist(), got[tuple(diff[0])].item(), want[tuple(diff[0])].item())


# ---------------------------------------------------------------------------------------------------- models
def _vits_case():
    from oracle.make_golden import case_inputs
    return case_inputs(json.load(open(os.path.join(GOLD, 'vits_case0.json'))))


def _patchfusion(cfg, sd, cuda):
    from patchfusion_b200.model import PatchFusion
    m = PatchFusion(cfg)
    m.load_state_dict(sd, strict=True)
    return m.to(cuda).eval()


def _build(key, cuda):
    """vits / fp8 / static (all three 'fp8_static' paths, calibrated) on the vits_case0 weights, vitb / vitl on seeded
    synthetic weights, normed / hybrid1 / hybrid2 on the bin-centre fixture weights"""
    from patchfusion_b200.configs import depth_anything_patchfusion
    from patchfusion_b200.params import synthetic_state_dict
    if key in ('vits', 'fp8', 'static'):
        cfg, sd, _ = _vits_case()
        cfg = dict(cfg, **{'vits': {}, 'fp8': dict(fusion_precision='fp8'), 'static': STATIC}[key])
    elif key in ('vitb', 'vitl'):
        cfg = depth_anything_patchfusion(key)
        sd = synthetic_state_dict(cfg, seed=0)
    else:
        from oracle.make_golden_bin_centers import case_inputs
        cfg, sd, _ = case_inputs(key)
    m = _patchfusion(cfg, sd, cuda)
    if key == 'static':
        cal = torch.rand(2, 3, 1080, 1920, generator=torch.Generator().manual_seed(7)).to(cuda)
        random.seed(1)
        m.calibrate_fp8(m.make_lr(cal), cal, cai_mode='m1', process_num=2)
    return m


class _Models:
    """The model of the last key asked for (building another drops it).  release() drops its engine (packed panels,
    arenas, graphs) and the coarse views into them, then hands the freed memory back to the driver: the suite may share
    the GPU with other test processes, and these tests' workspaces run to gigabytes."""

    def __init__(self, cuda):
        self.cuda, self.key, self.model = cuda, None, None

    def __call__(self, key):
        if key != self.key:
            self.model = self.key = None
            self.release()
            self.model, self.key = _build(key, self.cuda), key
        return self.model

    def release(self):
        if self.model is not None:
            self.model.invalidate()
            self.model._coarse = None
        gc.collect()
        torch.cuda.empty_cache()


@pytest.fixture(scope='module')
def models(cuda):
    m = _Models(cuda)
    yield m
    m.model = m.key = None
    m.release()


@pytest.fixture(autouse=True)
def _release_after(models):
    yield
    models.release()


def _rand(shape, seed):
    return torch.rand(shape, generator=torch.Generator(device='cuda').manual_seed(seed), device='cuda')


def _clone_maps(maps):
    from patchfusion_b200.engine import Map
    return [Map(m.t.clone(), m.C) for m in maps]


def _fusion_inputs(eng, T, B):
    """crops, boxes, fine depth / maps, coarse depth / maps and G2L maps of a B-image coarse batch (cloned out of the
    engine's own arenas), and the tiles' images (None when B = 1)"""
    H, W = eng.P
    cd, cf = eng.branch('coarse', _rand((B, 3, H, W), 10 + B))
    cd, cf = cd.clone(), _clone_maps(cf)
    g2l = _clone_maps(eng.g2l(cf))
    crops = _rand((T, 3, H, W), 20 + T)
    fd, ff = eng.branch('fine', crops)
    fd, ff = fd.clone(), _clone_maps(ff)
    boxes = torch.tensor([[x1 * W, y1 * H, x2 * W, y2 * H] for (x1, y1, x2, y2) in BOXES[:T]], device='cuda')
    ti = torch.tensor(TILE_IMAGE[:T], dtype=torch.int32, device='cuda') if B > 1 else None
    torch.cuda.synchronize()
    eng.arenas.clear()          # the stage under test runs on the test's own arena
    torch.cuda.empty_cache()
    return crops, boxes, fd, ff, cd if B > 1 else cd[0].contiguous(), cf, g2l, ti


# ---------------------------------------------------------------------------------------------------- e4m3 pad bytes
def _pad64(c):
    return (c + 63) // 64 * 64


def _e4m3_channels(eng, which, name):
    """the logical channel counts of the sources packed (each padded to 64) into e4m3 tap `name`, or None for a map
    without pad bytes (the ViT operands: D and 4 D are multiples of 64)"""
    parts = name.split('.')
    if parts[0] == 'e4m3s':                       # e4m3s.<layer>.<in|out>.<H>x<W> (fusion U-Net)
        pw = eng.W['fusion']['.'.join(parts[1:3])]
        return list(pw.src_c) if parts[3] == 'in' else [pw.N]
    if parts[0] == 'e4m3d':                       # e4m3d.<conv>.<in|out|copy> (DPT decoder of `which`)
        conv, part = '.'.join(parts[1:-1]), parts[-1]
        if part == 'copy':
            return [eng.hp[which]['features']]
        if conv.startswith('layer'):
            key = 'rn%d' % (int(conv[5]) - 1)
        elif conv == 'output_conv1':
            key = 'oc1'
        else:
            key = 'ff%s.u%s.c%s' % re.fullmatch(r'refinenet(\d)\.resConfUnit(\d)\.conv(\d)', conv).groups()
        pw = eng.W[which][key]
        return list(pw.src_c) if part == 'in' else [pw.N]
    assert parts[0] == 'e4m3v', name
    return None


def _check_e4m3_pads(eng, which, taps):
    n = 0
    for name, t in taps.items():
        if t.dtype != torch.uint8:
            continue
        chans = _e4m3_channels(eng, which, name)
        if chans is None:
            continue
        assert t.shape[-1] == sum(_pad64(c) for c in chans), (name, t.shape, chans)
        o = 0
        for c in chans:
            pad = t[..., o + c:o + _pad64(c)]
            assert (pad == 0).all(), '%s: %d non-zero pad bytes in channels [%d, %d)' % (
                name, (pad != 0).sum().item(), o + c, o + _pad64(c))
            o += _pad64(c)
        n += 1
    return n


# ---------------------------------------------------------------------------------------------------- stage runs
def _on_arena(run, need, fill, off):
    """run((arena, off)) -> {name: tensor} on an arena of off + need + SLACK bytes filled with `fill`; the bytes before
    `off` and past the last allocation must still hold it"""
    arena = torch.full((off + need + SLACK,), fill, dtype=torch.uint8, device='cuda')
    out = run((arena, off))
    torch.cuda.synchronize()
    before = (arena[:off] != fill).nonzero()
    assert before.numel() == 0, 'wrote %d bytes before the stage offset %d, first at %d' % (
        before.shape[0], off, before[0].item())
    after = (arena[off + need - 256:] != fill).nonzero()
    assert after.numel() == 0, 'wrote %d bytes past the last allocation (need %d), first at need - 256 + %d' % (
        after.shape[0], need, after[0].item())
    return out


def _check_stage(tag, run, need, eng=None, which=None):
    clean = _on_arena(run, need, 0, 0)
    for k, v in clean.items():
        if v.is_floating_point():
            assert torch.isfinite(v.float()).all(), '%s: %s is not finite on a zeroed workspace' % (tag, k)
    n8 = _check_e4m3_pads(eng, which, {k[4:]: v for k, v in clean.items() if k.startswith('tap.')}) if eng else 0
    for pname, fill in FILLS.items():
        got = _on_arena(run, need, fill, OFF)
        assert sorted(got) == sorted(clean), tag
        for k in clean:
            _same_bits('%s %s: %s' % (tag, pname, k), got[k], clean[k])
        del got
    print('%s: %d tensors (%d e4m3 maps) bit-identical on NaN- and 3.0-poisoned workspaces, need %d bytes' %
          (tag, len(clean), n8, need))


def _branch_run(eng, which, imgs):
    seq = (eng.P[0] // 14) * (eng.P[1] // 14) + 1

    def run(ws):
        taps = {}
        d, feats = eng.branch(which, imgs, taps, ws=ws)
        for k in [k for k in taps if k.endswith('.qkv.vt')]:
            taps[k] = taps[k][:, :seq]      # V^T [B D, seq_pad]: the attention kernel reads only the seq columns
        out = {'depth': d.clone()}
        for i, f in enumerate(feats):
            assert (f.t[..., f.C:] == 0).all(), 'map %d: pad columns [%d, %d) not zero' % (i, f.C, f.t.shape[-1])
            out['feat%d' % i] = f.t[..., :f.C].clone()
        out.update({'tap.' + k: v for k, v in taps.items()})
        return out
    return run, eng.branch_bytes(which, imgs.shape[0])


BRANCH_CASES = [('vits', 'coarse', 1), ('vits', 'fine', 1), ('vits', 'coarse', 3), ('vits', 'fine', 3),
                ('vitb', 'fine', 1), ('vitl', 'coarse', 1), ('static', 'coarse', 1), ('static', 'fine', 3),
                ('normed', 'coarse', 1), ('hybrid1', 'coarse', 1), ('hybrid2', 'fine', 1)]


@pytest.mark.parametrize('key,which,B', BRANCH_CASES, ids=['%s-%s-B%d' % c for c in BRANCH_CASES])
def test_branch_workspace(cuda, models, key, which, B):
    eng = models(key).engine()
    imgs = _rand((B, 3) + eng.P, B)
    run, need = _branch_run(eng, which, imgs)
    _check_stage('%s %s branch B=%d' % (key, which, B), run, need, eng, which)


@pytest.mark.parametrize('B', [1, 3])
def test_g2l_workspace(cuda, models, B):
    """Engine.g2l places the stage at the start of eng.arenas['g2l']: a view of the test's arena at OFF"""
    from patchfusion_b200 import stage
    eng = models('vits').engine()
    cd, cf = eng.branch('coarse', _rand((B, 3) + eng.P, 30 + B))
    cf = _clone_maps(cf)
    need = stage.g2l_workspace_bytes(eng.c_fusion, eng._pf_maps(cf))
    saved = eng.arenas.get('g2l')

    def run(ws):
        arena, off = ws
        eng.arenas['g2l'] = arena[off:]
        out = {}
        for i, m in enumerate(eng.g2l(cf)):
            assert m.t.shape[0] == B and (m.t[..., m.C:] == 0).all(), i
            out['g2l%d' % i] = m.t[..., :m.C].clone()
        return out
    try:
        _check_stage('g2l B=%d' % B, run, need)
    finally:
        if saved is None:
            eng.arenas.pop('g2l', None)
        else:
            eng.arenas['g2l'] = saved


FUSION_CASES = [('vits', 1, 1, 0), ('vits', 5, 3, 0), ('vits', 2, 1, 1), ('fp8', 2, 1, 0), ('fp8', 2, 1, 1),
                ('static', 2, 1, 0), ('static', 2, 1, 1), ('vitl', 2, 1, 0), ('normed', 2, 1, 0),
                ('hybrid1', 2, 1, 0), ('hybrid2', 2, 1, 0)]


@pytest.mark.parametrize('key,T,B,fused', FUSION_CASES,
                         ids=['%s-T%d-B%d%s' % (k, t, b, '-fused' if f else '') for k, t, b, f in FUSION_CASES])
def test_fusion_workspace(cuda, models, key, T, B, fused):
    """T tiles over a B-image coarse batch (T = 5: tile_image [2, 0, 1, 1, 2]); fused: PF_OPT_FUSED_RESAMPLE = 1"""
    from patchfusion_b200 import lib
    eng = models(key).engine()
    crops, boxes, fd, ff, cd, cf, g2l, ti = _fusion_inputs(eng, T, B)

    def run(ws):
        taps = {}
        out = torch.full((T,) + eng.P, float('nan'), device='cuda')
        eng.fusion(crops, boxes, fd, ff, cd, cf, g2l, taps=taps, depth_out=out, ws=ws, tile_image=ti)
        return dict(depth=out, **{'tap.' + k: v for k, v in taps.items()})
    with _Opt(lib.OPT_FUSED_RESAMPLE, fused, default=0):
        _check_stage('%s fusion T=%d B=%d%s' % (key, T, B, ' fused resample' if fused else ''), run,
                     eng.fusion_bytes(T, g2l), eng, 'fusion')


# ---------------------------------------------------------------------------------------------------- too small
def _direct(eng, kind):
    """(need, call(arena, ws_bytes) -> [outputs]) of one stage entry point called directly at a declared size"""
    from patchfusion_b200 import stage
    H, W = eng.P
    if kind == 'branch':
        B = 3
        imgs = _rand((B, 3, H, W), 40)
        cb = eng._branch_struct('fine')

        def call(arena, nbytes):
            o = stage.branch_forward(cb, imgs, B, arena.data_ptr(), nbytes)
            return [eng._view(arena, o.depth, (B, H, W), torch.float32).clone()] + \
                [m.t.clone() for m in eng._maps(arena, o.feats)]
        return stage.branch_workspace_bytes(cb, B), call
    # the pf_map arrays are built inside each call, as Engine does: the closures keep the input maps alive
    if kind == 'g2l':
        _, cf = eng.branch('coarse', _rand((3, 3, H, W), 41))
        cf = _clone_maps(cf)
        eng.arenas.clear()

        def call(arena, nbytes):
            out = stage.g2l_forward(eng.c_fusion, eng._pf_maps(cf), arena.data_ptr(), nbytes)
            return [m.t.clone() for m in eng._maps(arena, out)]
        return stage.g2l_workspace_bytes(eng.c_fusion, eng._pf_maps(cf)), call
    crops, boxes, fd, ff, cd, cf, g2l, ti = _fusion_inputs(eng, 5, 3)
    cfu = eng._fusion_struct()

    def call(arena, nbytes):
        out = torch.full((5, H, W), float('nan'), device='cuda')
        stage.fusion_forward(cfu, crops, boxes, 5, fd, eng._pf_maps(ff), cd, eng._pf_maps(cf), eng._pf_maps(g2l),
                             arena.data_ptr(), nbytes, out, tile_image=ti)
        return [out]
    return stage.fusion_workspace_bytes(cfu, 5, eng._pf_maps(g2l)), call


@pytest.mark.parametrize('key,kind', [('vits', 'branch'), ('vits', 'g2l'), ('vits', 'fusion'), ('static', 'branch'),
                                      ('static', 'fusion')])
def test_workspace_too_small(cuda, models, key, kind):
    """A declared size of need - 257 (the last allocation no longer fits) or need / 2 raises PFError before any launch
    reaches [ws_bytes, end): the arena behind it always covers need, so a launch issued into a failed allocation lands
    in the test's own memory and shows as changed bytes.  The next, correctly sized call returns the clean bits."""
    from patchfusion_b200 import lib
    eng = models(key).engine()
    need, call = _direct(eng, kind)
    clean = call(torch.zeros(need + SLACK, dtype=torch.uint8, device='cuda'), need)
    for nbytes in (need - 257, need // 2):
        arena = torch.full((need + SLACK,), 0x40, dtype=torch.uint8, device='cuda')
        with pytest.raises(lib.PFError, match='workspace too small'):
            call(arena, nbytes)
        torch.cuda.synchronize()
        bad = (arena[nbytes:] != 0x40).nonzero()
        assert bad.numel() == 0, '%s %s, %d of %d bytes declared: %d bytes written past them, first at +%d' % (
            key, kind, nbytes, need, bad.shape[0], bad[0].item())
        for i, (g, w) in enumerate(zip(call(arena, need), clean)):
            _same_bits('%s %s output %d after a refused %d-byte call' % (key, kind, i, nbytes), g, w)
        del arena
    print('%s %s: need %d; %d and %d bytes refused, nothing written past them' % (key, kind, need, need - 257, need // 2))


# ---------------------------------------------------------------------------------------------------- calibration
def test_calibration_on_poisoned_arenas(cuda, models):
    """The U-Net (per-tile 'fp8' arithmetic), ViT and DPT calibrations reduce their taps NaN-propagating: a read of
    unwritten arena memory changes a table or makes it NaN (which calibrate_fp8 refuses)"""
    m = models('static')
    cal = torch.rand(2, 3, 1080, 1920, generator=torch.Generator().manual_seed(8)).to(cuda)
    lr = m.make_lr(cal)
    keys = ('fusion_fp8_amax', 'vit_fp8_amax', 'dpt_fp8_amax')

    def calibrate():
        random.seed(2)
        m.calibrate_fp8(lr, cal, cai_mode='r4', process_num=2, reset=True)
        return {k: dict(m.config[k]) for k in keys}
    calibrate()                                 # the arenas at their calibration sizes
    eng = m.engine()
    gen = eng.generation
    tables = {}
    for name, fill in (('clean', 0),) + tuple(FILLS.items()):
        for t in eng.arenas.values():
            t.fill_(fill)
        tables[name] = calibrate()
        assert eng.generation == gen, 'calibration reallocated an arena'
    for name in FILLS:
        for k in keys:
            assert tables[name][k] == tables['clean'][k], (name, k)
    print('calibration tables (%s) identical on zeroed, NaN- and 3.0-poisoned arenas' %
          ', '.join('%d %s' % (len(tables['clean'][k]), k) for k in keys))


# ---------------------------------------------------------------------------------------------------- model level
def _poisoned_replays(tag, engine, run):
    """run() -> output tensors; it is run until its graphs are captured over arenas that no longer grow, then again on
    arenas zeroed and filled with each pattern in place (the graphs keep their addresses).  Same bits every time."""
    run()
    run()
    eng = engine()
    gen = eng.generation
    outs = {}
    for name, fill in (('clean', 0),) + tuple(FILLS.items()):
        for t in eng.arenas.values():
            t.fill_(fill)
        outs[name] = run()
        assert eng.generation == gen, '%s: an arena was reallocated' % tag
    assert all(torch.isfinite(y).all() for y in outs['clean']), tag
    for name in FILLS:
        for i, (g, w) in enumerate(zip(outs[name], outs['clean'])):
            _same_bits('%s %s output %d' % (tag, name, i), g, w)
    print('%s: %d arenas (%d bytes) poisoned, output bit-identical' %
          (tag, len(eng.arenas), sum(t.numel() for t in eng.arenas.values())))


def _infer(model, seed, **kw):
    def run():
        random.seed(seed)
        y, _ = model(mode='infer', **kw)
        return [t.clone() for t in (y if isinstance(y, (list, tuple)) else [y])]
    return run


MODEL_CASES = ['m1', 'm2', 'r4', 'batch2', 'mixed', 'static']


@pytest.mark.parametrize('case', MODEL_CASES)
def test_model_poisoned_arenas(cuda, case):
    cfg, sd, img = _vits_case()
    model = _patchfusion(cfg if case != 'static' else dict(cfg, **STATIC), sd, cuda)
    imgs = torch.cat([img, torch.rand(1, 3, 1080, 1920, generator=torch.Generator().manual_seed(101))]).to(cuda)
    if case == 'static':
        random.seed(1)
        model.calibrate_fp8(model.make_lr(imgs), imgs, cai_mode='m1', process_num=2)
    if case in ('m1', 'm2', 'r4', 'static'):
        kw = dict(image_lr=model.make_lr(imgs[:1]), image_hr=imgs[:1], cai_mode='m2' if case == 'static' else case,
                  process_num=2)
    elif case == 'batch2':
        kw = dict(image_lr=model.make_lr(imgs), image_hr=imgs, cai_mode='r4', process_num=3)
    else:
        shapes = [((1080, 1920), (2, 2)), ((720, 1280), (2, 4)), ((540, 960), (1, 1))]
        mi = [torch.rand(1, 3, *hw, generator=torch.Generator().manual_seed(10 + i)).to(cuda)
              for i, (hw, _) in enumerate(shapes)]
        kw = dict(image_lr=model.make_lr(mi), image_hr=mi, cai_mode=['m2', 'r4', 'm1'], process_num=3,
                  tile_cfg=[{'image_raw_shape': list(hw), 'patch_split_num': list(p)} for hw, p in shapes])
    _poisoned_replays('PatchFusion %s' % case, model.engine, _infer(model, 4, **kw))


@pytest.mark.parametrize('target', ['coarse', 'fine'])
def test_baseline_pretrain_poisoned_arenas(cuda, target):
    import torch.nn.functional as F
    from oracle.make_golden import case_inputs
    from patchfusion_b200.baseline import BaselinePretrain
    from test_baseline_host import pretrain_model_cfg
    case = json.load(open(os.path.join(GOLD, 'vits_baseline0.json')))
    _, sd, img = case_inputs(case)
    kw = dict(image_raw_shape=tuple(case['image_raw_shape']), patch_split_num=tuple(case['patch_split_num']))
    cfg = pretrain_model_cfg(case['encoder'], target, **(kw if target == 'fine' else {}))
    cfg.pop('type')
    m = BaselinePretrain(**cfg)
    pre = target + '_branch.'
    m.load_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)})
    m = m.to(cuda).eval()
    img = img.to(cuda)
    if target == 'coarse':
        run = _infer(m, 0, image_lr=F.interpolate(img, (392, 518), mode='bilinear', align_corners=True), image_hr=None)
    else:
        run = _infer(m, 0, image_lr=None, image_hr=img, cai_mode='r4', process_num=2)
    _poisoned_replays('BaselinePretrain %s' % target, lambda: m._engine, run)
