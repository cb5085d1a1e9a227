"""Calibrated FP8 BaselinePretrain on the GPU: branch_vit_precision / branch_dpt_precision 'fp8_static' for the coarse and
fine targets (vits, the vits_baseline0 weights): the refusal without a table, calibration (deterministic, merged by max,
reset, a changed table), its tables against PatchFusion.calibrate_fp8's on the same branch weights, the model against
BaselineOracle under the static FP8 emulations of tests/fp8_vit_ref.py and tests/fp8_dpt_ref.py, the bit-exact
invariances, the unchanged default path, a poisoned-workspace run of an FP8 branch stage, vitl at coarse B = 32, another
input size and fine process_num 16 on the E4M3 kernels, and tools/calibrate_fp8.py -> tools/test.py end to end."""
import gc
import json
import os
import random
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import fp8_dpt_ref as dref
import fp8_vit_ref as vref
from test_baseline_host import pretrain_model_cfg
from test_gpu_baseline import _build, _same

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden')
MAX_DEPTH = 80.0
BOTH = dict(branch_vit_precision='fp8_static', branch_dpt_precision='fp8_static')


def _fine(model, img, seed, **kw):
    random.seed(seed)
    return model(mode='infer', image_lr=None, image_hr=img, **kw)[0].clone()


def _coarse(model, lr):
    return model(mode='infer', image_lr=lr, image_hr=None)[0].clone()


@pytest.fixture(scope='module')
def vits(cuda):
    from oracle.make_golden import case_inputs
    case = json.load(open(os.path.join(GOLD, 'vits_baseline0.json')))
    cfg, sd, img = case_inputs(case)
    shape = tuple(case['image_raw_shape'])
    imgs = torch.cat([img] + [torch.rand(1, 3, *shape, generator=torch.Generator().manual_seed(s))
                              for s in (101, 202)]).to(cuda)
    cal = torch.rand(2, 3, *shape, generator=torch.Generator().manual_seed(7)).to(cuda)
    split = dict(image_raw_shape=shape, patch_split_num=tuple(case['patch_split_num']))
    v = dict(case=case, pf_cfg=cfg, enc='vits', sd=sd, imgs=imgs, cal=cal, split=split)

    def make(target, **kw):
        return _build(target, v, cuda, **(dict(split, **kw) if target == 'fine' else kw))[1]
    v['make'] = make
    v['lr'] = F.interpolate(imgs, (392, 518), mode='bilinear', align_corners=True)
    v['cal_lr'] = F.interpolate(cal, (392, 518), mode='bilinear', align_corners=True)
    # calibrated vit + dpt models of both targets (fine: m2 at process_num 4, coarse: the two calibration images at once)
    v['coarse8'] = make('coarse', **BOTH)
    v['coarse8'].calibrate_fp8(v['cal_lr'], None)
    v['fine8'] = make('fine', **BOTH)
    random.seed(1)
    v['fine8'].calibrate_fp8(None, cal, cai_mode='m2', process_num=4)
    yield v
    # the later test modules share this process and the GPU: hand back the engines' panels, arenas and graphs
    for k in ('coarse8', 'fine8'):
        v[k].invalidate()
    v.clear()
    gc.collect()
    torch.cuda.empty_cache()


def test_forward_without_table_refuses(cuda, vits):
    v = vits
    for kw in (dict(branch_vit_precision='fp8_static'), dict(branch_dpt_precision='fp8_static'), BOTH):
        with pytest.raises(RuntimeError, match='calibrate_fp8'):
            _coarse(v['make']('coarse', **kw), v['lr'][:1])
        with pytest.raises(RuntimeError, match='calibrate_fp8'):
            _fine(v['make']('fine', **kw), v['imgs'][:1], 0, cai_mode='m1', process_num=2)


@pytest.mark.parametrize('target', ['coarse', 'fine'])
def test_calibration(cuda, vits, target):
    """every name of the branch, deterministic, merged by max, reset; a changed table re-points the stage (graphs
    dropped) and equals a freshly built model with it"""
    from patchfusion_b200.params import dpt_fp8_layers, vit_fp8_layers
    v = vits
    cfg = {'coarse_branch': v['pf_cfg']['coarse_branch'], 'fine_branch': v['pf_cfg']['fine_branch']}
    vn, dn = vit_fp8_layers(cfg, (target,)), dpt_fp8_layers(cfg, (target,))
    m = v['make'](target, **BOTH)
    if target == 'coarse':
        def cal(i, reset=False):
            return m.calibrate_fp8(v['lr'][i], None, reset=reset)

        def run(model):
            return _coarse(model, v['lr'][:2])
    else:
        def cal(i, reset=False):
            return m.calibrate_fp8(None, v['imgs'][i], cai_mode='m1', process_num=2, reset=reset)

        def run(model):
            return _fine(model, v['imgs'][:1], 4, cai_mode='m2', process_num=4)
    a = cal(slice(0, 1))
    assert tuple(a) == vn and all(x > 0 for x in a.values())
    assert tuple(m.branch_dpt_fp8_amax) == dn and all(x > 0 for x in m.branch_dpt_fp8_amax.values())
    b = cal(slice(0, 1), reset=True)
    assert a == b
    d1 = dict(m.branch_dpt_fp8_amax)
    cal(slice(1, 2))
    merged = (dict(m.branch_vit_fp8_amax), dict(m.branch_dpt_fp8_amax))
    assert all(merged[0][k] >= a[k] for k in vn) and all(merged[1][k] >= d1[k] for k in dn)
    two = cal(slice(0, 2), reset=True)
    assert (two, dict(m.branch_dpt_fp8_amax)) == merged
    y0 = run(m)
    _same('%s graph replay' % target, run(m), y0)
    assert m._graphs
    other = v[target + '8']
    m.branch_vit_fp8_amax = dict(other.branch_vit_fp8_amax)
    m.branch_dpt_fp8_amax = dict(other.branch_dpt_fp8_amax)
    m.engine(m._engine.P)
    assert m._graphs == {}
    y1 = run(m)
    fresh = v['make'](target, **BOTH, branch_vit_fp8_amax=dict(other.branch_vit_fp8_amax),
                      branch_dpt_fp8_amax=dict(other.branch_dpt_fp8_amax))
    _same('%s changed table vs fresh model' % target, y1, run(fresh))
    assert not torch.equal(y0, y1)


def test_tables_match_patchfusion(cuda, vits):
    """the same branch weights calibrated on the same images: the coarse baseline on image_lr and the fine baseline in
    m1 / m2 give exactly the coarse.* / fine.* entries of PatchFusion.calibrate_fp8's tables"""
    from patchfusion_b200.model import PatchFusion
    v = vits
    pf = PatchFusion(dict(v['pf_cfg'], vit_precision='fp8_static', dpt_precision='fp8_static'))
    pf.load_state_dict(v['sd'], strict=True)
    pf = pf.to(cuda).eval()
    imgs = v['cal']
    lr = pf.make_lr(imgs)
    coarse = v['make']('coarse', **BOTH)
    coarse.calibrate_fp8(lr, None)
    fine = v['make']('fine', **BOTH)
    for mode in ('m1', 'm2'):
        pf.calibrate_fp8(lr, imgs, cai_mode=mode, process_num=2, reset=True)
        fine.calibrate_fp8(None, imgs, cai_mode=mode, process_num=2, reset=True)
        for b, m in (('coarse', coarse), ('fine', fine)):
            for pk, bk in (('vit_fp8_amax', 'branch_vit_fp8_amax'), ('dpt_fp8_amax', 'branch_dpt_fp8_amax')):
                want = {k: x for k, x in pf.config[pk].items() if k.startswith(b + '.')}
                assert getattr(m, bk) == want, (mode, b, pk)
        print('%s: %d ViT and %d DPT entries of each branch equal PatchFusion\'s' %
              (mode, len(coarse.branch_vit_fp8_amax), len(coarse.branch_dpt_fp8_amax)))


def _emulated(orc, table_v, table_d, *a, **kw):
    with torch.no_grad(), vref.fp8_static_vit(table_v), dref.fp8_static_dpt(table_d):
        return orc.infer(*a, **kw)


def _vs(tag, got, want, bf):
    want = want.to(got.device).view(got.shape)
    err, rng = (got - want).abs().max().item(), (want.max() - want.min()).item()
    d16 = (got - bf).abs()
    print('%s: FP8 vs FP8 emulation max-abs %.3e (/80 %.3e, /range %.3e); vs bf16 max %.3e mean %.3e'
          % (tag, err, err / MAX_DEPTH, err / rng, d16.max().item(), d16.mean().item()))
    assert torch.isfinite(got).all(), tag
    assert err / MAX_DEPTH < 1e-3, tag


def test_vs_fp8_emulation(cuda, vits):
    from oracle.baseline_oracle import BaselineOracle
    v = vits
    sdc = {k: x.to(cuda) for k, x in v['sd'].items()}
    m = v['coarse8']
    cfg = pretrain_model_cfg('vits', 'coarse')
    orc = BaselineOracle(sdc, cfg, 'coarse')
    bf = v['make']('coarse')
    for lr in (v['lr'][:1], F.interpolate(v['imgs'][:1], (266, 350), mode='bilinear', align_corners=True)):
        tag = 'coarse B=1 %dx%d (392x518 table)' % lr.shape[-2:]
        _vs(tag, _coarse(m, lr), _emulated(orc, m.branch_vit_fp8_amax, m.branch_dpt_fp8_amax, lr, None),
            _coarse(bf, lr))
    m = v['fine8']
    orc = BaselineOracle(sdc, pretrain_model_cfg('vits', 'fine', **v['split']), 'fine')
    bf = v['make']('fine')
    img, pn = v['imgs'][:1], v['case']['process_num']
    for mode in ('m1', 'm2', 'r4'):
        got = _fine(m, img, 0, cai_mode=mode, process_num=pn)
        random.seed(0)
        want = _emulated(orc, m.branch_vit_fp8_amax, m.branch_dpt_fp8_amax, None, img, cai_mode=mode, process_num=pn)
        _vs('fine %s' % mode, got, want, _fine(bf, img, 0, cai_mode=mode, process_num=pn))


def test_invariances(cuda, vits):
    v = vits
    m, imgs = v['fine8'], v['imgs']
    _same('fine m2 process_num 9 vs 4', _fine(m, imgs[:1], 3, cai_mode='m2', process_num=9),
          _fine(m, imgs[:1], 3, cai_mode='m2', process_num=4))
    for mode in ('m2', 'r4'):
        random.seed(5)
        want = torch.cat([m(mode='infer', image_lr=None, image_hr=imgs[b:b + 1], cai_mode=mode, process_num=2)[0].clone()
                          for b in range(3)])
        _same('fine %s B=3 vs 3 x B=1' % mode, _fine(m, imgs, 5, cai_mode=mode, process_num=2), want)
        _same('fine %s emulated world 8' % mode, _fine(m, imgs, 5, cai_mode=mode, process_num=2, shard=('emulate', 8)),
              want)
    shapes = [((1080, 1920), (2, 2)), ((720, 1280), (2, 4)), ((540, 960), (1, 1))]
    mi = [torch.rand(1, 3, *hw, generator=torch.Generator().manual_seed(10 + i)).to(cuda)
          for i, (hw, _) in enumerate(shapes)]
    cfgs = [{'image_raw_shape': list(hw), 'patch_split_num': list(p)} for hw, p in shapes]
    modes = ['m2', 'r4', 'm1']
    random.seed(7)
    want = [m(mode='infer', image_lr=None, image_hr=mi[b], tile_cfg=cfgs[b], cai_mode=modes[b],
              process_num=9)[0].clone() for b in range(3)]
    random.seed(7)
    got, _ = m(mode='infer', image_lr=None, image_hr=mi, tile_cfg=cfgs, cai_mode=modes, process_num=9)
    for b in range(3):
        _same('fine mixed geometry image %d' % b, got[b], want[b])
    c = v['coarse8']
    lr8 = F.interpolate(torch.cat([imgs, v['cal'], imgs]), (392, 518), mode='bilinear', align_corners=True)
    y = _coarse(c, lr8)
    _same('coarse B=8 vs 8 x B=1', y, torch.cat([_coarse(c, lr8[i:i + 1]) for i in range(8)]))


def _profiled_names(fn):
    from patchfusion_b200 import lib
    prof = lib.Profiler()
    lib.PROFILER = prof
    try:
        prof.start()
        fn()
        recs = prof.stop()
    finally:
        lib.PROFILER = None
    return [r[0] for r in recs]


def test_default_path_unaffected(cuda, vits):
    """no new key, the new keys at 'bf16', and PatchFusion's keys alone (any value): the plain model's bits and its
    kernel sequence; the FP8 models' kernels on top of that"""
    v = vits
    ignored = dict(vit_precision='fp8_static', dpt_precision='fp8_static', vit_fp8_amax={'x': 1.0}, fusion_precision='fp8')
    for target in ('coarse', 'fine'):
        if target == 'coarse':
            def run(model):
                return _coarse(model, v['lr'][:2])
        else:
            def run(model):
                return _fine(model, v['imgs'][:1], 9, cai_mode='m2', process_num=4)
        plain = v['make'](target)
        want, names = run(plain), _profiled_names(lambda: run(plain))
        assert 'pf_gemm_pp_e4m3_kernel' not in names and 'quant_static_kernel' not in names
        for kw in (dict(branch_vit_precision='bf16', branch_dpt_precision='bf16'), ignored):
            m = v['make'](target, **kw)
            _same('%s %s vs plain' % (target, sorted(kw)), run(m), want)
            _same('%s %s replay vs plain' % (target, sorted(kw)), run(m), want)
            assert _profiled_names(lambda: run(m)) == names, (target, kw)
        f8 = _profiled_names(lambda: run(v[target + '8']))
        calls = f8.count('assemble_tokens_kernel')
        assert calls == names.count('assemble_tokens_kernel') > 0
        depth = 12
        assert f8.count('pf_gemm_pp_e4m3_kernel') == 3 * depth * calls
        assert f8.count('pf_conv3_halo_e4m3_res_kernel') == 11 * calls and f8.count('quant_static_kernel') == 5 * calls
        assert len(f8) == len(names) + 5 * calls
        print('%s: %d launches bf16, %d FP8 (%d branch calls)' % (target, len(names), len(f8), calls))


@pytest.mark.parametrize('target,B', [('fine', 3), ('coarse', 2)])
def test_fp8_branch_workspace(cuda, vits, target, B):
    """the FP8 branch stage of a baseline's engine on NaN- and 3.0-poisoned workspaces with guard bytes
    (tests/test_gpu_workspace.py's check, e4m3 pad bytes included)"""
    from test_gpu_workspace import _branch_run, _check_stage, _rand
    eng = vits[target + '8'].engine((392, 518))
    assert eng.vit_amax is not None and eng.dpt_amax is not None
    run, need = _branch_run(eng, target, _rand((B, 3) + eng.P, 40 + B))
    _check_stage('baseline FP8 %s branch B=%d' % (target, B), run, need, eng, target)
    eng.arenas.clear()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------- vitl coverage
def _vitl(cuda, target, **kw):
    from patchfusion_b200.baseline import BaselinePretrain
    cfg = pretrain_model_cfg('vitl', target, **kw)
    cfg.pop('type')
    return BaselinePretrain(**cfg).init_synthetic_weights(0).to(cuda).eval()


def _close(tag, got, bf):
    d = (got - bf).abs()
    print('%s: FP8 vs bf16 max-abs %.3e (/80 %.3e) mean %.3e' % (tag, d.max().item(), d.max().item() / MAX_DEPTH,
                                                                   d.mean().item()))
    assert torch.isfinite(got).all(), tag
    assert d.max().item() / MAX_DEPTH < 2e-3, tag


def test_vitl_coarse_batch32_and_other_size(cuda):
    """the vitl coarse target at B = 32 (392x518) and at 546x728 (one table calibrated at 392x518): every ViT linear
    on the E4M3 ping-pong GEMM and every covered DPT conv on the E4M3 convs, close to bf16"""
    g = torch.Generator().manual_seed(11)
    m8 = _vitl(cuda, 'coarse', **BOTH)
    bf = _vitl(cuda, 'coarse')
    m8.calibrate_fp8(torch.rand(4, 3, 392, 518, generator=g).to(cuda), None)
    for B, h, w in ((32, 392, 518), (2, 546, 728)):
        lr = torch.rand(B, 3, h, w, generator=g).to(cuda)
        names = _profiled_names(lambda: _coarse(m8, lr))
        assert names.count('assemble_tokens_kernel') == 1
        assert names.count('pf_gemm_pp_e4m3_kernel') == 3 * 24 and names.count('pf_conv3_halo_e4m3_res_kernel') == 11
        got = _coarse(m8, lr)
        _same('vitl coarse B=%d %dx%d replay' % (B, h, w), _coarse(m8, lr), got)
        _close('vitl coarse B=%d %dx%d' % (B, h, w), got, _coarse(bf, lr))
        del lr, got
    m8.invalidate()
    bf.invalidate()
    torch.cuda.empty_cache()


def test_vitl_fine_process_num_16(cuda):
    """the vitl fine target at 4K m2 with micro-batches of 16 tiles on the E4M3 kernels: the same bits as process_num
    4, close to bf16"""
    g = torch.Generator().manual_seed(12)
    m8 = _vitl(cuda, 'fine', **BOTH)
    random.seed(0)
    m8.calibrate_fp8(None, torch.rand(1, 3, 2160, 3840, generator=g).to(cuda), cai_mode='m1', process_num=16)
    img = torch.rand(1, 3, 2160, 3840, generator=g).to(cuda)
    names = _profiled_names(lambda: _fine(m8, img, 0, cai_mode='m2', process_num=16))
    calls = names.count('assemble_tokens_kernel')
    assert calls == 4 and names.count('pf_gemm_pp_e4m3_kernel') == 3 * 24 * calls     # 49 tiles: 16 + 16 + 16 + 1
    got = _fine(m8, img, 0, cai_mode='m2', process_num=16)
    _same('vitl fine m2 process_num 16 vs 4', got, _fine(m8, img, 0, cai_mode='m2', process_num=4))
    m8.invalidate()
    bf = _vitl(cuda, 'fine')
    _close('vitl fine 4K m2 process_num 16', got, _fine(bf, img, 0, cai_mode='m2', process_num=16))
    bf.invalidate()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------- command line
def _write_case(root, target, n_frames=2):
    """a U4K tree, a shipped-schema depthanything_vits_<target>_pretrain_u4k.py reading it and a synthetic branch
    checkpoint ({'model_state_dict': unprefixed branch weights}, what the baseline trainer saves)"""
    from patchfusion_b200 import eval_tree as et
    from patchfusion_b200.baseline import BaselinePretrain
    split = et.write_u4k_tree(os.path.join(root, 'u4k'), n_frames, seed=3)
    model = pretrain_model_cfg('vits', target)
    kw = dict(model)
    kw.pop('type')
    ckpt = os.path.join(root, 'vits_%s_synthetic.pth' % target)
    torch.save({'model_state_dict': BaselinePretrain(**kw).init_synthetic_weights(0).get_save_dict()}, ckpt)
    conf = os.path.join(root, 'depthanything_vits_%s_pretrain_u4k.py' % target)
    with open(conf, 'w') as f:
        f.write('model = %r\nval_dataloader = dict(batch_size=1, num_workers=2, dataset=dict(type="UnrealStereo4kDataset", '
                'mode="infer", data_root=%r, split=%r, min_depth=1e-3, max_depth=80, '
                'transform_cfg=dict(network_process_size=[392, 518]), resize_mode="depth-anything"))\n'
                % (model, os.path.join(root, 'u4k'), split))
    return conf, ckpt


@pytest.mark.parametrize('target', ['coarse', 'fine'])
def test_calibrate_tool_then_test_tool(cuda, tmp_path, target):
    from patchfusion_b200 import datasets as D
    from patchfusion_b200.params import dpt_fp8_layers, vit_fp8_layers
    conf, ckpt = _write_case(str(tmp_path), target)
    out = tmp_path / 'calibrated'
    cmd = [sys.executable, os.path.join(ROOT, 'tools', 'calibrate_fp8.py'), conf, '--ckp-path', ckpt, '--num-images',
           '2', '--out', str(out), '--cai-mode', 'm1', '--image-raw-shape', '2160', '3840', '--patch-split-num', '2', '2']
    if target == 'fine':
        cmd += ['--cfg-options', 'model.branch_dpt_precision=fp8_static']
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(tmp_path), timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    lines = r.stdout.splitlines()
    printed = json.loads('\n'.join(lines[max(i for i, l in enumerate(lines) if l == '{'):]))
    cfg = pretrain_model_cfg('vits', target)
    assert printed['images'] == 2 and tuple(printed['branch_vit_fp8_amax']) == vit_fp8_layers(cfg, (target,))
    assert ('branch_dpt_fp8_amax' in printed) == (target == 'fine')
    if target == 'fine':
        assert tuple(printed['branch_dpt_fp8_amax']) == dpt_fp8_layers(cfg, (target,))
    name = 'depthanything_vits_%s_pretrain_u4k' % target
    assert sorted(os.listdir(out)) == [name + '.pth', name + '.py']
    wd = tmp_path / 'eval'
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'test.py'), str(out / (name + '.py')), '--ckp-path',
                        str(out / (name + '.pth')), '--cai-mode', 'm1', '--work-dir', str(wd), '--image-raw-shape',
                        '2160', '3840', '--patch-split-num', '2', '2'],
                       capture_output=True, text=True, cwd=str(tmp_path), timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    metrics = json.load(open(wd / 'metrics.json'))
    print('%s: %s' % (target, metrics))
    assert list(metrics) == list(D.METRIC_KEYS)
