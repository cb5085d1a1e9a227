"""State-dict layout, parameter tree and synthetic weights for the PatchFusion hot path.

The drop-in contract (SURVEY.md §8b, Appendix B) is that a checkpoint written by the reference
(`estimator/models/patchfusion.py:57-173`, HF `from_pretrained`) loads into this package unchanged.  The layout
is therefore restated here as data: `state_layout(config)` yields every key, shape and dtype in the order the
reference's `state_dict()` emits them; `ParamTree` materialises it as nested `nn.Module` containers (so
`state_dict()/load_state_dict()/to()` behave like the reference module), and `synthetic_state_dict` fills it with
seeded, variance-preserving random weights (no network, no checkpoints in this environment).

tests/test_layout.py checks the layout against tests/golden/state_dict_layout_{vits,vitl}.json, which were dumped
from the reference itself by oracle/make_golden.py.
"""
from collections import OrderedDict
import math
import numbers

import torch
import torch.nn as nn

# DINOv2 encoders as instantiated by hubconf (`hubconf.py:24-67`, `vision_transformer.py:339-378`) and the DPT
# widths chosen in `zoedepth/models/base_models/depth_anything.py:345-353`.
ENCODERS = {
    'vits': dict(dim=384, depth=12, heads=6, out_channels=[48, 96, 192, 384], features=64),
    'vitb': dict(dim=768, depth=12, heads=12, out_channels=[96, 192, 384, 768], features=128),
    'vitl': dict(dim=1024, depth=24, heads=16, out_channels=[256, 512, 1024, 1024], features=256),
}
PATCH = 14
POS_GRID = 37          # 518 / 14: pos_embed holds 1 + 37*37 entries (`hubconf.py:38`, img_size=518)
N_MIDAS_OUT = 32       # `patchfusion.py:119`, `zoedepth_v1.py:79`
WINDOW = 12            # `guided_fusion_model.py:133`
G2L_DEPTH = [2, 2, 3, 3, 4, 4]          # high -> low resolution (`guided_fusion_model.py:109`)
G2L_HEADS = [8, 8, 16, 16, 32, 32]      # (`guided_fusion_model.py:110`)


def _get(cfg, key, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


FUSION_PRECISIONS = ('bf16', 'fp8', 'fp8_static')
# The Guided-Fusion U-Net's 34 3x3 convs that run E4M3 under 'fp8' / 'fp8_static', by their names in
# Engine._pack_fusion: the two convs X.0 -> ReLU -> X.1 -> ReLU of each of the 17 DoubleConvs
FP8_LAYERS = tuple(['inc.0', 'inc.1'] + ['down%d.%d' % (i, j) for i in range(5) for j in (0, 1)] +
                   ['up%d.%d' % (i, j) for i in range(1, 6) for j in (0, 1)] +
                   ['cv%d.%d' % (i, j) for i in range(6) for j in (0, 1)])


def fusion_precision(config):
    """Top-level `fusion_precision`: what the Guided-Fusion U-Net's 3x3 convs (inc, down_conv_list, up_conv_list, convs)
    compute in.  'bf16' (default) is the path every other layer takes; 'fp8' runs them on E4M3 operands with one
    scale per tile and input and one per output channel (include/pf_b200.h, DESIGN.md section 7); 'fp8_static' does
    the same with one calibrated scale per conv input (`fusion_fp8_amax`, PatchFusion.calibrate_fp8)."""
    p = _get(config, 'fusion_precision', 'bf16')
    if p not in FUSION_PRECISIONS:
        raise ValueError("fusion_precision should be one of 'bf16', 'fp8', 'fp8_static'")
    return p


def fusion_fp8_amax(config):
    """Top-level `fusion_fp8_amax`: the calibrated amax of each FP8 conv's input, {layer name of FP8_LAYERS: float >= 0}
    with exactly those 34 names, or None when the config has no table.  Anything else raises ValueError."""
    t = _get(config, 'fusion_fp8_amax', None)
    if t is None:
        return None
    if not isinstance(t, dict):
        raise ValueError('fusion_fp8_amax should be a dict of the 34 FP8 layer names to their input amax')
    missing = [k for k in FP8_LAYERS if k not in t]
    unknown = sorted(str(k) for k in t if k not in FP8_LAYERS)
    if missing or unknown:
        raise ValueError('fusion_fp8_amax: missing layers %s, unknown layers %s' % (missing, unknown))
    out = {}
    for k in FP8_LAYERS:
        v = t[k]
        if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(v) or v < 0:
            raise ValueError('fusion_fp8_amax[%r] = %r: a finite float >= 0 is required' % (k, v))
        out[k] = float(v)
    return out


VIT_PRECISIONS = ('bf16', 'fp8_static')
# The ViT linears that run E4M3 under vit_precision 'fp8_static', per block of each branch's encoder
VIT_FP8_LINEARS = ('qkv', 'fc1', 'fc2')


def vit_precision(config):
    """Top-level `vit_precision`: what the qkv, fc1 and fc2 linears of both branches' DINOv2 encoders compute in.
    'bf16' (default), or 'fp8_static': E4M3 operands with one calibrated scale per linear input (`vit_fp8_amax`,
    PatchFusion.calibrate_fp8) and one per output channel.  Independent of fusion_precision."""
    p = _get(config, 'vit_precision', 'bf16')
    if p not in VIT_PRECISIONS:
        raise ValueError("vit_precision should be one of 'bf16', 'fp8_static'")
    return p


def vit_fp8_layers(config):
    """The names of vit_fp8_amax: '{coarse|fine}.{i}.{qkv|fc1|fc2}' for every block i of each branch's encoder"""
    names = []
    for b in ('coarse', 'fine'):
        depth = branch_hparams(_get(config, b + '_branch'))['depth']
        names += ['%s.%d.%s' % (b, i, k) for i in range(depth) for k in VIT_FP8_LINEARS]
    return tuple(names)


def vit_fp8_amax(config):
    """Top-level `vit_fp8_amax`: the calibrated amax of each E4M3 ViT linear's input, {name of vit_fp8_layers: float
    >= 0} with exactly those 6 * depth names, or None when the config has no table.  Anything else raises ValueError."""
    t = _get(config, 'vit_fp8_amax', None)
    if t is None:
        return None
    names = vit_fp8_layers(config)
    if not isinstance(t, dict):
        raise ValueError('vit_fp8_amax should be a dict of the %d ViT linear names to their input amax' % len(names))
    known = set(names)
    missing = [k for k in names if k not in t]
    unknown = sorted(str(k) for k in t if k not in known)
    if missing or unknown:
        raise ValueError('vit_fp8_amax: missing layers %s, unknown layers %s' % (missing, unknown))
    out = {}
    for k in names:
        v = t[k]
        if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(v) or v < 0:
            raise ValueError('vit_fp8_amax[%r] = %r: a finite float >= 0 is required' % (k, v))
        out[k] = float(v)
    return out


DPT_PRECISIONS = ('bf16', 'fp8_static')
# The DPT decoder's 3x3 convs that run E4M3 under dpt_precision 'fp8_static', by their names in each branch's
# depth_head.scratch: the four reassemble convs, the ResidualConvUnits that run (refinenet4 uses only resConfUnit2)
# and output_conv1
DPT_FP8_CONVS = tuple(['layer%d_rn' % i for i in range(1, 5)] +
                      ['refinenet%d.resConfUnit%d.conv%d' % (i, u, k) for i in (1, 2, 3) for u in (1, 2) for k in (1, 2)] +
                      ['refinenet4.resConfUnit2.conv%d' % k for k in (1, 2)] + ['output_conv1'])


def dpt_precision(config):
    """Top-level `dpt_precision`: what the DPT decoders' covered 3x3 convs (DPT_FP8_CONVS) of both branches compute in.
    'bf16' (default), or 'fp8_static': E4M3 operands with one calibrated scale per conv input (`dpt_fp8_amax`,
    PatchFusion.calibrate_fp8) and one per output channel.  Independent of fusion_precision and vit_precision."""
    p = _get(config, 'dpt_precision', 'bf16')
    if p not in DPT_PRECISIONS:
        raise ValueError("dpt_precision should be one of 'bf16', 'fp8_static'")
    return p


def dpt_fp8_layers(config=None):
    """The names of dpt_fp8_amax: '{coarse|fine}.<conv>' for every conv of DPT_FP8_CONVS, 38 in all"""
    return tuple('%s.%s' % (b, n) for b in ('coarse', 'fine') for n in DPT_FP8_CONVS)


def dpt_fp8_amax(config):
    """Top-level `dpt_fp8_amax`: the calibrated amax of each E4M3 DPT conv's input, {name of dpt_fp8_layers: float >= 0}
    with exactly those 38 names, or None when the config has no table.  Anything else raises ValueError."""
    t = _get(config, 'dpt_fp8_amax', None)
    if t is None:
        return None
    names = dpt_fp8_layers(config)
    if not isinstance(t, dict):
        raise ValueError('dpt_fp8_amax should be a dict of the %d DPT conv names to their input amax' % len(names))
    known = set(names)
    missing = [k for k in names if k not in t]
    unknown = sorted(str(k) for k in t if k not in known)
    if missing or unknown:
        raise ValueError('dpt_fp8_amax: missing layers %s, unknown layers %s' % (missing, unknown))
    out = {}
    for k in names:
        v = t[k]
        if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(v) or v < 0:
            raise ValueError('dpt_fp8_amax[%r] = %r: a finite float >= 0 is required' % (k, v))
        out[k] = float(v)
    return out


def branch_hparams(branch_cfg):
    enc = _get(branch_cfg, 'midas_model_type')
    if enc not in ENCODERS:
        raise NotImplementedError(
            "backbone %r is not vendored in the reference tree (only Depth-Anything vits/vitb/vitl are; the "
            "ZoeDepth-N BEiT-L backbone comes from an un-vendored torch.hub repo, SURVEY.md §8c)" % (enc,))
    hp = dict(ENCODERS[enc])
    hp['encoder'] = enc
    hp['n_bins'] = _get(branch_cfg, 'n_bins', 64)
    hp['bin_embedding_dim'] = _get(branch_cfg, 'bin_embedding_dim', 128)
    hp['n_attractors'] = list(_get(branch_cfg, 'n_attractors', [16, 8, 4, 1]))
    hp['bin_centers_type'] = _get(branch_cfg, 'bin_centers_type', 'softplus')
    if hp['bin_centers_type'] not in ('normed', 'softplus', 'hybrid1', 'hybrid2'):
        raise ValueError("bin_centers_type should be one of 'normed', 'softplus', 'hybrid1', 'hybrid2'")
    # config fields that change the reference's arithmetic (zoedepth_v1.py:41-42 constructor defaults): honour the
    # ones the kernels implement, refuse the rest instead of silently computing something else
    hp['attractor_kind'] = _get(branch_cfg, 'attractor_kind', 'sum')
    hp['attractor_type'] = _get(branch_cfg, 'attractor_type', 'exp')
    if hp['attractor_kind'] not in ('mean', 'sum') or hp['attractor_type'] not in ('inv', 'exp'):
        raise ValueError('attractor_kind must be mean|sum and attractor_type inv|exp')
    if _get(branch_cfg, 'inverse_midas', False):
        raise NotImplementedError('inverse_midas=True (zoedepth_v1.py:198-202) is not built: no PatchFusion config sets it')
    if _get(branch_cfg, 'do_resize', False):
        raise NotImplementedError('do_resize=True (depth_anything.py:177-190 resizer) is not built: PatchFusion feeds '
                                  'tiles already at patch_process_shape')
    return hp


def normed_seed(bin_centers_type):
    """the head's seed regressor is SeedBinRegressor (`zoedepth_v1.py:90-105`): ReLU widths normalised and cumulated into centres"""
    return bin_centers_type in ('normed', 'hybrid1')


def normed_attractors(bin_centers_type):
    """the head's attractors are AttractorLayer (`zoedepth_v1.py:90-105`): normalised centres, sorted and clipped metric output"""
    return bin_centers_type in ('normed', 'hybrid2')


def _f(shape):
    return (tuple(shape), torch.float32, 'param')


def _conv(L, name, cout, cin, k, bias=True):
    L[name + '.weight'] = _f((cout, cin, k, k))
    if bias:
        L[name + '.bias'] = _f((cout,))


def _linear(L, name, cout, cin):
    L[name + '.weight'] = _f((cout, cin))
    L[name + '.bias'] = _f((cout,))


def _norm(L, name, c):
    L[name + '.weight'] = _f((c,))
    L[name + '.bias'] = _f((c,))


def _bn(L, name, c):
    L[name + '.weight'] = _f((c,))
    L[name + '.bias'] = _f((c,))
    L[name + '.running_mean'] = ((c,), torch.float32, 'buffer')
    L[name + '.running_var'] = ((c,), torch.float32, 'buffer')
    L[name + '.num_batches_tracked'] = ((), torch.int64, 'buffer')


def _metric_head(L, pre, C, hp):
    """seed regressor / projectors / attractors / conditional log-binomial (`zoedepth_v1.py:103-123`,
    `patchfusion.py:149-170`)."""
    E = hp['bin_embedding_dim']
    _conv(L, pre + 'seed_bin_regressor._net.0', 256, C, 1)
    _conv(L, pre + 'seed_bin_regressor._net.2', hp['n_bins'], 256, 1)
    _conv(L, pre + 'seed_projector._net.0', 128, C, 1)
    _conv(L, pre + 'seed_projector._net.2', E, 128, 1)
    for i in range(4):
        _conv(L, pre + 'projectors.%d._net.0' % i, 128, C, 1)
        _conv(L, pre + 'projectors.%d._net.2' % i, E, 128, 1)
    # AttractorLayer emits 2 channels per attractor (`attractor.py:80-85`), AttractorLayerUnnormed one (:157-162)
    per_attractor = 2 if normed_attractors(hp['bin_centers_type']) else 1
    for i in range(4):
        _conv(L, pre + 'attractors.%d._net.0' % i, 128, E, 1)
        _conv(L, pre + 'attractors.%d._net.2' % i, per_attractor * hp['n_attractors'][i], 128, 1)
    L[pre + 'conditional_log_binomial.log_binomial_transform.k_idx'] = ((1, hp['n_bins'], 1, 1), torch.int64, 'buffer')
    L[pre + 'conditional_log_binomial.log_binomial_transform.K_minus_1'] = ((1, 1, 1, 1), torch.float32, 'buffer')
    cin = N_MIDAS_OUT + 1 + E
    _conv(L, pre + 'conditional_log_binomial.mlp.0', cin // 2, cin, 1)
    _conv(L, pre + 'conditional_log_binomial.mlp.2', 4, cin // 2, 1)


def _branch(L, pre, hp):
    D, C, oc = hp['dim'], hp['features'], hp['out_channels']
    vit = pre + 'core.core.pretrained.'
    L[vit + 'cls_token'] = _f((1, 1, D))
    L[vit + 'pos_embed'] = _f((1, 1 + POS_GRID * POS_GRID, D))
    L[vit + 'mask_token'] = _f((1, D))
    _conv(L, vit + 'patch_embed.proj', D, 3, PATCH)
    for b in range(hp['depth']):
        p = vit + 'blocks.%d.' % b
        _norm(L, p + 'norm1', D)
        _linear(L, p + 'attn.qkv', 3 * D, D)
        _linear(L, p + 'attn.proj', D, D)
        L[p + 'ls1.gamma'] = _f((D,))
        _norm(L, p + 'norm2', D)
        _linear(L, p + 'mlp.fc1', 4 * D, D)
        _linear(L, p + 'mlp.fc2', D, 4 * D)
        L[p + 'ls2.gamma'] = _f((D,))
    _norm(L, vit + 'norm', D)
    dh = pre + 'core.core.depth_head.'
    for i in range(4):
        _conv(L, dh + 'projects.%d' % i, oc[i], D, 1)
    _conv(L, dh + 'resize_layers.0', oc[0], oc[0], 4)   # ConvTranspose2d k4 s4: weight (in, out, 4, 4)
    _conv(L, dh + 'resize_layers.1', oc[1], oc[1], 2)   # ConvTranspose2d k2 s2
    _conv(L, dh + 'resize_layers.3', oc[3], oc[3], 3)   # Conv2d k3 s2 p1
    for i in range(4):
        _conv(L, dh + 'scratch.layer%d_rn' % (i + 1), C, oc[i], 3, bias=False)
    for i in range(1, 5):
        r = dh + 'scratch.refinenet%d.' % i
        _conv(L, r + 'out_conv', C, C, 1)
        for u in (1, 2):
            _conv(L, r + 'resConfUnit%d.conv1' % u, C, C, 3)
            _conv(L, r + 'resConfUnit%d.conv2' % u, C, C, 3)
    _conv(L, dh + 'scratch.output_conv1', C // 2, C, 3)
    _conv(L, dh + 'scratch.output_conv2.0', N_MIDAS_OUT, C // 2, 3)
    _conv(L, dh + 'scratch.output_conv2.2', 1, N_MIDAS_OUT, 1)
    _conv(L, pre + 'conv2', C, C, 1)
    _metric_head(L, pre, C, hp)


def guided_fusion_hparams(gf_cfg, patch_process_shape):
    in_ch = list(_get(gf_cfg, 'in_channels', [32, 256, 256, 256, 256, 256]))
    num_patches = list(_get(gf_cfg, 'num_patches',
                            [384 * 512, 192 * 256, 96 * 128, 48 * 64, 24 * 32, 12 * 16]))
    return dict(in_channels=in_ch, num_patches=num_patches, n_channels=_get(gf_cfg, 'n_channels', 5),
                depth=list(_get(gf_cfg, 'depth', G2L_DEPTH)), num_heads=list(_get(gf_cfg, 'num_heads', G2L_HEADS)))


def state_layout(config):
    """OrderedDict key -> (shape, dtype, 'param'|'buffer') in the reference's `state_dict()` order."""
    hp_c = branch_hparams(_get(config, 'coarse_branch'))
    hp_f = branch_hparams(_get(config, 'fine_branch'))
    gf = guided_fusion_hparams(_get(config, 'guided_fusion'), _get(config, 'patch_process_shape'))
    L = OrderedDict()
    _branch(L, 'coarse_branch.', hp_c)
    _branch(L, 'fine_branch.', hp_f)
    C = hp_f['features']
    for i in range(6):
        c = N_MIDAS_OUT if i == 5 else C
        _conv(L, 'fusion_conv_list.%d' % i, c, 2 * c, 3)
    ic = gf['in_channels']
    g = 'guided_fusion.'

    def double_conv_bn(pre, cin, cout):
        _conv(L, pre + 'double_conv.0', cout, cin, 3, bias=False)
        _bn(L, pre + 'double_conv.1', cout)
        _conv(L, pre + 'double_conv.3', cout, cout, 3, bias=False)
        _bn(L, pre + 'double_conv.4', cout)

    def double_conv(pre, cin, cmid, cout):
        _conv(L, pre + 'double_conv.0', cmid, cin, 3)
        _conv(L, pre + 'double_conv.2', cout, cmid, 3)

    double_conv_bn(g + 'inc.', gf['n_channels'], ic[0])
    for i in range(5):
        double_conv_bn(g + 'down_conv_list.%d.maxpool_conv.1.' % i, ic[i], ic[i + 1])
    inv = ic[::-1]
    for i in range(1, 6):
        cin = inv[i] + 2 * inv[i - 1]
        double_conv(g + 'up_conv_list.%d.conv.' % (i - 1), cin, cin, inv[i])
    depth_inv, heads_inv, np_inv = gf['depth'][::-1], gf['num_heads'][::-1], gf['num_patches'][::-1]
    for i in range(6):
        c, p = inv[i], g + 'g2l_list.%d.' % i
        L[p + 'absolute_pos_embed'] = _f((1, np_inv[i], c))
        for b in range(depth_inv[i]):
            q = p + 'g2l_layer.blocks.%d.' % b
            _norm(L, q + 'norm1', c)
            L[q + 'attn.relative_position_bias_table'] = _f(((2 * WINDOW - 1) ** 2, heads_inv[i]))
            L[q + 'attn.relative_position_index'] = ((WINDOW * WINDOW, WINDOW * WINDOW), torch.int64, 'buffer')
            _linear(L, q + 'attn.qkv', 3 * c, c)
            _linear(L, q + 'attn.proj', c, c)
            _norm(L, q + 'norm2', c)
            _linear(L, q + 'mlp.fc1', 4 * c, c)
            _linear(L, q + 'mlp.fc2', c, 4 * c)
        _norm(L, p + 'g2l_layer_norm', c)
        _conv(L, p + 'embed_proj', c, 1, 1)
    for i in range(6):
        double_conv(g + 'convs.%d.' % i, 2 * inv[i], inv[i], inv[i])
    _metric_head(L, '', C, hp_c)
    return L


def branch_layout(branch_cfg, prefix):
    """Layout of ONE branch (`BaselinePretrain` builds only the coarse or only the fine branch, BP:67-85): the keys of
    `state_layout` under `prefix`, in the same order."""
    L = OrderedDict()
    _branch(L, prefix, branch_hparams(branch_cfg))
    return L


def relative_position_index(ws=WINDOW):
    """Swin relative-position lookup (`swin_layers.py:108-118`): index (i, j) -> row of the (2ws-1)^2 bias table."""
    ys, xs = torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing='ij')
    co = torch.stack([ys.flatten(), xs.flatten()])               # 2, ws*ws
    rel = co[:, :, None] - co[:, None, :] + (ws - 1)              # 2, N, N  in [0, 2ws-2]
    return rel[0] * (2 * ws - 1) + rel[1]


class _Node(nn.Module):
    """Pure container; exists so dotted state-dict paths map onto sub-modules."""


class ParamTree(nn.Module):
    """Base class materialising `state_layout(config)` as parameters/buffers at the reference's dotted paths."""

    def _build_tree(self, layout):
        for key, (shape, dtype, kind) in layout.items():
            parts = key.split('.')
            node = self
            for p in parts[:-1]:
                if p not in node._modules:
                    node.add_module(p, _Node())
                node = node._modules[p]
            t = torch.zeros(shape, dtype=dtype)
            if kind == 'param':
                node.register_parameter(parts[-1], nn.Parameter(t, requires_grad=False))
            else:
                node.register_buffer(parts[-1], t)


# (pattern, gain) in priority order: gain 2 where a ReLU follows (variance preserving), < 1 on residual branches and
# after sums so the DPT / U-Net activations stay O(1) and the log-binomial head works in its smooth regime.
_GAINS = [
    ('resConfUnit1.conv2', 0.25), ('resConfUnit2.conv2', 0.25), ('resConfUnit', 2.0),
    ('refinenet', 0.5),                        # FFB out_conv after path + skip
    ('layer1_rn', 1.0), ('layer2_rn', 1.0), ('layer3_rn', 1.0), ('layer4_rn', 1.0),
    ('projects', 1.0), ('resize_layers', 1.0),
    ('output_conv1', 1.0), ('output_conv2.0', 2.0), ('output_conv2.2', 1.0),
    ('conditional_log_binomial.mlp.0', 1.0), ('conditional_log_binomial.mlp.2', 1.0),
    ('attractors', None), ('_net.0', 2.0), ('_net.2', 1.0),
    ('fusion_conv_list', 1.0), ('double_conv', 2.0), ('embed_proj', 1.0),
    ('patch_embed', 1.0), ('conv2.weight', 1.0),
    ('attn.qkv', 1.0), ('attn.proj', 1.0), ('mlp.fc1', 2.0), ('mlp.fc2', 1.0),
]


def _gain(key):
    for pat, g in _GAINS:
        if pat in key:
            if g is None:                      # attractor MLPs: '_net.0' relu, '_net.2' softplus head
                return 2.0 if '_net.0' in key else 1.0
            return g
    raise AssertionError('no init rule for ' + key)


def synthetic_state_dict(config, seed=0, dtype=torch.float32, prefix=''):
    """Seeded random weights with O(1) activations through the whole network.

    Linear/conv weights ~ N(0, gain/fan_in); the residual branches of the ViT/Swin blocks and the DPT RCUs are
    scaled down so the stream does not blow up; BN stats near identity; position tables small.  The values are a
    function of (key order, shapes, seed) only, so the GPU box regenerates exactly the weights the oracle and the
    golden fixtures were produced with.

    prefix: keep only the keys under it (e.g. 'fine_branch.'), drawn from the same stream as the full dict, so a
    single-branch model and a PatchFusion built from one seed hold identical branch weights.
    """
    g = torch.Generator().manual_seed(seed)
    layout = state_layout(config)
    sd = OrderedDict()

    def rn(shape, std):
        return torch.randn(shape, generator=g, dtype=torch.float32) * std

    for key, (shape, dt, kind) in layout.items():
        if prefix and sd and not key.startswith(prefix):
            break                                                # past the requested block: nothing left to keep
        leaf = key.split('.')[-1]
        if key.endswith('relative_position_index'):
            t = relative_position_index()
        elif leaf == 'k_idx':
            t = torch.arange(shape[1]).view(shape)
        elif leaf == 'K_minus_1':
            t = torch.full(shape, float(layout[key.replace('K_minus_1', 'k_idx')][0][1] - 1))
        elif leaf == 'num_batches_tracked':
            t = torch.zeros((), dtype=torch.int64)
        elif leaf == 'running_mean':
            t = rn(shape, 0.1)
        elif leaf == 'running_var':
            t = 1.0 + 0.2 * torch.rand(shape, generator=g)
        elif leaf == 'gamma':                                    # LayerScale
            t = 0.3 + 0.1 * torch.rand(shape, generator=g)
        elif leaf in ('cls_token', 'mask_token'):
            t = rn(shape, 0.5)
        elif leaf == 'pos_embed' or leaf == 'absolute_pos_embed':
            t = rn(shape, 0.3)
        elif leaf == 'relative_position_bias_table':
            t = rn(shape, 0.5)
        elif leaf == 'bias':
            t = rn(shape, 0.05)
        elif leaf == 'weight' and len(shape) == 1:               # LayerNorm / BatchNorm scale
            t = 1.0 + rn(shape, 0.1)
        elif leaf == 'weight':
            fan_in = 1
            for s_ in shape[1:]:
                fan_in *= s_
            if 'resize_layers.0' in key or 'resize_layers.1' in key:
                fan_in = shape[0]                                # ConvTranspose k==s: one tap per output pixel
            t = rn(shape, math.sqrt(_gain(key) / fan_in))
        else:
            raise AssertionError(key)
        if key.startswith(prefix):
            sd[key] = t.to(dt if dt != torch.float32 else dtype)
    return sd


def default_init_state_dict(config, seed=0):
    """Seeded weights drawn from the distributions the REFERENCE's own constructor uses (no checkpoints are reachable
    offline and the reference's exact RNG stream cannot be replayed on the GPU box, which has no reference tree):
    DINOv2 `init_weights` (`vision_transformer.py:172-177,331-336`: trunc_normal(0.02) linears with zero bias,
    pos_embed trunc_normal(0.02), cls N(0,1e-6), LayerScale 1.0 from `hubconf.py:38`), torch's default
    kaiming_uniform(a=sqrt 5) = U(+-1/sqrt(fan_in)) for every other Conv2d / ConvTranspose2d / Linear and its bias,
    identity LayerNorm / BatchNorm, trunc_normal(0.02) Swin position tables (`swin_layers.py:130,408`).
    oracle/make_golden.py checks the per-tensor statistics against a freshly constructed reference model.  With
    these weights the network output is nearly constant (every branch is far from trained), the regime the
    variance-preserving `synthetic_state_dict` deliberately avoids."""
    g = torch.Generator().manual_seed(seed)
    layout = state_layout(config)
    sd = OrderedDict()

    def tn(shape, std):
        return (torch.randn(shape, generator=g, dtype=torch.float32) * std).clamp_(-2.0, 2.0)   # trunc_normal_(a=-2, b=2)

    def uni(shape, bound):
        return (torch.rand(shape, generator=g, dtype=torch.float32) * 2 - 1) * bound

    fan = {}
    for key, (shape, dt, kind) in layout.items():
        leaf = key.split('.')[-1]
        vit = 'core.core.pretrained.' in key
        if key.endswith('relative_position_index'):
            t = relative_position_index()
        elif leaf == 'k_idx':
            t = torch.arange(shape[1]).view(shape)
        elif leaf == 'K_minus_1':
            t = torch.full(shape, float(layout[key.replace('K_minus_1', 'k_idx')][0][1] - 1))
        elif leaf == 'num_batches_tracked':
            t = torch.zeros((), dtype=torch.int64)
        elif leaf == 'running_mean':
            t = torch.zeros(shape)
        elif leaf == 'running_var':
            t = torch.ones(shape)
        elif leaf == 'gamma':
            t = torch.ones(shape)
        elif leaf == 'cls_token':
            t = torch.randn(shape, generator=g) * 1e-6
        elif leaf == 'mask_token':
            t = torch.zeros(shape)
        elif leaf in ('pos_embed', 'absolute_pos_embed', 'relative_position_bias_table'):
            t = tn(shape, 0.02)
        elif leaf == 'weight' and len(shape) == 1:
            t = torch.ones(shape)
        elif leaf == 'weight':
            if 'resize_layers.0' in key or 'resize_layers.1' in key:        # ConvTranspose2d weight (in, out, k, k)
                fan_in = shape[1] * shape[2] * shape[3]
            else:
                fan_in = 1
                for s_ in shape[1:]:
                    fan_in *= s_
            fan[key[:-len('weight')]] = fan_in
            if vit and 'patch_embed' not in key:
                t = tn(shape, 0.02)
            else:
                t = uni(shape, 1.0 / math.sqrt(fan_in))
        elif leaf == 'bias':
            pre = key[:-len('bias')]
            if (pre + 'weight') in layout and len(layout[pre + 'weight'][0]) == 1:    # LayerNorm / BatchNorm
                t = torch.zeros(shape)
            elif vit and 'patch_embed' not in key:
                t = torch.zeros(shape)
            else:
                t = uni(shape, 1.0 / math.sqrt(fan[pre]))
        else:
            raise AssertionError(key)
        sd[key] = t.to(dt)
    return sd
