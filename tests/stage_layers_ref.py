"""The bf16 GEMMs and convs each stage call issues, derived from the config alone, and fp64 references of the
reference's modules built from the state dict (tests/test_gpu_stage_layers.py on the GPU, test_stage_layers_host.py on
the CPU).

`layer_specs(cfg, call)` lists, in issue order, the layers of one call of pf_branch_forward ('coarse' / 'fine'),
pf_g2l_forward ('g2l') or pf_fusion_forward ('fusion').  Each spec names the layer as its "L.<key>.*" taps do (the
engine's weight key), the state-dict modules it computes, its sources' channels, N, the grid its output covers per image
and its epilogue.  Every conv / linear weight of the state dict belongs to exactly one spec or to `never_run`.

`reference(spec, sd, ins, ...)` is the module applied in fp64 to the tapped inputs, with the bound the kernel must meet:
  ulp_bf16(ref) (2^-24 |ref| for fp32 outputs) + (K + 2) 2^-24 (|a| * |w| + |b|) through the epilogue, the second term
  computed in fp64 by the same op on absolute values.
The path stores weights in bf16 (pf_pack_weight), so the module's effective weight (a BatchNorm's scale folded in) is
rounded to bf16 once; everything else is fp64.  Activation errors are the documented ones of test_gpu_epilogue_act.py.
"""
import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24
GELU_LIP = 1.13          # max |GELU'(z)| = 1.1289 (at z = 2^0.5)


def _pad(n, m):
    return (n + m - 1) // m * m


def _hp(cfg):
    from patchfusion_b200.params import branch_hparams, guided_fusion_hparams
    P = tuple(cfg['patch_process_shape'])
    return P, branch_hparams(cfg['coarse_branch']), branch_hparams(cfg['fine_branch']), \
        guided_fusion_hparams(cfg['guided_fusion'], P)


def branch_grids(P):
    """per-image grids of a branch: the ViT grid, the four reassembled maps, output_conv1's and the image's"""
    gh, gw = P[0] // 14, P[1] // 14
    sz = [(gh * 4, gw * 4), (gh * 2, gw * 2), (gh, gw), ((gh - 1) // 2 + 1, (gw - 1) // 2 + 1)]
    return dict(g=(gh, gw), sz=sz, p1=(gh * 8, gw * 8), P=tuple(P))


def coarse_map_grids(P):
    """the six maps a branch returns, low -> high: x_d0, r4, r3, r2, r1, out_conv (the G2L / decoder levels)"""
    g = branch_grids(P)
    return [g['sz'][3], g['sz'][2], g['sz'][1], g['sz'][0], g['p1'], g['P']]


def _spec(key, mods, srcs, N, grid, kind='conv', k=1, act='none', **kw):
    s = dict(key=key, mods=mods, srcs=list(srcs), N=N, grid=tuple(grid), kind=kind, k=k, act=act, act2=None,
             res=0, gamma=None, copy=False, vt=False, f32=False, skip_main=False, tail=None, bn=None, in_grid=None)
    s.update(kw)
    return s


def _head(pre, C, hp, x_grid, block_grids, P, rel):
    from patchfusion_b200.params import normed_attractors, normed_seed
    t = hp['bin_centers_type']
    E, nb = hp['bin_embedding_dim'], hp['n_bins']
    sact = 'relu' if normed_seed(t) else 'softplus'
    aact = 'relu' if normed_attractors(t) else 'softplus'
    out = [_spec('head.seed_bin_regressor.0', [pre + 'seed_bin_regressor._net.0'], [C], 256, x_grid, act='relu'),
           _spec('head.seed_bin_regressor.2', [pre + 'seed_bin_regressor._net.2'], [256], nb, x_grid, act=sact,
                 f32=True),
           _spec('head.seed_projector.0', [pre + 'seed_projector._net.0'], [C], 128, x_grid, act='relu'),
           _spec('head.seed_projector.2', [pre + 'seed_projector._net.2'], [128], E, x_grid)]
    for i in range(4):
        m = 'projectors.%d' % i
        out += [_spec('head.%s.0' % m, [pre + m + '._net.0'], [C], 128, block_grids[i], act='relu'),
                _spec('head.%s.2' % m, [pre + m + '._net.2'], [128], E, block_grids[i])]
        m = 'attractors.%d' % i
        out.append(_spec('head.%s.0' % m, [pre + m + '._net.0', pre + m + '._net.2'], [E], 128, block_grids[i],
                         act='relu', tail=pre + m + '._net.2', act2=aact, skip_main=True,
                         n2=hp['n_attractors'][i], even=normed_attractors(t)))
    c = pre + 'conditional_log_binomial.'
    cin = 32 + 1 + E
    out.append(_spec('head.clb.0', [c + 'mlp.0', c + 'mlp.2'], [32, 1, E] if rel else [32, E], cin // 2, P, act='gelu',
                     tail=c + 'mlp.2', act2='softplus', skip_main=True, n2=4, drop_rel=not rel))
    return out


def branch_specs(cfg, which):
    P, hpc, hpf, _ = _hp(cfg)
    hp = hpc if which == 'coarse' else hpf
    pre = which + '_branch.'
    vit, dh = pre + 'core.core.pretrained.', pre + 'core.core.depth_head.'
    D, C, oc = hp['dim'], hp['features'], hp['out_channels']
    g = branch_grids(P)
    gh, gw = g['g']
    sz = g['sz']
    seq = (gh * gw + 1, 1)
    out = [_spec('patch', [vit + 'patch_embed.proj'], [588], D, (gh, gw), kind='linear', f32=True)]
    for i in range(hp['depth']):
        b = vit + 'blocks.%d.' % i
        out += [_spec('b%d.qkv' % i, [b + 'attn.qkv'], [D], 3 * D, seq, kind='linear', vt=True),
                _spec('b%d.proj' % i, [b + 'attn.proj'], [D], D, seq, kind='linear', f32=True, gamma=b + 'ls1.gamma'),
                _spec('b%d.fc1' % i, [b + 'mlp.fc1'], [D], 4 * D, seq, kind='linear', act='gelu'),
                _spec('b%d.fc2' % i, [b + 'mlp.fc2'], [4 * D], D, seq, kind='linear', f32=True, gamma=b + 'ls2.gamma')]
    for i in range(4):
        out.append(_spec('proj%d' % i, [dh + 'projects.%d' % i], [D], oc[i], (gh, gw)))
        if i < 2:
            out.append(_spec('rs%d' % i, [dh + 'resize_layers.%d' % i], [oc[i]], oc[i], sz[i], k='T%d' % (4 >> i),
                             in_grid=(gh, gw)))
        elif i == 3:
            out.append(_spec('rs3', [dh + 'resize_layers.3'], [oc[3]], oc[3], sz[3], k='s2', in_grid=(gh, gw)))
    s = dh + 'scratch.'
    for i in range(4):
        out.append(_spec('rn%d' % i, [s + 'layer%d_rn' % (i + 1)], [oc[i]], C, sz[i], k=3, copy=True))
    for wi in (4, 3, 2, 1):
        r = s + 'refinenet%d.' % wi
        for u in ((2,) if wi == 4 else (1, 2)):
            out += [_spec('ff%d.u%d.c1' % (wi, u), [r + 'resConfUnit%d.conv1' % u], [C], C, sz[wi - 1], k=3, act='relu'),
                    _spec('ff%d.u%d.c2' % (wi, u), [r + 'resConfUnit%d.conv2' % u], [C], C, sz[wi - 1], k=3,
                          res=2 if u == 1 else 1, copy=u == 1)]
        out.append(_spec('ff%d.out' % wi, [r + 'out_conv'], [C], C, sz[wi - 1]))
    out += [_spec('oc1', [s + 'output_conv1'], [C], C // 2, g['p1'], k=3),
            _spec('oc2.0', [s + 'output_conv2.0', s + 'output_conv2.2'], [C // 2], 32, P, k=3, act='relu',
                  tail=s + 'output_conv2.2', act2='relu', n2=1),
            _spec('conv2', [pre + 'conv2'], [C], C, sz[3])]
    return out + _head(pre, C, hp, sz[3], [sz[2], sz[1], sz[0], g['p1']], P, rel=True)


def g2l_specs(cfg):
    P, _, _, gf = _hp(cfg)
    inv = gf['in_channels'][::-1]
    depth = gf['depth'][::-1]
    out = []
    for i, (h, w) in enumerate(coarse_map_grids(P)):
        c, p = inv[i], 'guided_fusion.g2l_list.%d.g2l_layer.blocks.' % i
        pad = (_pad(h, 12), _pad(w, 12))
        for b in range(depth[i]):
            q = p + '%d.' % b
            out += [_spec('g2l%d.b%d.qkv' % (i, b), [q + 'attn.qkv'], [c], 3 * c, pad, kind='linear'),
                    _spec('g2l%d.b%d.proj' % (i, b), [q + 'attn.proj'], [c], c, pad, kind='linear', f32=True),
                    _spec('g2l%d.b%d.fc1' % (i, b), [q + 'mlp.fc1'], [c], 4 * c, (h, w), kind='linear', act='gelu'),
                    _spec('g2l%d.b%d.fc2' % (i, b), [q + 'mlp.fc2'], [4 * c], c, (h, w), kind='linear', f32=True,
                          gamma='ones')]
    return out


def fusion_specs(cfg):
    P, hpc, hpf, gf = _hp(cfg)
    C = hpf['features']
    ic = gf['in_channels']
    inv = ic[::-1]
    grids = coarse_map_grids(P)
    out = [_spec('fc%d' % i, ['fusion_conv_list.%d' % i], [C, C], C, grids[i], k=3) for i in range(5)]
    g = 'guided_fusion.'

    def dcbn(key, pre, cin, cout, grid):
        return [_spec(key + '.0', [pre + 'double_conv.0'], [cin], cout, grid, k=3, act='relu',
                      bn=pre + 'double_conv.1'),
                _spec(key + '.1', [pre + 'double_conv.3'], [cout], cout, grid, k=3, act='relu',
                      bn=pre + 'double_conv.4')]
    out += dcbn('inc', g + 'inc.', gf['n_channels'], ic[0], P)
    h, w = P
    for i in range(5):
        h, w = h // 2, w // 2
        out += dcbn('down%d' % i, g + 'down_conv_list.%d.maxpool_conv.1.' % i, ic[i], ic[i + 1], (h, w))
    for i in range(6):
        if i > 0:
            p = g + 'up_conv_list.%d.conv.double_conv.' % (i - 1)
            cin = inv[i] + 2 * inv[i - 1]
            out += [_spec('up%d.0' % i, [p + '0'], [inv[i], inv[i - 1], inv[i - 1]], cin, grids[i], k=3, act='relu'),
                    _spec('up%d.1' % i, [p + '2'], [cin], inv[i], grids[i], k=3, act='relu')]
        p = g + 'convs.%d.double_conv.' % i
        out += [_spec('cv%d.0' % i, [p + '0'], [inv[i], inv[i]], inv[i], grids[i], k=3, act='relu'),
                _spec('cv%d.1' % i, [p + '2'], [inv[i]], inv[i], grids[i], k=3, act='relu')]
    return out + _head('', inv[0], hpc, grids[0], grids[1:5], P, rel=False)


def layer_specs(cfg, call):
    if call in ('coarse', 'fine'):
        return branch_specs(cfg, call)
    return g2l_specs(cfg) if call == 'g2l' else fusion_specs(cfg)


def never_run(cfg):
    """conv / linear modules of the state dict that inference never runs"""
    out = []
    for b in ('coarse', 'fine'):
        # refinenet4's FeatureFusionBlock has no second input, so its resConfUnit1 is skipped (blocks.py:135-140)
        out += ['%s_branch.core.core.depth_head.scratch.refinenet4.resConfUnit1.conv%d' % (b, u) for u in (1, 2)]
    out.append('fusion_conv_list.5')            # level 5's fused map is never read by the U-Net (GF:198)
    # G2L's embed_proj embeds the area prior, which is None on the inference path (swin_layers.py:414-416, GF:201)
    out += ['guided_fusion.g2l_list.%d.embed_proj' % i for i in range(6)]
    return out


def weight_modules(sd):
    """the conv / linear modules of a state dict (a weight of two or more dimensions)"""
    return [k[:-len('.weight')] for k, v in sd.items() if k.endswith('.weight') and v.dim() >= 2]


# ---------------------------------------------------------------------------------------------------- fp64 references
def bf16_ulp(x):
    """spacing of bf16 values at |x| (the smallest normal spacing below 2^-126)"""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _act(name, z):
    if name == 'relu':
        return z.clamp_min(0)
    if name == 'gelu':
        return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))
    if name == 'softplus':          # torch.nn.Softplus(threshold=20)
        return torch.where(z > 20, z, torch.log1p(torch.exp(z.clamp_max(20))))
    return z


def _act_err(name, z, e_z):
    """|act(z + e) - act(z)| for |e| <= e_z plus the fp32 evaluation error of act (test_gpu_epilogue_act.py)"""
    if name == 'gelu':
        return GELU_LIP * e_z + z.abs() * (0.75e-7 + 4 * U) + 2.0 ** -126
    if name == 'softplus':
        return e_z + 8 * U * _act('softplus', z).abs() + 2.0 ** -126
    return e_z


def module_weight(spec, sd):
    """(the module's weight in fp64 rounded to bf16 as the path stores it, its bias in fp64 or None)"""
    m = spec['mods'][0]
    w = sd[m + '.weight'].double()
    b = sd[m + '.bias'].double() if (m + '.bias') in sd else None
    if spec['bn'] is not None:
        n = spec['bn']
        s = sd[n + '.weight'].double() / torch.sqrt(sd[n + '.running_var'].double() + 1e-5)
        w = w * s.view(-1, *([1] * (w.dim() - 1)))
        b = sd[n + '.bias'].double() - sd[n + '.running_mean'].double() * s
    if spec['key'] == 'patch':
        w = w.reshape(w.shape[0], -1)
    return w.to(torch.bfloat16).double(), b


def _nchw(t, B, grid):
    return t.double().reshape(B, grid[0], grid[1], -1).permute(0, 3, 1, 2)


def _rows(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def apply(spec, w, b, x, B):
    """the module on x (fp64: [rows, K] for a linear, NCHW for a conv) -> [rows, N]"""
    k = spec['k']
    if spec['kind'] == 'linear' or spec['key'] in ('patch',) or spec['key'].startswith('proj'):
        if x.dim() == 4:
            x = _rows(x)
        return F.linear(x, w.reshape(w.shape[0], -1), b)
    if isinstance(k, str) and k.startswith('T'):
        return _rows(F.conv_transpose2d(x, w, b, stride=int(k[1:])))
    if k == 's2':
        return _rows(F.conv2d(x, w, b, stride=2, padding=1))
    return _rows(F.conv2d(x, w, b, padding=w.shape[-1] // 2))


def reference(spec, sd, ins, B, extra):
    """fp64 reference and bound of every output part of one layer.  ins: the tapped sources, NHWC-able [rows, C] each
    (rs3: its producer's output at the ViT-grid resolution, as F.conv2d's input); extra: the tapped 'x', 'res1', 'res2'.
    -> {part: (ref, bound)} with parts out / out2 / out3 / vt as the layer has them."""
    w, b = module_weight(spec, sd)
    key = spec['key']
    if spec['kind'] == 'linear' or key.startswith('proj'):
        x = torch.cat([t.double() for t in ins], 1)
        if key == 'patch':
            x = x[:, :588]
    else:
        grid = spec['in_grid'] or spec['grid']
        x = torch.cat([_nchw(t, B, grid) for t in ins], 1)
        if spec.get('drop_rel'):                  # rel_cond is identically zero in the fusion head (PF:300,326-328)
            x = torch.cat([x[:, :32], torch.zeros_like(x[:, :1]), x[:, 32:]], 1)
    K = x.shape[1] * (w.shape[-1] * w.shape[-2] if w.dim() == 4 else 1)
    if isinstance(spec['k'], str) and spec['k'].startswith('T'):
        K = x.shape[1]                            # one tap per output pixel
    z = apply(spec, w, b, x, B)
    za = apply(spec, w.abs(), b.abs() if b is not None else None, x.abs(), B)
    e = (K + 2) * U * za
    v = _act(spec['act'], z)
    e = _act_err(spec['act'], z, e)
    parts = {}
    if spec['tail'] is not None:
        # the fused trailing layer reads the activated fp32 row v, not its bf16 store (include/pf_b200.h, pf_gemm_desc:
        # "out3[row, i] = act2(b2[i] + sum_j w2[i*N + j] * v[j])" on the activated row; pf_gemm.cu epilogue_chunk
        # accumulates it before any store), with the fp32 w2 as given
        t = spec['tail']
        w2 = sd[t + '.weight'].double().reshape(sd[t + '.weight'].shape[0], -1)
        b2 = sd[t + '.bias'].double()
        if spec.get('even'):                      # AttractorLayer reads only the even channels (attractor.py:104-106)
            w2, b2 = w2[0::2], b2[0::2]
        y = v @ w2.t() + b2
        ey = e @ w2.abs().t() + (spec['N'] + 2) * U * (v.abs() @ w2.abs().t() + b2.abs())
        ref3 = _act(spec['act2'], y)
        parts['out3'] = (ref3, _act_err(spec['act2'], y, ey) + U * ref3.abs())
    if spec['vt']:
        D = spec['N'] // 3
        parts['vt'] = (v[:, 2 * D:], bf16_ulp(v[:, 2 * D:]) + e[:, 2 * D:])
        v, e = v[:, :2 * D], e[:, :2 * D]
    if spec['gamma'] is not None:
        g = torch.ones(spec['N'], dtype=torch.float64, device=v.device) if spec['gamma'] == 'ones' else \
            sd[spec['gamma']].double()
        xs = extra['x'].double()
        r = xs + g * v
        e = g.abs() * e + 2 * U * (xs.abs() + (g * v).abs())
        v = r
    for i in range(spec['res']):
        rr = extra['res%d' % (i + 1)].double()
        e = e + 2 * U * (v.abs() + rr.abs())
        v = v + rr
    if not spec['skip_main']:
        tol = U * v.abs() if spec['f32'] else bf16_ulp(v)
        parts['out'] = (v, tol + e)
    if spec['copy']:
        parts['out2'] = (v.clamp_min(0), bf16_ulp(v) + e)
    return parts
