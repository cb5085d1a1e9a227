"""CPU oracle for the PatchFusion per-tile inference hot path — TEST INFRASTRUCTURE, NOT PRODUCT.

A plain PyTorch fp32 restatement (functional, straight from a state dict, NCHW like the reference) of
`PatchFusion.forward(mode='infer')` and everything under it.  Only tests/, `__graft_entry__.smoke()` and
bench.py's `cpu_baseline` / `--impl reference` leg may import this module; the product package
(patchfusion_b200/) never does and fails loudly when its CUDA library is missing.

Pinning: oracle/make_golden.py runs the *real* reference (imported from a checkout through oracle/shims) and this restatement on the same seeded weights/inputs, asserts they agree to fp32 rounding
and writes tests/golden/*.npz; tests/test_oracle_golden.py re-checks the restatement against those fixtures
wherever the reference tree is absent.

Reference citations (paths in the zhyever/PatchFusion tree):
  PF  estimator/models/patchfusion.py            BP  estimator/models/baseline_pretrain.py
  GF  estimator/models/blocks/guided_fusion_model.py   SW  estimator/models/blocks/swin_layers.py
  MU  estimator/models/utils.py                  ZD  external/zoedepth/models/zoedepth/zoedepth_v1.py
  DAC external/zoedepth/models/base_models/depth_anything.py
  ATT/DIS/LB external/zoedepth/models/layers/{attractor,dist_layers,localbins_layers}.py
  DPT/BLK external/depth_anything/{dpt,blocks}.py
  VIT external/torchhub/facebookresearch_dinov2_main/vision_transformer.py  DL .../dinov2/layers/*.py
"""
import math
import random

import numpy as np
import torch
import torch.nn.functional as F

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
WINDOW = 12


def _get(cfg, k, d=None):
    return cfg.get(k, d) if isinstance(cfg, dict) else getattr(cfg, k, d)


def up(x, size):
    """bilinear, align_corners=True — the only resize the network itself uses (BLK:147-149, ATT:175-183, GF:98)."""
    if tuple(x.shape[-2:]) == tuple(size):
        return x
    return F.interpolate(x, size=tuple(size), mode='bilinear', align_corners=True)


class Weights:
    """Prefix view over a flat state dict."""

    def __init__(self, sd, prefix=''):
        self.sd, self.prefix = sd, prefix

    def sub(self, p):
        return Weights(self.sd, self.prefix + p)

    def __call__(self, k):
        return self.sd[self.prefix + k]

    def has(self, k):
        return (self.prefix + k) in self.sd

    def conv(self, name, x, stride=1, padding=0):
        b = self(name + '.bias') if self.has(name + '.bias') else None
        return F.conv2d(x, self(name + '.weight'), b, stride=stride, padding=padding)

    def linear(self, name, x):
        return F.linear(x, self(name + '.weight'), self(name + '.bias'))

    def ln(self, name, x, eps):
        return F.layer_norm(x, (x.shape[-1],), self(name + '.weight'), self(name + '.bias'), eps)


# --------------------------------------------------------------------------------------------------------------
# DINOv2 encoder (VIT:179-231, 271-321; DL/block.py:82-107; DL/attention.py:49-62; DL/mlp.py:35-41)
# --------------------------------------------------------------------------------------------------------------
def interpolated_pos_embed(pos_embed, gh, gw):
    """VIT:179-210 — bicubic resample of the 37x37 table with scale_factor=((gh+0.1)/37, (gw+0.1)/37)."""
    n = pos_embed.shape[1] - 1
    s = int(math.sqrt(n))
    if gh == s and gw == s:
        return pos_embed
    cls_pe, patch_pe = pos_embed[:, :1], pos_embed[:, 1:]
    d = pos_embed.shape[-1]
    grid = patch_pe.reshape(1, s, s, d).permute(0, 3, 1, 2)
    grid = F.interpolate(grid, scale_factor=((gh + 0.1) / s, (gw + 0.1) / s), mode='bicubic', antialias=False)
    assert grid.shape[-2:] == (gh, gw)
    return torch.cat([cls_pe, grid.permute(0, 2, 3, 1).reshape(1, gh * gw, d)], dim=1)


def vit_tokens(w, x):
    """patch embed + cls + pos (VIT:212-219).  x: (B,3,H,W) already normalised."""
    B, _, H, W = x.shape
    t = w.conv('patch_embed.proj', x, stride=14).flatten(2).transpose(1, 2)
    t = torch.cat([w('cls_token').expand(B, -1, -1), t], dim=1)
    return t + interpolated_pos_embed(w('pos_embed'), H // 14, W // 14)


def vit_block(w, x, heads):
    B, N, D = x.shape
    hd = D // heads
    h = w.ln('norm1', x, 1e-6)
    qkv = w.linear('attn.qkv', h).reshape(B, N, 3, heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0] * hd ** -0.5, qkv[1], qkv[2]
    a = (q @ k.transpose(-2, -1)).softmax(dim=-1)
    h = (a @ v).transpose(1, 2).reshape(B, N, D)
    x = x + w('ls1.gamma') * w.linear('attn.proj', h)
    h = w.ln('norm2', x, 1e-6)
    h = w.linear('mlp.fc2', F.gelu(w.linear('mlp.fc1', h)))
    return x + w('ls2.gamma') * h


def vit_last4(w, x, depth, heads, taps=None):
    """get_intermediate_layers(x, 4): final-LN'd outputs of the LAST four blocks, cls dropped (DPT:149, VIT:297-321)."""
    t = vit_tokens(w, x)
    if taps is not None:
        taps['tokens'] = t
    outs = []
    for i in range(depth):
        t = vit_block(w.sub('blocks.%d.' % i), t, heads)
        if taps is not None:
            taps['block%d' % i] = t
        if i >= depth - 4:
            outs.append(w.ln('norm', t, 1e-6)[:, 1:])
    return outs


# --------------------------------------------------------------------------------------------------------------
# DPT head (DPT:97-130, BLK:69-153) — returns rel depth and the six hooked taps (DAC:299-321)
# --------------------------------------------------------------------------------------------------------------
def _rcu(w, x):
    y = w.conv('conv1', F.relu(x), padding=1)
    y = w.conv('conv2', F.relu(y), padding=1)
    return y + x


def _ffb(w, x, skip, size):
    if skip is not None:
        x = x + _rcu(w.sub('resConfUnit1.'), skip)
    x = _rcu(w.sub('resConfUnit2.'), x)
    x = up(x, size)
    return w.conv('out_conv', x)


def dpt_head(w, feats, gh, gw):
    lay = []
    for i, f in enumerate(feats):
        B, _, D = f.shape
        x = f.permute(0, 2, 1).reshape(B, D, gh, gw)
        x = w.conv('projects.%d' % i, x)
        if i == 0:
            x = F.conv_transpose2d(x, w('resize_layers.0.weight'), w('resize_layers.0.bias'), stride=4)
        elif i == 1:
            x = F.conv_transpose2d(x, w('resize_layers.1.weight'), w('resize_layers.1.bias'), stride=2)
        elif i == 3:
            x = w.conv('resize_layers.3', x, stride=2, padding=1)
        lay.append(x)
    s = w.sub('scratch.')
    rn = [s.conv('layer%d_rn' % (i + 1), lay[i], padding=1) for i in range(4)]
    p4 = _ffb(s.sub('refinenet4.'), rn[3], None, rn[2].shape[-2:])
    p3 = _ffb(s.sub('refinenet3.'), p4, rn[2], rn[1].shape[-2:])
    p2 = _ffb(s.sub('refinenet2.'), p3, rn[1], rn[0].shape[-2:])
    p1 = _ffb(s.sub('refinenet1.'), p2, rn[0], (rn[0].shape[-2] * 2, rn[0].shape[-1] * 2))
    o = s.conv('output_conv1', p1, padding=1)
    o = up(o, (gh * 14, gw * 14))
    out_conv = F.relu(s.conv('output_conv2.0', o, padding=1))          # hook 'out_conv' = post-ReLU (DAC:302-304)
    rel = F.relu(s.conv('output_conv2.2', out_conv))                   # + F.relu in DPT:155 (idempotent)
    return rel, dict(out_conv=out_conv, l4_rn=rn[3], r4=p4, r3=p3, r2=p2, r1=p1)


# --------------------------------------------------------------------------------------------------------------
# Metric-bins head (ZD:173-219, PF:297-339, ATT:164-208, DIS:36-121, LB:84-117)
# --------------------------------------------------------------------------------------------------------------
def _mlp2(w, x, act2=None):
    x = w.conv('_net.2', F.relu(w.conv('_net.0', x)))
    return act2(x) if act2 is not None else x


def inv_attractor(dx, alpha=300.0, gamma=2):
    """ATT:44-57 with its TorchScript DEFAULTS — the layer never forwards the configured alpha/gamma (ATT:191-195)."""
    return dx / (1 + alpha * dx.pow(gamma))


def exp_attractor(dx, alpha=300.0, gamma=2):
    """ATT:29-41, same defaults."""
    return torch.exp(-alpha * dx.abs().pow(gamma)) * dx


def attractor_update(A, b_prev, kind='sum', attractor_type='exp'):
    """One AttractorLayerUnnormed step after its MLP (ATT:179-205): A (B,nA,h,w) attractor points, b_prev
    (B,nbins,h',w') bin centres up-sampled to (h, w) and shifted by the mean or sum over the attractors."""
    b = up(b_prev, A.shape[-2:])
    dist = exp_attractor if attractor_type == 'exp' else inv_attractor                            # ATT:186-189
    delta = dist(A.unsqueeze(2) - b.unsqueeze(1))
    delta = delta.mean(dim=1) if kind == 'mean' else delta.sum(dim=1)
    return b + delta


def log_binomial_depth(pt, b_centers, min_t, max_t):
    """ConditionalLogBinomial after its MLP (DIS:110-121, LogBinomial DIS:51-69) and the expectation over the bin
    centres up-sampled to pt's size (ZD:214-219): pt (B,4,H,W) softplus outputs, b_centers (B,K,h,w) -> (B,1,H,W)."""
    p, t = pt[:, :2] + 1e-4, pt[:, 2:] + 1e-4
    p = p[:, 0] / (p[:, 0] + p[:, 1])
    t = (t[:, 0] / (t[:, 0] + t[:, 1])).unsqueeze(1)
    t = (max_t - min_t) * t + min_t
    # LogBinomial (DIS:51-69), Stirling form of log C(K-1, k)
    K = b_centers.shape[1]
    k = torch.arange(K, dtype=torch.float32, device=pt.device).view(1, K, 1, 1)
    n_ = torch.tensor(float(K - 1), device=pt.device) + 1e-7
    k_ = k + 1e-7
    logc = n_ * torch.log(n_) - k_ * torch.log(k_) - (n_ - k_) * torch.log(n_ - k_ + 1e-7)
    p = p.unsqueeze(1)
    q = torch.clamp(1 - p, 1e-4, 1)
    p = torch.clamp(p, 1e-4, 1)
    y = logc + k * torch.log(p) + (K - 1 - k) * torch.log(q)
    prob = torch.softmax(y / t, dim=1)
    return torch.sum(prob * up(b_centers, pt.shape[-2:]), dim=1, keepdim=True)


def metric_head(w, x, x_blocks, last, rel_cond, hp, taps=None):
    """x: bottleneck (B,C,h0,w0); x_blocks: 4 maps low->high; last: (B,32,H,W); rel_cond: (B,1,H,W)."""
    b_prev = _mlp2(w.sub('seed_bin_regressor.'), x, F.softplus)
    prev_emb = _mlp2(w.sub('seed_projector.'), x)
    for i, xb in enumerate(x_blocks):
        emb = _mlp2(w.sub('projectors.%d.' % i), xb)
        A = _mlp2(w.sub('attractors.%d.' % i), emb + up(prev_emb, xb.shape[-2:]), F.softplus)
        b_prev = attractor_update(A, b_prev, _get(hp, 'attractor_kind', 'sum'), _get(hp, 'attractor_type', 'exp'))
        prev_emb = emb
        if taps is not None:
            taps['b%d' % i] = b_prev
    size = last.shape[-2:]
    z = torch.cat([last, up(rel_cond, size), up(prev_emb, size)], dim=1)
    c = w.sub('conditional_log_binomial.')
    pt = F.softplus(c.conv('mlp.2', F.gelu(c.conv('mlp.0', z))))
    return log_binomial_depth(pt, b_prev, _get(hp, 'min_temp'), _get(hp, 'max_temp'))


# --------------------------------------------------------------------------------------------------------------
# One branch = ZoeDepth over Depth-Anything (PF:189-225 -> ZD:125-233 -> DAC:262-278)
# --------------------------------------------------------------------------------------------------------------
def branch_forward(sd, prefix, image, hp, taps=None):
    """image (B,3,H,W) in [0,1], un-normalised.  Returns depth (B,1,H,W) and the 6 features low->high
    [x_d0, r4, r3, r2, r1, out_conv] (PF:198-204)."""
    from patchfusion_b200.params import ENCODERS
    enc = ENCODERS[_get(hp, 'midas_model_type')]
    w = Weights(sd, prefix)
    mean = torch.tensor(IMAGENET_MEAN, device=image.device).view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD, device=image.device).view(1, 3, 1, 1)
    x = (image - mean) / std
    H, W = x.shape[-2:]
    feats = vit_last4(w.sub('core.core.pretrained.'), x, enc['depth'], enc['heads'], taps)
    if taps is not None:
        for i, f in enumerate(feats):
            taps['vit_out%d' % i] = f
    rel, t = dpt_head(w.sub('core.core.depth_head.'), feats, H // 14, W // 14)
    x_d0 = w.conv('conv2', t['l4_rn'])
    blocks = [t['r4'], t['r3'], t['r2'], t['r1']]
    depth = metric_head(w, x_d0, blocks, t['out_conv'], rel, hp, taps)
    if taps is not None:
        taps['rel'] = rel
    return depth, [x_d0] + blocks + [t['out_conv']]


# --------------------------------------------------------------------------------------------------------------
# ROI crop-zoom (PF:240-257, GF:202): torchvision.ops.roi_align(feat, boxes, (h,w), h/Hp, aligned=True) restated.
# With roi no larger than the output grid the adaptive sampling ratio is ceil(roi/out)=1: ONE bilinear tap per bin
# centre, torchvision edge rules (zero outside [-1, size], clamp to the border otherwise).
# --------------------------------------------------------------------------------------------------------------
def roi_crop_zoom(feat, boxes, scale):
    """feat (1,C,h,w); boxes (T,4) x1,y1,x2,y2 in patch_process pixel units; -> (T,C,h,w)."""
    _, C, h, w = feat.shape
    outs = []
    for bx in boxes.tolist():
        x1, y1, x2, y2 = [v * scale - 0.5 for v in bx]
        bw, bh = (x2 - x1) / w, (y2 - y1) / h
        assert math.ceil(bw) <= 1 and math.ceil(bh) <= 1, "roi larger than output: multi-sample bins not restated"
        ys = y1 + (torch.arange(h, dtype=torch.float32, device=feat.device) + 0.5) * bh
        xs = x1 + (torch.arange(w, dtype=torch.float32, device=feat.device) + 0.5) * bw

        def prep(c, size):
            valid = (c >= -1.0) & (c <= size)
            c = c.clamp(min=0)
            lo = c.floor().long()
            edge = lo >= size - 1
            lo = torch.where(edge, torch.full_like(lo, size - 1), lo)
            hi = torch.where(edge, lo, lo + 1)
            c = torch.where(edge, lo.float(), c)
            frac = c - lo.float()
            return lo, hi, frac, valid

        yl, yh, fy, vy = prep(ys, h)
        xl, xh, fx, vx = prep(xs, w)
        f = feat[0]
        top = f[:, yl][:, :, xl] * (1 - fx) + f[:, yl][:, :, xh] * fx
        bot = f[:, yh][:, :, xl] * (1 - fx) + f[:, yh][:, :, xh] * fx
        o = top * (1 - fy)[:, None] + bot * fy[:, None]
        o = o * (vy[:, None] & vx[None, :]).float()
        outs.append(o)
    return torch.stack(outs)


# --------------------------------------------------------------------------------------------------------------
# G2L window attention (SW:133-164, 218-268, 325-355, 410-432) on the whole-image coarse feature
# --------------------------------------------------------------------------------------------------------------
def _windows(x, ws):
    B, H, W, C = x.shape
    x = x.view(B, H // ws, ws, W // ws, ws, C)
    return x.permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, C)


def _unwindows(win, ws, H, W):
    C = win.shape[-1]
    x = win.view(-1, H // ws, W // ws, ws, ws, C)
    return x.permute(0, 1, 3, 2, 4, 5).reshape(-1, H, W, C)


def shift_mask(Hp, Wp, ws, device):
    """SW:327-345."""
    sh = ws // 2
    img = torch.zeros(1, Hp, Wp, 1, device=device)
    cnt = 0
    for hs in (slice(0, -ws), slice(-ws, -sh), slice(-sh, None)):
        for wsl in (slice(0, -ws), slice(-ws, -sh), slice(-sh, None)):
            img[:, hs, wsl, :] = cnt
            cnt += 1
    mw = _windows(img, ws).squeeze(-1)
    m = mw.unsqueeze(1) - mw.unsqueeze(2)
    return torch.where(m != 0, torch.full_like(m, -100.0), torch.zeros_like(m))


def window_attention(qkv, table, index, heads, mask=None):
    """SW:139-161 without the projections: qkv (nW, N, 3C) of the windowed tokens, the (2ws-1)^2 x heads bias table,
    the (N, N) relative position index and the (nW, N, N) shift mask (None: no shift) -> (nW, N, C)."""
    nW, N, C3 = qkv.shape
    C = C3 // 3
    hd = C // heads
    qkv = qkv.reshape(nW, N, 3, heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0] * hd ** -0.5, qkv[1], qkv[2]
    a = q @ k.transpose(-2, -1)
    bias = table[index.reshape(-1)]
    a = a + bias.view(N, N, heads).permute(2, 0, 1).unsqueeze(0)
    if mask is not None:
        a = a + mask.unsqueeze(1)
    a = a.softmax(dim=-1)
    return (a @ v).transpose(1, 2).reshape(nW, N, C)


def swin_block(w, x, H, W, heads, shift, mask):
    B, L, C = x.shape
    ws = WINDOW
    h = w.ln('norm1', x, 1e-5).view(B, H, W, C)
    pb, pr = (ws - H % ws) % ws, (ws - W % ws) % ws
    h = F.pad(h, (0, 0, 0, pr, 0, pb))
    Hp, Wp = H + pb, W + pr
    if shift:
        h = torch.roll(h, shifts=(-shift, -shift), dims=(1, 2))
    win = _windows(h, ws)
    o = window_attention(w.linear('attn.qkv', win), w('attn.relative_position_bias_table'),
                         w('attn.relative_position_index'), heads, mask if shift else None)
    o = w.linear('attn.proj', o)
    o = _unwindows(o, ws, Hp, Wp)
    if shift:
        o = torch.roll(o, shifts=(shift, shift), dims=(1, 2))
    o = o[:, :H, :W, :].reshape(B, H * W, C)
    x = x + o
    h = w.ln('norm2', x, 1e-5)
    return x + w.linear('mlp.fc2', F.gelu(w.linear('mlp.fc1', h)))


def g2l_forward(w, feat, depth, heads):
    """feat (1,C,h,w) -> (1,C,h,w).  area_prior is None on the inference path (GF:201)."""
    B, C, H, W = feat.shape
    x = feat.flatten(2).transpose(1, 2) + w('absolute_pos_embed')
    ws = WINDOW
    Hp, Wp = math.ceil(H / ws) * ws, math.ceil(W / ws) * ws
    mask = shift_mask(Hp, Wp, ws, feat.device)
    for b in range(depth):
        x = swin_block(w.sub('g2l_layer.blocks.%d.' % b), x, H, W, heads, 0 if b % 2 == 0 else ws // 2, mask)
    x = w.ln('g2l_layer_norm', x, 1e-5)
    return x.view(B, H, W, C).permute(0, 3, 1, 2).contiguous()


# --------------------------------------------------------------------------------------------------------------
# Guided fusion U-Net (GF:163-207) and fusion_forward (PF:259-340)
# --------------------------------------------------------------------------------------------------------------
def _double_conv_bn(w, x):
    for ci, bi in ((0, 1), (3, 4)):
        x = w.conv('double_conv.%d' % ci, x, padding=1)
        p = 'double_conv.%d.' % bi
        x = F.batch_norm(x, w(p + 'running_mean'), w(p + 'running_var'), w(p + 'weight'), w(p + 'bias'),
                         training=False, eps=1e-5)
        x = F.relu(x)
    return x


def _double_conv(w, x):
    x = F.relu(w.conv('double_conv.0', x, padding=1))
    return F.relu(w.conv('double_conv.2', x, padding=1))


def g2l_all(sd, coarse_feats, gf_hp):
    """The six tile-invariant G2L maps (hoisted: GF:201 recomputes them per micro-batch with identical input)."""
    from patchfusion_b200.params import G2L_DEPTH, G2L_HEADS
    depth = list(_get(gf_hp, 'depth', G2L_DEPTH))[::-1]
    heads = list(_get(gf_hp, 'num_heads', G2L_HEADS))[::-1]
    w = Weights(sd, 'guided_fusion.')
    return [g2l_forward(w.sub('g2l_list.%d.' % i), coarse_feats[i], depth[i], heads[i]) for i in range(6)]


def fusion_forward(sd, cfg, fine_depth, crops, fine_feats, boxes, coarse_depth_roi, coarse_feats_roi, g2l_maps,
                   taps=None):
    """PF:259-340.  boxes (p,4) in patch_process units.  g2l_maps: outputs of g2l_all on the whole-image feats."""
    P = _get(cfg, 'patch_process_shape')
    w = Weights(sd)
    guide = [w.conv('fusion_conv_list.%d' % i, torch.cat([coarse_feats_roi[i], fine_feats[i]], 1), padding=1)
             for i in range(5)]                      # level 5's fused map is never read by the U-Net (GF:198)
    g = w.sub('guided_fusion.')
    x = _double_conv_bn(g.sub('inc.'), torch.cat([coarse_depth_roi, fine_depth, crops], dim=1))
    enc = [x]
    for i in range(5):
        x = _double_conv_bn(g.sub('down_conv_list.%d.maxpool_conv.1.' % i), F.max_pool2d(x, 2))
        enc.append(x)
    enc = enc[::-1]
    outs, prev = [], None
    for i in range(6):
        h, wd = g2l_maps[i].shape[-2:]
        e = up(enc[i], (h, wd))
        if i > 0:
            e = _double_conv(g.sub('up_conv_list.%d.conv.' % (i - 1)),
                             torch.cat([e, up(torch.cat([prev, guide[i - 1]], 1), (h, wd))], 1))
        c = roi_crop_zoom(g2l_maps[i], boxes, h / P[0])
        prev = _double_conv(g.sub('convs.%d.' % i), torch.cat([e, c], 1))
        outs.append(prev)
        if taps is not None:
            taps['fuse%d' % i] = prev
    hp = _get(cfg, 'coarse_branch')
    last = outs[5]
    rel = torch.zeros(last.shape[0], 1, *last.shape[-2:], device=last.device)
    return metric_head(w, outs[0], outs[1:5], last, rel, hp, taps)


# --------------------------------------------------------------------------------------------------------------
# Tiling / stitching (BP:91-119, 143-331; MU:21-47; PF:401-453)
# --------------------------------------------------------------------------------------------------------------
def prepare_tile_cfg(image_raw_shape, patch_split_num, patch_process_shape):
    H, W = image_raw_shape
    sh, sw = patch_split_num
    assert H % (2 * sh) == 0, 'image height should be divisible by 2 * patch_split_num[0]'
    assert W % (2 * sw) == 0, 'image width should be divisible by 2 * patch_split_num[1]'
    return dict(patch_split_num=(sh, sw), image_raw_shape=(H, W), patch_raw_shape=(H // sh, W // sw),
                patch_reensemble_shape=(patch_process_shape[0] * sh, patch_process_shape[1] * sw))


def gaussian_mask(size):
    """MU:38-47 via OpenCV (a host-side library call in the reference too)."""
    import cv2
    m = np.zeros(size, dtype=np.float32)
    sigma = int(size[0] / 16)
    k = int(2 * np.ceil(2 * int(size[0] / 16)) + 1)
    m[int(0.1 * size[0]):size[0] - int(0.1 * size[0]), int(0.1 * size[1]):size[1] - int(0.1 * size[1])] = 1
    m = cv2.GaussianBlur(m, (k, k), sigma)
    return ((m - m.min()) / (m.max() - m.min())).astype(np.float32)


class RunningAverage:
    """MU:21-36 — sequential running average, kept literal (full-canvas updates) on purpose."""

    def __init__(self, pred, cnt):
        self.avg, self.cnt = pred / cnt, cnt

    def update(self, pred, cnt):
        self.avg = (pred + self.cnt * self.avg) / (self.cnt + cnt)
        self.cnt = self.cnt + cnt

    def resize(self, size):
        self.avg = F.interpolate(self.avg[None, None], size=tuple(size)).squeeze()            # nearest
        self.cnt = F.interpolate(self.cnt[None, None], size=tuple(size), mode='bilinear', align_corners=True).squeeze()


def tile_plan(tile_cfg, patch_process_shape, cai_mode):
    """Regular passes as [(raw (y,x), process (y,x))...] per pass (BP:232-254, PF:417-439)."""
    H, W = tile_cfg['image_raw_shape']
    h, w = tile_cfg['patch_raw_shape']
    ph, pw = patch_process_shape
    RH, RW = tile_cfg['patch_reensemble_shape']
    offs = [((0, 0), (0, 0))]
    if cai_mode == 'm2' or cai_mode[0] == 'r':
        offs += [((0, w // 2), (0, pw // 2)), ((h // 2, 0), (ph // 2, 0)), ((h // 2, w // 2), (ph // 2, pw // 2))]
    passes = []
    for (oy, ox), (py, px) in offs:
        ny, nx = (H - oy) // h, (W - ox) // w
        assert ny == (RH - py) // ph and nx == (RW - px) // pw
        passes.append([((h * a + oy, w * b + ox), (ph * a + py, pw * b + px)) for a in range(ny) for b in range(nx)])
    return passes


class Oracle:
    """Whole `forward(mode='infer')` (PF:401-453)."""

    def __init__(self, sd, cfg):
        self.sd, self.cfg = sd, cfg
        self.P = tuple(_get(cfg, 'patch_process_shape'))
        self.hp_c, self.hp_f = _get(cfg, 'coarse_branch'), _get(cfg, 'fine_branch')

    def resizer(self, x):
        return up(x, self.P)

    def coarse(self, image_lr, taps=None):
        return branch_forward(self.sd, 'coarse_branch.', image_lr, self.hp_c, taps)

    def tiles(self, image_hr, raw_boxes, coarse_depth, coarse_feats, g2l_maps, process_num, tile_cfg):
        """raw_boxes: list of (y, x) tile origins in raw pixels; returns (T,1,ph,pw) fused depth."""
        h, w = tile_cfg['patch_raw_shape']
        H, W = tile_cfg['image_raw_shape']
        crops = torch.cat([self.resizer(image_hr[:, :, y:y + h, x:x + w]) for (y, x) in raw_boxes])
        fx, fy = 1 / W * self.P[1], 1 / H * self.P[0]
        factor = torch.tensor([[fx, fy, fx, fy]], device=image_hr.device)             # fp32, as BP:275-282
        boxes = torch.tensor([[x, y, x + w, y + h] for (y, x) in raw_boxes], device=image_hr.device).int() * factor
        preds = []
        for s in range(0, len(raw_boxes), process_num):
            bx, cr = boxes[s:s + process_num], crops[s:s + process_num]
            c_roi = [roi_crop_zoom(f, bx, f.shape[-2] / self.P[0]) for f in coarse_feats]
            d_roi = roi_crop_zoom(coarse_depth, bx, coarse_depth.shape[-2] / self.P[0])
            fd, ff = branch_forward(self.sd, 'fine_branch.', cr, self.hp_f)
            preds.append(fusion_forward(self.sd, self.cfg, fd, cr, ff, bx, d_roi, c_roi, g2l_maps))
        return torch.cat(preds)

    def infer(self, image_lr, image_hr, tile_cfg=None, cai_mode='m1', process_num=4):
        cfg = self.cfg
        if tile_cfg is None:
            tile_cfg = dict(image_raw_shape=_get(cfg, 'image_raw_shape'), patch_split_num=_get(cfg, 'patch_split_num'))
        tc = prepare_tile_cfg(tile_cfg['image_raw_shape'], tile_cfg['patch_split_num'], self.P)
        assert image_hr.shape[0] == 1
        cd, cf = self.coarse(image_lr)
        g2l = g2l_all(self.sd, cf, _get(cfg, 'guided_fusion'))
        dev = image_hr.device
        mask = torch.tensor(gaussian_mask(self.P) + 1e-3, device=dev)
        ph, pw = self.P
        avg = None
        for pi, tiles in enumerate(tile_plan(tc, self.P, cai_mode)):
            preds = self.tiles(image_hr, [t[0] for t in tiles], cd, cf, g2l, process_num, tc)
            if pi == 0:
                cnt = torch.zeros(tc['patch_reensemble_shape'], device=dev)
                acc = torch.zeros(tc['patch_reensemble_shape'], device=dev)
                for (_, (py, px)), d in zip(tiles, preds):
                    cnt[py:py + ph, px:px + pw] = mask
                    acc[py:py + ph, px:px + pw] = d[0] * mask
                avg = RunningAverage(acc, cnt)
            else:
                for (_, (py, px)), d in zip(tiles, preds):
                    cnt = torch.zeros(tc['patch_reensemble_shape'], device=dev)
                    acc = torch.zeros(tc['patch_reensemble_shape'], device=dev)
                    cnt[py:py + ph, px:px + pw] = mask
                    acc[py:py + ph, px:px + pw] = d[0] * mask
                    avg.update(acc, cnt)
        if cai_mode[0] == 'r':
            h, w = tc['patch_raw_shape']
            H, W = tc['image_raw_shape']
            mask = torch.tensor(gaussian_mask((h, w)) + 1e-3, device=dev)
            avg.resize((H, W))
            for _ in range(int(cai_mode[1:]) // process_num):
                ys = [random.randint(0, H - h - 1) for _ in range(process_num)]     # BP:155-156 draw order
                x0 = random.randint(0, W - w - 1)
                preds = self.tiles(image_hr, [(y, x0) for y in ys], cd, cf, g2l, process_num, tc)
                preds = F.interpolate(preds, (h, w))                                 # nearest (BP:203)
                for y, d in zip(ys, preds):
                    cnt = torch.zeros((H, W), device=dev)
                    acc = torch.zeros((H, W), device=dev)
                    cnt[y:y + h, x0:x0 + w] = mask
                    acc[y:y + h, x0:x0 + w] = d[0] * mask
                    avg.update(acc, cnt)
        return avg.avg[None, None]
