"""Device-side execution of the PatchFusion hot path on libpf_b200.

`Engine` packs the weights once (pf_pack_weight), describes them to the library as C structs (patchfusion_b200/stage.py
<-> include/pf_b200.h) and owns the workspaces; the kernel SEQUENCES live inside the library
(csrc/pf_stage.cu: pf_branch_forward / pf_g2l_forward / pf_fusion_forward), one call per stage:

    coarse/fine branch   reference `estimator/models/patchfusion.py:189-225` -> zoedepth_v1.py:125-233 ->
                         depth_anything.py:262-278 -> dpt.py:97-157 -> dinov2 vision_transformer.py:297-321
    G2L maps             `estimator/models/blocks/swin_layers.py:410-432` (once per image; the reference recomputes
                         them per micro-batch with identical input, guided_fusion_model.py:201)
    fusion               `estimator/models/patchfusion.py:259-340`, guided_fusion_model.py:163-207
    tiling / stitch      `estimator/models/baseline_pretrain.py:143-331`, estimator/models/utils.py:21-47

Nothing here touches torch for arithmetic on the path: torch allocates memory, owns the stream, and runs the
one-off load-time transforms (pos-embed bicubic resample, BatchNorm folding constants).  Workspace addresses are a
function of (weights, batch) only, so TMA tensor maps are cached and every stage call is CUDA-graph capturable.
"""
import ctypes as ct
import math

import torch
import torch.nn.functional as F

from . import lib, ops
from .ops import ACT_GELU, ACT_NONE, ACT_RELU, ACT_SOFTPLUS, call, pad_to, stream_ptr
from .params import FP8_LAYERS, VIT_FP8_LINEARS, WINDOW, branch_hparams, fusion_fp8_amax, fusion_precision, \
    guided_fusion_hparams, normed_attractors, vit_fp8_amax, vit_fp8_layers, vit_precision, DPT_FP8_CONVS, dpt_fp8_amax, \
    dpt_fp8_layers, dpt_precision, _get

BF16, F32 = torch.bfloat16, torch.float32


class Map:
    """NHWC bf16 activation: tensor [B,H,W,ld] + logical channel count."""
    __slots__ = ('t', 'C')

    def __init__(self, t, C):
        self.t, self.C = t, C

    @property
    def B(self):
        return self.t.shape[0]

    @property
    def hw(self):
        return self.t.shape[1], self.t.shape[2]

    def rows(self):
        return self.t.view(-1, self.t.shape[-1])


class Engine:
    def __init__(self, config, state_dict, device, parts=('coarse', 'fine', 'fusion')):
        """parts: the stages to pack and describe.  A single-branch model (BaselinePretrain) passes ('coarse',) or
        ('fine',) with a state dict holding only that branch; the fusion stage reads the coarse and fine hparams."""
        self.cfg = config
        self.parts = tuple(parts)
        self.dev = torch.device(device)
        self.P = tuple(_get(config, 'patch_process_shape'))
        branches = [b for b in ('coarse', 'fine') if b in self.parts or 'fusion' in self.parts]
        self.hp = {b: branch_hparams(_get(config, b + '_branch')) for b in branches}
        self.bcfg = {b: _get(config, b + '_branch') for b in branches}
        self.gf = guided_fusion_hparams(_get(config, 'guided_fusion'), self.P) if 'fusion' in self.parts else None
        self.bufs = {}
        self.arenas = {}
        self.generation = 0
        self._keep = []
        self.sd = {k: v.to(self.dev) for k, v in state_dict.items()}
        H, W = self.P
        assert H % 14 == 0 and W % 14 == 0
        self.gh, self.gw = H // 14, W // 14
        # vit_precision 'fp8_static': qkv, fc1 and fc2 of both encoders get e4m3 panels next to their bf16 ones
        # (calibration runs the bf16 encoder).  c_branch carries the calibrated input amax (set_vit_fp8_amax), c_branch_bf16
        # is the same stage without them.
        # dpt_precision 'fp8_static' does the same for the 19 DPT_FP8_CONVS of each decoder (set_dpt_fp8_amax); their
        # e4m3 panels are left out of c_branch_bf16, which runs them in bf16.
        self.vit_fp8_static = vit_precision(config) == 'fp8_static'
        self.dpt_fp8_static = dpt_precision(config) == 'fp8_static'
        self.W = {}
        self._pack_all()
        self.sd = None   # fp32 originals are no longer needed on the device
        # the branches this engine packs: both for PatchFusion, the built one for a single-branch model, whose config
        # (and calibration tables) name that branch only
        self.branches = tuple(b for b in ('coarse', 'fine') if b in self.parts)
        self.c_branch = {b: self._c_branch(b) for b in self.branches}
        self.c_branch_bf16 = dict(self.c_branch)
        self.vit_amax = None
        self.dpt_amax = None
        self._branch_amax = {}
        if self.vit_fp8_static:
            self.set_vit_fp8_amax(vit_fp8_amax(config, branches=self.branches))
        if self.dpt_fp8_static:
            self.set_dpt_fp8_amax(dpt_fp8_amax(config, branches=self.branches))
        self.c_fusion = self._c_fusion() if 'fusion' in self.parts else None
        # 'fp8_static': c_fusion carries the calibrated input amax of each FP8 conv (set_fp8_amax); c_fusion_tiles is the
        # same stage with per-tile scales, which calibration runs.  `calib` (a dict while PatchFusion.calibrate_fp8 runs)
        # collects each conv's input amax from the per-tile stage.
        self.c_fusion_tiles = self.c_fusion
        self.fp8_static = 'fusion' in self.parts and fusion_precision(config) == 'fp8_static'
        self.fp8_amax = None
        self.calib = None
        if self.fp8_static:
            self.set_fp8_amax(fusion_fp8_amax(config))

    # ------------------------------------------------------------------ buffers
    def buf(self, key, shape, dtype=BF16):
        k = (key, tuple(shape), dtype)
        t = self.bufs.get(k)
        if t is None:
            t = torch.zeros(shape, dtype=dtype, device=self.dev)
            self.bufs[k] = t
        return t

    def map(self, key, B, h, w, C):
        return Map(self.buf(key, (B, h, w, pad_to(C, 8))), C)

    # ------------------------------------------------------------------ weight packing
    def _w(self, k):
        return self.sd[k]

    def _dpt_conv(self, name, bias=True):
        """a DPT conv of DPT_FP8_CONVS: its e4m3 panel too under dpt_precision 'fp8_static'"""
        return self._conv(name, bias=bias, fp8='keep_bf16' if self.dpt_fp8_static else None)

    def _conv(self, name, src_c=None, bias=True, fp8=None):
        """fp8: None packs bf16; 'only' / 'keep_bf16' packs e4m3 (pack_weight_e4m3), the latter with the bf16 panel
        too (a conv that may read its input through the fused resample)."""
        b = self._w(name + '.bias') if bias and (name + '.bias') in self.sd else None
        if fp8:
            return ops.pack_weight_e4m3(self._w(name + '.weight'), b, src_c=src_c, keep_bf16=fp8 == 'keep_bf16')
        return ops.pack_weight(self._w(name + '.weight'), b, src_c=src_c)

    def _conv_bn(self, conv, bn, fp8=None):
        g, b = self._w(bn + '.weight'), self._w(bn + '.bias')
        m, v = self._w(bn + '.running_mean'), self._w(bn + '.running_var')
        scale = g / torch.sqrt(v + 1e-5)
        if fp8:
            return ops.pack_weight_e4m3(self._w(conv + '.weight'), None, scale=scale, shift=b - m * scale)
        return ops.pack_weight(self._w(conv + '.weight'), None, scale=scale, shift=b - m * scale)

    def _f32(self, k):
        return self._w(k).float().contiguous()

    def _pack_head(self, pre, C, hp, drop_rel):
        Wd = {}
        for n in ['seed_bin_regressor', 'seed_projector'] + ['projectors.%d' % i for i in range(4)] + \
                 ['attractors.%d' % i for i in range(4)]:
            Wd[n + '.0'] = self._conv(pre + n + '._net.0')
            w2, b2 = self._w(pre + n + '._net.2.weight'), self._w(pre + n + '._net.2.bias')
            if n.startswith('attractors') and normed_attractors(hp['bin_centers_type']):
                # AttractorLayer reads only the even channels of its 2 nA outputs (attractor.py:104-106)
                w2, b2 = w2[0::2].contiguous(), b2[0::2].contiguous()
            Wd[n + '.2'] = ops.pack_weight(w2, b2)
            if w2.shape[0] <= 16:       # narrow second layer: fused into the first layer's epilogue (fp32 weights)
                Wd[n + '.tail'] = (w2.reshape(w2.shape[0], -1).float().contiguous(), b2.float().contiguous())
        w0 = self._w(pre + 'conditional_log_binomial.mlp.0.weight')
        b0 = self._w(pre + 'conditional_log_binomial.mlp.0.bias')
        E = hp['bin_embedding_dim']
        if drop_rel:      # rel_cond is identically zero in the fusion head (patchfusion.py:300,326-328)
            w0 = torch.cat([w0[:, :32], w0[:, 33:]], 1).contiguous()
            Wd['clb.0'] = ops.pack_weight(w0, b0, src_c=[32, E])
        else:
            Wd['clb.0'] = ops.pack_weight(w0, b0, src_c=[32, 1, E])
        Wd['clb.tail'] = (self._w(pre + 'conditional_log_binomial.mlp.2.weight').reshape(4, -1).float().contiguous(),
                          self._f32(pre + 'conditional_log_binomial.mlp.2.bias'))
        return Wd

    def _pack_branch(self, which):
        pre = which + '_branch.'
        hp = self.hp[which]
        D, C, oc = hp['dim'], hp['features'], hp['out_channels']
        vit = pre + 'core.core.pretrained.'
        Wd = {}
        Wd['patch'] = ops.pack_weight(self._w(vit + 'patch_embed.proj.weight').reshape(D, 588),
                                      self._w(vit + 'patch_embed.proj.bias'))
        # pos-embed resample is input-shape-only: done once here with the reference's exact call
        # (vision_transformer.py:189-210: bicubic, scale_factor=((gh+0.1)/37, (gw+0.1)/37), no antialias)
        pe = self._w(vit + 'pos_embed').float()
        n = pe.shape[1] - 1
        s = int(math.sqrt(n))
        if (self.gh, self.gw) != (s, s):
            grid = pe[:, 1:].reshape(1, s, s, D).permute(0, 3, 1, 2)
            grid = F.interpolate(grid, scale_factor=((self.gh + 0.1) / s, (self.gw + 0.1) / s), mode='bicubic',
                                 antialias=False)
            assert grid.shape[-2:] == (self.gh, self.gw)
            pe = torch.cat([pe[:, :1], grid.permute(0, 2, 3, 1).reshape(1, self.gh * self.gw, D)], 1)
        Wd['pos'] = pe[0].contiguous()
        Wd['cls'] = self._f32(vit + 'cls_token').reshape(D)

        def lin(name):      # qkv / fc1 / fc2: e4m3 panels too under vit_precision 'fp8_static'
            w, b = self._w(name + '.weight'), self._w(name + '.bias')
            if self.vit_fp8_static:
                return ops.pack_weight_e4m3(w, b, keep_bf16=True)
            return ops.pack_weight(w, b)
        for i in range(hp['depth']):
            p = vit + 'blocks.%d.' % i
            Wd['b%d' % i] = dict(
                n1w=self._f32(p + 'norm1.weight'), n1b=self._f32(p + 'norm1.bias'),
                n2w=self._f32(p + 'norm2.weight'), n2b=self._f32(p + 'norm2.bias'),
                qkv=lin(p + 'attn.qkv'), proj=ops.pack_weight(self._w(p + 'attn.proj.weight'), self._w(p + 'attn.proj.bias')),
                fc1=lin(p + 'mlp.fc1'), fc2=lin(p + 'mlp.fc2'),
                ls1=self._f32(p + 'ls1.gamma'), ls2=self._f32(p + 'ls2.gamma'))
        Wd['nw'], Wd['nb'] = self._f32(vit + 'norm.weight'), self._f32(vit + 'norm.bias')
        dh = pre + 'core.core.depth_head.'
        for i in range(4):
            Wd['proj%d' % i] = self._conv(dh + 'projects.%d' % i)
        Wd['rs0'] = ops.pack_weight_convT(self._w(dh + 'resize_layers.0.weight'), self._w(dh + 'resize_layers.0.bias'), 4)
        Wd['rs1'] = ops.pack_weight_convT(self._w(dh + 'resize_layers.1.weight'), self._w(dh + 'resize_layers.1.bias'), 2)
        rs3 = self._conv(dh + 'resize_layers.3')
        assert oc[3] % 64 == 0
        rs3.taps, rs3.src_c = 1, [9 * oc[3]]          # consumed as a plain GEMM over pf_im2col_3x3_s2 rows
        Wd['rs3'] = rs3
        for i in range(4):
            Wd['rn%d' % i] = self._dpt_conv(dh + 'scratch.layer%d_rn' % (i + 1), bias=False)
        for i in range(1, 5):
            r = dh + 'scratch.refinenet%d.' % i
            Wd['ff%d.out' % i] = self._conv(r + 'out_conv')
            for u in (1, 2):
                # refinenet4's resConfUnit1 never runs (its FeatureFusionBlock has no second input): bf16 only
                conv = self._conv if (i, u) == (4, 1) else self._dpt_conv
                Wd['ff%d.u%d.c1' % (i, u)] = conv(r + 'resConfUnit%d.conv1' % u)
                Wd['ff%d.u%d.c2' % (i, u)] = conv(r + 'resConfUnit%d.conv2' % u)
        Wd['oc1'] = self._dpt_conv(dh + 'scratch.output_conv1')
        Wd['oc2.0'] = self._conv(dh + 'scratch.output_conv2.0')
        Wd['oc2.tail'] = (self._w(dh + 'scratch.output_conv2.2.weight').reshape(1, -1).float().contiguous(),
                          self._f32(dh + 'scratch.output_conv2.2.bias'))
        Wd['conv2'] = self._conv(pre + 'conv2')
        Wd['head'] = self._pack_head(pre, C, hp, drop_rel=False)
        return Wd

    def _pack_fusion(self):
        hp = self.hp['fine']
        C = hp['features']
        Wd = {}
        # fusion_precision 'fp8' / 'fp8_static': the U-Net's 3x3 convs get e4m3 panels; the convs whose input can come through the
        # fused resample (up*.0, cv*.0) keep their bf16 panel for that path too.  fusion_conv_list, G2L and the head
        # stay bf16.
        f8 = 'only' if fusion_precision(self.cfg) in ('fp8', 'fp8_static') else None
        f8rs = 'keep_bf16' if f8 else None
        for i in range(5):      # level 5's fused map is dead in the U-Net (guided_fusion_model.py:198)
            Wd['fc%d' % i] = self._conv('fusion_conv_list.%d' % i, src_c=[C, C])
        g = 'guided_fusion.'
        ic = self.gf['in_channels']
        Wd['inc.0'] = self._conv_bn(g + 'inc.double_conv.0', g + 'inc.double_conv.1', fp8=f8)
        Wd['inc.1'] = self._conv_bn(g + 'inc.double_conv.3', g + 'inc.double_conv.4', fp8=f8)
        for i in range(5):
            p = g + 'down_conv_list.%d.maxpool_conv.1.double_conv.' % i
            Wd['down%d.0' % i] = self._conv_bn(p + '0', p + '1', fp8=f8)
            Wd['down%d.1' % i] = self._conv_bn(p + '3', p + '4', fp8=f8)
        inv = ic[::-1]
        for i in range(1, 6):
            p = g + 'up_conv_list.%d.conv.double_conv.' % (i - 1)
            Wd['up%d.0' % i] = self._conv(p + '0', src_c=[inv[i], inv[i - 1], inv[i - 1]], fp8=f8rs)
            Wd['up%d.1' % i] = self._conv(p + '2', fp8=f8)
        depth, heads = self.gf['depth'][::-1], self.gf['num_heads'][::-1]
        for i in range(6):
            c, p = inv[i], g + 'g2l_list.%d.' % i
            L = dict(ape=self._f32(p + 'absolute_pos_embed').reshape(-1, c), C=c, heads=heads[i],
                     nw=self._f32(p + 'g2l_layer_norm.weight'), nb=self._f32(p + 'g2l_layer_norm.bias'),
                     ones=torch.ones(c, dtype=F32, device=self.dev), blocks=[])
            for b in range(depth[i]):
                q = p + 'g2l_layer.blocks.%d.' % b
                L['blocks'].append(dict(
                    n1w=self._f32(q + 'norm1.weight'), n1b=self._f32(q + 'norm1.bias'),
                    n2w=self._f32(q + 'norm2.weight'), n2b=self._f32(q + 'norm2.bias'),
                    table=self._f32(q + 'attn.relative_position_bias_table'),
                    qkv=ops.pack_weight(self._w(q + 'attn.qkv.weight'), self._w(q + 'attn.qkv.bias')),
                    proj=ops.pack_weight(self._w(q + 'attn.proj.weight'), self._w(q + 'attn.proj.bias')),
                    fc1=ops.pack_weight(self._w(q + 'mlp.fc1.weight'), self._w(q + 'mlp.fc1.bias')),
                    fc2=ops.pack_weight(self._w(q + 'mlp.fc2.weight'), self._w(q + 'mlp.fc2.bias'))))
            Wd['g2l%d' % i] = L
            p = g + 'convs.%d.double_conv.' % i
            Wd['cv%d.0' % i] = self._conv(p + '0', src_c=[c, c], fp8=f8rs)
            Wd['cv%d.1' % i] = self._conv(p + '2', fp8=f8)
        Wd['head'] = self._pack_head('', C, self.hp['coarse'], drop_rel=True)
        return Wd

    def _pack_all(self):
        for b in ('coarse', 'fine'):
            if b in self.parts:
                self.W[b] = self._pack_branch(b)
        if 'fusion' in self.parts:
            self.W['fusion'] = self._pack_fusion()
        torch.cuda.synchronize(self.dev)

    # ------------------------------------------------------------------ C structs for the stage-level ABI
    def _c_head(self, Wh, hp, bcfg, has_rel, depth_cfg):
        """depth_cfg: where the head's min_depth / max_depth come from: the branch config for a branch head, the
        top-level config for the fusion head (patchfusion.py:149-164)."""
        from . import stage
        H = stage.PfHead()

        def L(name):
            return stage.layer(Wh[name], Wh.get(name[:-2] + '.tail') if name.endswith('.0') else None)

        H.seed0, H.seed2 = L('seed_bin_regressor.0'), L('seed_bin_regressor.2')
        H.seedproj0, H.seedproj2 = L('seed_projector.0'), L('seed_projector.2')
        for i in range(4):
            H.proj0[i], H.proj2[i] = L('projectors.%d.0' % i), L('projectors.%d.2' % i)
            H.att0[i], H.att2[i] = L('attractors.%d.0' % i), L('attractors.%d.2' % i)
            H.n_attractors[i] = hp['n_attractors'][i]
        H.clb0 = stage.layer(Wh['clb.0'], Wh['clb.tail'])
        H.n_bins, H.bin_embedding_dim = hp['n_bins'], hp['bin_embedding_dim']
        H.attractor_flags = (1 if hp['attractor_kind'] == 'mean' else 0) | (2 if hp['attractor_type'] == 'exp' else 0)
        H.has_rel = 1 if has_rel else 0
        H.min_temp, H.max_temp = float(_get(bcfg, 'min_temp')), float(_get(bcfg, 'max_temp'))
        H.bin_centers_type = lib.BINS_TYPES[hp['bin_centers_type']]
        # ZoeDepth's constructor defaults (zoedepth_v1.py:40)
        H.min_depth, H.max_depth = float(_get(depth_cfg, 'min_depth', 1e-3)), float(_get(depth_cfg, 'max_depth', 10))
        return H

    def _c_branch(self, which, amax=None, dpt_amax=None):
        """amax: {'<i>.<qkv|fc1|fc2>': address of its fp32 input amax} of a calibrated 'fp8_static' encoder, or None;
        dpt_amax: {conv of DPT_FP8_CONVS: address of its fp32 input amax} of a calibrated 'fp8_static' decoder, or None
        (the decoder then runs in bf16: its e4m3 panels are not passed)"""
        from . import stage
        Wd, hp = self.W[which], self.hp[which]
        B = stage.PfBranch()
        B.H, B.W = self.P
        B.dim, B.depth, B.heads, B.features = hp['dim'], hp['depth'], hp['heads'], hp['features']
        for i in range(4):
            B.out_channels[i] = hp['out_channels'][i]
        B.patch = stage.layer(Wd['patch'])
        B.pos, B.cls = Wd['pos'].data_ptr(), Wd['cls'].data_ptr()
        blocks = (stage.PfVitBlock * hp['depth'])()
        for i in range(hp['depth']):
            bw, cb = Wd['b%d' % i], blocks[i]
            for k in ('n1w', 'n1b', 'n2w', 'n2b', 'ls1', 'ls2'):
                setattr(cb, k, bw[k].data_ptr())
            for k in ('qkv', 'proj', 'fc1', 'fc2'):
                setattr(cb, k, stage.layer(bw[k]))
            if amax is not None:
                for k in VIT_FP8_LINEARS:
                    getattr(cb, k).a_amax = amax['%d.%s' % (i, k)]
        self._keep.append(blocks)
        B.blocks = blocks
        B.nw, B.nb = Wd['nw'].data_ptr(), Wd['nb'].data_ptr()
        for i in range(4):
            B.proj[i] = stage.layer(Wd['proj%d' % i])
            B.rn[i] = stage.layer(Wd['rn%d' % i])
            B.ff_out[i] = stage.layer(Wd['ff%d.out' % (i + 1)])
            for u in (1, 2):
                B.ff_c1[i][u - 1] = stage.layer(Wd['ff%d.u%d.c1' % (i + 1, u)])
                B.ff_c2[i][u - 1] = stage.layer(Wd['ff%d.u%d.c2' % (i + 1, u)])
        B.rs0, B.rs1, B.rs3 = stage.layer(Wd['rs0']), stage.layer(Wd['rs1']), stage.layer(Wd['rs3'])
        B.oc1 = stage.layer(Wd['oc1'])
        dpt = [B.rn[i] for i in range(4)] + [B.ff_c1[i][u] for i in range(3) for u in (0, 1)] + \
            [B.ff_c2[i][u] for i in range(3) for u in (0, 1)] + [B.ff_c1[3][1], B.ff_c2[3][1], B.oc1]
        names = ['layer%d_rn' % i for i in range(1, 5)] + \
            ['refinenet%d.resConfUnit%d.conv1' % (i, u) for i in (1, 2, 3) for u in (1, 2)] + \
            ['refinenet%d.resConfUnit%d.conv2' % (i, u) for i in (1, 2, 3) for u in (1, 2)] + \
            ['refinenet4.resConfUnit2.conv1', 'refinenet4.resConfUnit2.conv2', 'output_conv1']
        assert sorted(names) == sorted(DPT_FP8_CONVS)
        for L, n in zip(dpt, names):
            if dpt_amax is None:
                L.w8, L.w_scale = None, None
            else:
                L.a_amax = dpt_amax[n]
        B.oc2 = stage.layer(Wd['oc2.0'], Wd['oc2.tail'])
        B.conv2 = stage.layer(Wd['conv2'])
        B.head = self._c_head(Wd['head'], hp, self.bcfg[which], True, self.bcfg[which])
        return B

    def set_fp8_amax(self, table):
        """'fp8_static': the calibrated input amax of the 34 FP8 convs ({name: float}, validated) that the stage runs
        with, or None (no table: the fusion stage refuses to run, calibration still can).  The values are read when a
        stage is issued, so graphs captured before a change must be dropped (PatchFusion.engine does)."""
        if table is None:
            self.fp8_amax, self.c_fusion = None, self.c_fusion_tiles
            return
        table = dict(table)
        arr = (ct.c_float * len(FP8_LAYERS))(*[table[k] for k in FP8_LAYERS])
        self._keep.append(arr)
        self.c_fusion = self._c_fusion({k: ct.addressof(arr) + 4 * i for i, k in enumerate(FP8_LAYERS)})
        self.fp8_amax = table

    def set_vit_fp8_amax(self, table):
        """vit_precision 'fp8_static': the calibrated input amax of the encoders' qkv / fc1 / fc2 ({name of
        vit_fp8_layers: float}, validated), or None (no table: the branches refuse to run, calibration still can).  Read
        when a stage is issued, so graphs captured before a change must be dropped (PatchFusion.engine does)."""
        if table is None:
            self.vit_amax, self.c_branch = None, dict(self.c_branch_bf16)
            return
        self.vit_amax = dict(table)
        self._set_branch_amax(vit_fp8_layers(self.cfg, self.branches), self.vit_amax, 'vit')

    def set_dpt_fp8_amax(self, table):
        """dpt_precision 'fp8_static': the calibrated input amax of the decoders' DPT_FP8_CONVS ({name of
        dpt_fp8_layers: float}, validated), or None (no table: the branches refuse to run, calibration still can).  Read
        when a stage is issued, so graphs captured before a change must be dropped (PatchFusion.engine does)."""
        self.dpt_amax = dict(table) if table is not None else None
        self._set_branch_amax(dpt_fp8_layers(self.cfg, self.branches), self.dpt_amax, 'dpt')

    def _set_branch_amax(self, names, table, kind):
        """re-points c_branch at the current ViT and DPT tables (kind: which of them `table` is)"""
        if table is None:
            self._branch_amax.pop(kind, None)
        else:
            arr = (ct.c_float * len(names))(*[table[k] for k in names])
            self._keep.append(arr)
            self._branch_amax[kind] = {k: ct.addressof(arr) + 4 * i for i, k in enumerate(names)}

        def per_branch(kind, b):
            addr = self._branch_amax.get(kind)
            return None if addr is None else {k[len(b) + 1:]: a for k, a in addr.items() if k.startswith(b + '.')}
        self.c_branch = {b: self._c_branch(b, per_branch('vit', b), per_branch('dpt', b)) for b in self.c_branch_bf16}

    def _branch_struct(self, which):
        if self.calib is not None:
            return self.c_branch_bf16[which]
        if self.vit_fp8_static and self.vit_amax is None:
            raise RuntimeError("vit_precision 'fp8_static' needs the calibrated input scales `vit_fp8_amax`: run "
                               "PatchFusion.calibrate_fp8 (or tools/calibrate_fp8.py) first")
        if self.dpt_fp8_static and self.dpt_amax is None:
            raise RuntimeError("dpt_precision 'fp8_static' needs the calibrated input scales `dpt_fp8_amax`: run "
                               "PatchFusion.calibrate_fp8 (or tools/calibrate_fp8.py) first")
        return self.c_branch[which]

    def _fusion_struct(self):
        if self.calib is not None:
            return self.c_fusion_tiles
        if self.fp8_static and self.fp8_amax is None:
            raise RuntimeError("fusion_precision 'fp8_static' needs the calibrated input scales `fusion_fp8_amax`: run "
                               "PatchFusion.calibrate_fp8 (or tools/calibrate_fp8.py) first")
        return self.c_fusion

    def _c_fusion(self, amax=None):
        """amax: {FP8 layer name: address of its fp32 amax} of a calibrated 'fp8_static' stage, or None"""
        from . import stage
        Wf = self.W['fusion']
        F_ = stage.PfFusion()
        F_.H, F_.W = self.P
        for i in range(5):
            F_.fc[i] = stage.layer(Wf['fc%d' % i])
            F_.down[i][0], F_.down[i][1] = stage.layer(Wf['down%d.0' % i]), stage.layer(Wf['down%d.1' % i])
            F_.up[i][0], F_.up[i][1] = stage.layer(Wf['up%d.0' % (i + 1)]), stage.layer(Wf['up%d.1' % (i + 1)])
        F_.inc[0], F_.inc[1] = stage.layer(Wf['inc.0']), stage.layer(Wf['inc.1'])
        for i in range(6):
            F_.cv[i][0], F_.cv[i][1] = stage.layer(Wf['cv%d.0' % i]), stage.layer(Wf['cv%d.1' % i])
            L, g = Wf['g2l%d' % i], F_.g2l[i]
            g.C, g.heads, g.depth = L['C'], L['heads'], len(L['blocks'])
            g.ape, g.ape_rows = L['ape'].data_ptr(), L['ape'].shape[0]
            g.nw, g.nb, g.ones = L['nw'].data_ptr(), L['nb'].data_ptr(), L['ones'].data_ptr()
            blocks = (stage.PfG2LBlock * len(L['blocks']))()
            for b, bw in enumerate(L['blocks']):
                for k in ('n1w', 'n1b', 'n2w', 'n2b', 'table'):
                    setattr(blocks[b], k, bw[k].data_ptr())
                for k in ('qkv', 'proj', 'fc1', 'fc2'):
                    setattr(blocks[b], k, stage.layer(bw[k]))
            self._keep.append(blocks)
            g.blocks = blocks
        F_.head = self._c_head(Wf['head'], self.hp['coarse'], self.bcfg['coarse'], False, self.cfg)
        if amax is not None:
            for i in range(5):
                F_.down[i][0].a_amax, F_.down[i][1].a_amax = amax['down%d.0' % i], amax['down%d.1' % i]
                F_.up[i][0].a_amax, F_.up[i][1].a_amax = amax['up%d.0' % (i + 1)], amax['up%d.1' % (i + 1)]
            F_.inc[0].a_amax, F_.inc[1].a_amax = amax['inc.0'], amax['inc.1']
            for i in range(6):
                F_.cv[i][0].a_amax, F_.cv[i][1].a_amax = amax['cv%d.0' % i], amax['cv%d.1' % i]
        return F_

    # ------------------------------------------------------------------ workspaces (one arena per stage role)
    def arena(self, name, nbytes):
        """Persistent uint8 workspace `name` of at least nbytes (grown once to the largest request; growing bumps
        `generation`, which invalidates graphs captured over the old addresses)."""
        t = self.arenas.get(name)
        if t is None or t.numel() < nbytes:
            self.arenas[name] = t = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=self.dev)
            self.generation += 1
        return t

    @staticmethod
    def _view(arena, ptr, shape, dtype):
        off = ptr - arena.data_ptr()
        n = 1
        for s_ in shape:
            n *= s_
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        assert 0 <= off and off + nbytes <= arena.numel()
        return arena[off:off + nbytes].view(dtype).view(shape)

    def _maps(self, arena, pf_maps):
        return [Map(self._view(arena, m.ptr, (m.B, m.H, m.W, m.ld), BF16), m.C) for m in pf_maps]

    def _tap_cb(self, arena, taps, inputs=()):
        """inputs: the Maps of the call's inputs outside `arena` that a layer tap may name (a conv's source)"""
        spans = [arena] + [m.t.reshape(-1).view(torch.uint8) for m in inputs]

        def cb(user, name, ptr, is_f32, rows, cols, ld):
            # is_f32: 0 bf16, 1 fp32, 2 e4m3 bytes (the static FP8 convs' operand maps)
            if name.startswith(b'amaxv.') or name.startswith(b'amaxd.'):
                return      # the bf16 branch's calibration inputs (_calib_vit_cb): not kept
            span = next(s_ for s_ in spans if 0 <= ptr - s_.data_ptr() < s_.numel())
            t = self._view(span, ptr, (rows, ld), (BF16, F32, torch.uint8)[is_f32])
            taps[name.decode()] = t[:, :cols].clone()
        return cb

    def _calib_cb(self, arena):
        """calibration: fold each FP8 conv's per-tile partial maxima (tap "amax.<layer>") into calib[layer], on the
        device and NaN-propagating"""
        def cb(user, name, ptr, is_f32, rows, cols, ld):
            name = name.decode()
            if not name.startswith('amax.'):
                return
            m = self._view(arena, ptr, (rows, ld), F32)[:, :cols].amax()
            k = name[5:]
            self.calib[k] = m if k not in self.calib else torch.maximum(self.calib[k], m)
        return cb

    def _calib_vit_cb(self, arena, which):
        """calibration of the 'fp8_static' encoders and decoders: fold the amax of each E4M3 linear's / DPT conv's bf16
        input (tap "amaxv.<i>.<lin>" / "amaxd.<conv>" of the bf16 stage) into calib['<which>.<i>.<lin>'] /
        calib['<which>.<conv>'], NaN-propagating, on the stream the branch is issued on (the current stream, as the
        launches)"""
        prefixes = tuple(p for p, on in (('amaxv.', self.vit_fp8_static), ('amaxd.', self.dpt_fp8_static)) if on)

        def cb(user, name, ptr, is_f32, rows, cols, ld):
            name = name.decode()
            if not name.startswith(prefixes):
                return
            lo, hi = torch.aminmax(self._view(arena, ptr, (rows, ld), BF16)[:, :cols])
            m = torch.maximum(-lo, hi).float()
            k = '%s.%s' % (which, name[6:])
            self.calib[k] = m if k not in self.calib else torch.maximum(self.calib[k], m)
        return cb

    # ------------------------------------------------------------------ stages (sequenced inside libpf_b200)
    def branch(self, which, images, taps=None, ws=None):
        """images: planar fp32 [B,3,H,W] in [0,1] (un-normalised).  Returns (depth fp32 [B,H,W], feats[6] Maps
        low->high: x_d0, r4, r3, r2, r1, out_conv) - views into the stage's workspace (`ws`: (arena, byte offset) to
        place it; default = the branch's own arena)."""
        from . import stage
        cb = self._branch_struct(which)
        B = images.shape[0]
        need = stage.branch_workspace_bytes(cb, B)
        if ws is None:
            arena, off = self.arena(which, need), 0
        else:
            arena, off = ws
        assert images.dtype == F32 and images.is_contiguous() and off % 256 == 0 and off + need <= arena.numel()
        tap = self._tap_cb(arena, taps) if taps is not None else None
        if tap is None and self.calib is not None and (self.vit_fp8_static or self.dpt_fp8_static):
            tap = self._calib_vit_cb(arena, which)
        out = stage.branch_forward(cb, images, B, arena.data_ptr() + off, need, tap)
        H, W = self.P
        depth = self._view(arena, out.depth, (B, H, W), F32)
        feats = self._maps(arena, out.feats)
        if taps is not None:
            taps['rel'] = taps['rel'].view(B, H, W)
            for k_ in list(taps):
                if k_[0] == 'b' and k_[1:].isdigit():
                    m = feats[1 + int(k_[1:])]
                    taps[k_] = taps[k_].view(B, m.hw[0], m.hw[1], -1)
                elif k_ in ('seed', 'centers'):         # x_d0's grid / the last attractor's (feats[4] = r1)
                    m = feats[0 if k_ == 'seed' else 4]
                    taps[k_] = taps[k_].view(B, m.hw[0], m.hw[1], -1)
        return depth, feats

    def branch_bytes(self, which, B):
        from . import stage
        return stage.branch_workspace_bytes(self._branch_struct(which), B)

    @staticmethod
    def _pf_maps(maps):
        from . import stage
        arr = (stage.PfMap * len(maps))()
        for i, m in enumerate(maps):
            arr[i].ptr, arr[i].C, arr[i].ld = m.t.data_ptr(), m.C, m.t.shape[-1]
            arr[i].B, arr[i].H, arr[i].W = m.t.shape[0], m.t.shape[1], m.t.shape[2]
        return arr

    def g2l(self, coarse_feats, taps=None):
        """The six tile-invariant G2L maps of the whole-image coarse taps (computed once per image).  The maps may hold
        a batch of B images: one call then computes the B images' maps, batch B out."""
        from . import stage
        cm = self._pf_maps(coarse_feats)
        need = stage.g2l_workspace_bytes(self.c_fusion, cm)
        arena = self.arena('g2l', need)
        tap = self._tap_cb(arena, taps) if taps is not None else None
        out = stage.g2l_forward(self.c_fusion, cm, arena.data_ptr(), need, tap)
        return self._maps(arena, out)

    def fusion_bytes(self, T, g2l_maps):
        from . import stage
        return stage.fusion_workspace_bytes(self._fusion_struct(), T, self._pf_maps(g2l_maps))

    def fusion(self, crops, boxes, fine_depth, fine_feats, coarse_depth, coarse_feats, g2l_maps, taps=None,
               depth_out=None, ws=None, tile_image=None):
        """crops planar fp32 [T,3,H,W]; boxes fp32 [T,4] (device, patch_process units); returns fp32 [T,H,W].
        tile_image (int32 [T] device tensor): tile t reads image tile_image[t] of the batch-B coarse depth [B,H,W],
        coarse maps and G2L maps; None reads image 0 (the single-image call)."""
        from . import stage
        T = crops.shape[0]
        H, W = self.P
        gm = self._pf_maps(g2l_maps)
        cfu = self._fusion_struct()
        need = stage.fusion_workspace_bytes(cfu, T, gm)
        if ws is None:
            arena, off = self.arena('fusion', need), 0
        else:
            arena, off = ws
        assert off % 256 == 0 and off + need <= arena.numel()
        if depth_out is None:
            depth_out = self.buf('fus.depth', (T, H, W), F32)
        assert depth_out.dtype == F32 and depth_out.is_contiguous() and tuple(depth_out.shape) == (T, H, W)
        for t_ in (crops, boxes, fine_depth, coarse_depth):
            assert t_.dtype == F32 and t_.is_contiguous()
        if tile_image is not None:
            assert tile_image.dtype == torch.int32 and tile_image.is_contiguous() and tile_image.numel() == T
        tap = self._tap_cb(arena, taps, fine_feats) if taps is not None else None
        if tap is None and self.calib is not None:
            tap = self._calib_cb(arena)
        stage.fusion_forward(cfu, crops, boxes, T, fine_depth, self._pf_maps(fine_feats), coarse_depth,
                             self._pf_maps(coarse_feats), gm, arena.data_ptr() + off, need, depth_out, tap,
                             tile_image=tile_image)
        if taps is not None:
            for i in range(6):
                m = g2l_maps[i]
                taps['fuse%d' % i] = taps['fuse%d' % i].view(T, m.hw[0], m.hw[1], -1)
        return depth_out
