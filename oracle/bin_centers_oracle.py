"""The metric-bins head for every `bin_centers_type` (ZD:90-105): SeedBinRegressor / AttractorLayer for 'normed',
'hybrid1', 'hybrid2' next to pf_oracle's softplus head.  `typed_heads(cfg)` runs pf_oracle's branch / fusion forwards
(and everything built on them) with this head.

  LB  external/zoedepth/models/layers/localbins_layers.py     ATT  external/zoedepth/models/layers/attractor.py
  ZD  external/zoedepth/models/zoedepth/zoedepth_v1.py         PF   estimator/models/patchfusion.py
"""
import contextlib

import torch
import torch.nn.functional as F

from oracle import pf_oracle as po


def seed_bins(S, min_depth, max_depth, normed_seed=True, to_unit=False):
    """The seed's bin centres from its `_net` output S (B,nbins,h,w).  normed_seed: SeedBinRegressor (LB:51-67): S is
    the ReLU output, widths (max - min) (S + 1e-3) / sum, edges the cumsum after a min_depth pad, centres the edge
    midpoints; else SeedBinRegressorUnnormed (LB:98-103): the softplus output is the centres.  to_unit: the b_prev the
    normed attractors take, (centres - min) / (max - min) (ZD:176-181, PF:301-306)."""
    c = S
    if normed_seed:
        Bw = S + 1e-3
        Bw = (max_depth - min_depth) * (Bw / Bw.sum(dim=1, keepdim=True))
        edges = torch.cumsum(F.pad(Bw, (0, 0, 0, 0, 1, 0), mode='constant', value=min_depth), dim=1)
        c = 0.5 * (edges[:, :-1] + edges[:, 1:])
    return (c - min_depth) / (max_depth - min_depth) if to_unit else c


def attractor_update_normed(A2, b_prev, min_depth, max_depth, kind='sum', attractor_type='exp'):
    """One AttractorLayer step after its MLP (ATT:100-135): A2 (B,2nA,h,w) the ReLU output.  Only the even channels,
    plus 1e-3, are the attractor points (A_normed is computed and then overwritten, ATT:105-106).  Returns the
    normalised, unsorted b_new and the metric centres sort((max - min) b_new + min) clipped to [min, max]."""
    b_new = po.attractor_update((A2 + 1e-3)[:, 0::2], b_prev, kind, attractor_type)
    Bc = torch.sort((max_depth - min_depth) * b_new + min_depth, dim=1).values
    return b_new, torch.clip(Bc, min_depth, max_depth)


def metric_head(w, x, x_blocks, last, rel_cond, hp, taps=None, depth_range=None):
    """pf_oracle.metric_head for hp['bin_centers_type'].  depth_range (min, max): the head's (default hp's own, as in a
    branch; the fusion head's is the top-level config's, PF:149-164).  Taps: 'seed', 'b0'..'b3', and 'centers' (the
    last level's sorted metric centres) for the AttractorLayer types."""
    typ = po._get(hp, 'bin_centers_type', 'softplus')
    lo, hi = depth_range or (po._get(hp, 'min_depth', 1e-3), po._get(hp, 'max_depth', 10))
    normed_seed, normed_att = typ in ('normed', 'hybrid1'), typ in ('normed', 'hybrid2')
    kind, atype = po._get(hp, 'attractor_kind', 'sum'), po._get(hp, 'attractor_type', 'exp')
    S = po._mlp2(w.sub('seed_bin_regressor.'), x, F.relu if normed_seed else F.softplus)
    b_prev = S if typ == 'softplus' else seed_bins(S, lo, hi, normed_seed, normed_att)
    taps = {} if taps is None else taps
    taps['seed'] = b_prev
    prev_emb = po._mlp2(w.sub('seed_projector.'), x)
    for i, xb in enumerate(x_blocks):
        emb = po._mlp2(w.sub('projectors.%d.' % i), xb)
        A = po._mlp2(w.sub('attractors.%d.' % i), emb + po.up(prev_emb, xb.shape[-2:]),
                     F.relu if normed_att else F.softplus)
        if normed_att:
            b_prev, taps['centers'] = attractor_update_normed(A, b_prev, lo, hi, kind, atype)
        else:
            b_prev = po.attractor_update(A, b_prev, kind, atype)
        prev_emb, taps['b%d' % i] = emb, b_prev
    size = last.shape[-2:]
    z = torch.cat([last, po.up(rel_cond, size), po.up(prev_emb, size)], dim=1)
    c = w.sub('conditional_log_binomial.')
    pt = F.softplus(c.conv('mlp.2', F.gelu(c.conv('mlp.0', z))))
    # only the last level's centres reach the expectation: sorted metric ones for AttractorLayer (ZD:217-219)
    bc = taps['centers'] if normed_att else b_prev
    return po.log_binomial_depth(pt, bc, po._get(hp, 'min_temp'), po._get(hp, 'max_temp'))


@contextlib.contextmanager
def typed_heads(cfg):
    """Inside the block pf_oracle's forwards use `metric_head`: each branch head its own type and range, the fusion
    head (the only one over un-prefixed weights, PF:297-339) the coarse type and cfg's top-level range."""
    real = po.metric_head

    def head(w, x, x_blocks, last, rel_cond, hp, taps=None):
        rng = (po._get(cfg, 'min_depth'), po._get(cfg, 'max_depth')) if w.prefix == '' else None
        return metric_head(w, x, x_blocks, last, rel_cond, hp, taps, rng)
    po.metric_head = head
    try:
        yield
    finally:
        po.metric_head = real
