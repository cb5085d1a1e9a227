"""References and input cases shared by the pf_attention tests (test_gpu_attn_parity.py on the GPU,
test_attn_reference.py on the CPU).

Two references, both plain torch on the bf16-rounded q / k / v the kernel consumes:
  attention_fp64      softmax(q k^T scale) v in fp64.
  attention_emulated  pf_attention_kernel's algorithm step by step: 128-key blocks zero-padded past `seq` (what TMA
                      fills) and masked to -inf, the fp32 online softmax in the exp2 domain, P rounded to bf16 before
                      P V, O and l rescaled when the row maximum moves, bf16(O * (1 / l)).  `bug` plants one of the
                      mistakes the suite must catch (PLANTED_BUGS).

The case constructors return fp32 q, k, v of shape [B, seq, heads, 64] and the softmax scale.  They take a torch
Generator, so the GPU tests and the CPU guard build the same kinds of inputs.
"""
import math

import torch

HD = 64
KEY_BLOCK = 128
LOG2E = 1.4426950408889634

# Global relative L-inf of the kernel against attention_fp64.  The emulation stays within 2-4e-3 (bf16 P and output);
# 8e-3 leaves 2x for summation order, and every planted bug lands at least 4x above it (test_attn_reference.py).
FP64_TOL = 8e-3

PLANTED_BUGS = (
    'mask_off_by_one',    # `key > kv_left` instead of `key >= kv_left`: one zero-filled key (logit 0, V = 0) leaks in
    'no_o_rescale',       # O is not multiplied by c when the running maximum moves
    'l_counts_masked',    # the row sum l also counts the masked (zero-filled) keys of the last block
)


def rb(x):
    return x.to(torch.bfloat16).float()


def attention_fp64(q, k, v, scale):
    """q [..., R, 64], k / v [..., seq, 64] -> fp64 [..., R, 64]"""
    q, k, v = (t.double() for t in (q, k, v))
    return torch.softmax(q @ k.transpose(-1, -2) * scale, -1) @ v


def attention_emulated(q, k, v, scale, bug=None):
    """q [..., R, 64], k / v [..., seq, 64], bf16-rounded values in fp32 -> fp32 holding bf16 values, [..., R, 64]."""
    assert bug is None or bug in PLANTED_BUGS
    seq = k.shape[-2]
    n_kv = (seq + KEY_BLOCK - 1) // KEY_BLOCK
    lead = k.shape[:-2]
    kp = torch.zeros(*lead, n_kv * KEY_BLOCK, HD, dtype=torch.float64, device=k.device)
    vp = torch.zeros_like(kp)
    kp[..., :seq, :] = k.double()
    vp[..., :seq, :] = v.double()
    # the host computes scale * log2(e) in fp32
    sl2 = (torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)).item()
    R = q.shape[-2]
    m = torch.full((*q.shape[:-1],), -math.inf, dtype=torch.float32, device=q.device)
    l = torch.zeros_like(m)
    o = torch.zeros(*q.shape, dtype=torch.float32, device=q.device)
    qd = q.double()
    for j in range(n_kv):
        ks, vs = kp[..., j * KEY_BLOCK:(j + 1) * KEY_BLOCK, :], vp[..., j * KEY_BLOCK:(j + 1) * KEY_BLOCK, :]
        s = (qd @ ks.transpose(-1, -2)).float()          # exact bf16 products, fp32 accumulation
        kv_left = seq - j * KEY_BLOCK
        masked = torch.zeros(KEY_BLOCK, dtype=torch.bool, device=q.device)
        if kv_left < KEY_BLOCK:
            masked[kv_left + (1 if bug == 'mask_off_by_one' else 0):] = True
        s_valid = s.masked_fill(masked, -math.inf)
        n = torch.maximum(m, s_valid.amax(-1) * sl2)
        c = torch.exp2(m - n)                             # 0 on the first block (m = -inf)
        m = n
        # fmaf(s, sl2, -n): the product of two floats is exact in fp64
        p = torch.exp2((s_valid.double() * sl2 - n.double()[..., None]).float())
        r = p.sum(-1)
        if bug == 'l_counts_masked':
            r = r + torch.exp2((s.double() * sl2 - n.double()[..., None]).float()).masked_fill(~masked, 0).sum(-1)
        l = l * c + r
        if bug != 'no_o_rescale':
            o = o * c[..., None]
        o = (o.double() + rb(p).double() @ vs).float()
    return rb(o * (1.0 / l)[..., None])


def bf16_ulp(x):
    """spacing of bf16 values at |x| (x > 0): 2^(floor(log2 x) - 7)"""
    return torch.exp2(torch.floor(torch.log2(x)) - 7)


def rel_linf(got, want):
    got, want = got.double(), want.double()
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-30)).item()


def ones_v_error(out):
    """largest distance from 1.0 in bf16 ulps at 1.0 (2^-7 above, 2^-8 below): a correct kernel gives <= 1"""
    out = out.double()
    return max(((out - 1).clamp_min(0) / 2 ** -7).max().item(), ((1 - out).clamp_min(0) / 2 ** -8).max().item())


# ---------------------------------------------------------------------------------------------------- input cases
def _direction(heads, gen, device):
    d = torch.randn(heads, HD, generator=gen, device=device)
    return d / d.norm(dim=-1, keepdim=True)


def case_random(B, seq, heads, gen, device, std=1.0, via='scale'):
    """randn q / k with logit standard deviation `std`, set either through the softmax scale (q, k ~ N(0, 1),
    scale = std / 8) or through the input magnitude (scale = 0.125, q, k ~ N(0, std))."""
    q, k, v = (torch.randn(B, seq, heads, HD, generator=gen, device=device) for _ in range(3))
    if via == 'scale':
        return q, k, v, std / 8.0
    assert via == 'magnitude'
    return q * math.sqrt(std), k * math.sqrt(std), v, 0.125


def case_all_negative(B, seq, heads, gen, device):
    """keys cluster on +d, queries on -d: every valid logit lies around -35 (within about -43 .. -28), so one leaked
    zero-filled key (logit 0, V = 0) outweighs all valid keys together and pulls the output to 0."""
    d = _direction(heads, gen, device)
    a = math.sqrt(280.0)
    q = -a * d + 0.5 * torch.randn(B, seq, heads, HD, generator=gen, device=device)
    k = a * d + 0.5 * torch.randn(B, seq, heads, HD, generator=gen, device=device)
    v = torch.randn(B, seq, heads, HD, generator=gen, device=device)
    return q, k, v, 0.125


def case_hot_last_key(B, seq, heads, gen, device):
    """every query row is one-hot on key seq - 1 (logit about 20, the others about 0 +- 0.7): the last valid key,
    inside the partial last block when seq % 128 != 0.  Its V row is 3x larger than the rest."""
    d = _direction(heads, gen, device)
    q = 0.5 * torch.randn(B, seq, heads, HD, generator=gen, device=device) + 4.0 * d
    k = torch.randn(B, seq, heads, HD, generator=gen, device=device)
    k[:, seq - 1] = 40.0 * d
    v = torch.randn(B, seq, heads, HD, generator=gen, device=device)
    v[:, seq - 1] *= 3.0
    return q, k, v, 0.125


def case_planted_next_image(B, seq, heads, gen, device, planted=32):
    """every query leans towards +d, and the first `planted` keys of images 1 .. B-1 sit far out on +d (logit about
    10 against about 0): image b's last KV tile must stop at its own seq and never reach image b + 1's keys."""
    assert B >= 2
    d = _direction(heads, gen, device)
    q = 0.5 * torch.randn(B, seq, heads, HD, generator=gen, device=device) + 2.0 * d
    k = torch.randn(B, seq, heads, HD, generator=gen, device=device)
    k[1:, :planted] = 40.0 * d + torch.randn(B - 1, planted, heads, HD, generator=gen, device=device)
    v = torch.randn(B, seq, heads, HD, generator=gen, device=device)
    v[1:, :planted] += 4.0
    return q, k, v, 0.125


def _block_ramp(seq, heads, gen, device, rising, step):
    """keys on +d with a magnitude that is constant inside a 128-key block and moves by `step` logits (at alpha = 1)
    from block to block"""
    d = _direction(heads, gen, device)
    n_kv = (seq + KEY_BLOCK - 1) // KEY_BLOCK
    blk = torch.arange(seq, device=device) // KEY_BLOCK
    level = (blk + 1) if rising else (n_kv - blk)
    beta = 8.0 * step * level.float()                        # logit = 0.125 * alpha * beta
    return d, beta[:, None, None] * d


def case_rising_max(B, seq, heads, gen, device):
    """the row maximum rises in every KV block.  Rows lean on +d with weight alpha in [0.02, 1]: the rescale factor c
    per block ranges from exp(-1.8) (alpha 0.02) to a flush to 0 (alpha >= 0.7, 90 logits per block)."""
    d, kd = _block_ramp(seq, heads, gen, device, True, 90.0)
    alpha = 0.02 + 0.98 * torch.rand(B, seq, heads, 1, generator=gen, device=device)
    q = alpha * d + 0.1 * torch.randn(B, seq, heads, HD, generator=gen, device=device)
    k = kd + 0.3 * torch.randn(B, seq, heads, HD, generator=gen, device=device)
    v = torch.randn(B, seq, heads, HD, generator=gen, device=device)
    return q, k, v, 0.125


def case_first_block_max(B, seq, heads, gen, device):
    """the row maximum sits in the first KV block and never moves again (c = 1 from the second block on; later
    blocks add p far below 1, down to flushed zeros)."""
    d, kd = _block_ramp(seq, heads, gen, device, False, 6.0)
    alpha = 0.05 + 0.95 * torch.rand(B, seq, heads, 1, generator=gen, device=device)
    q = alpha * d + 0.1 * torch.randn(B, seq, heads, HD, generator=gen, device=device)
    k = kd + 0.3 * torch.randn(B, seq, heads, HD, generator=gen, device=device)
    v = torch.randn(B, seq, heads, HD, generator=gen, device=device)
    return q, k, v, 0.125


CASES = {
    'random': case_random,
    'all_negative': case_all_negative,
    'hot_last_key': case_hot_last_key,
    'planted_next_image': case_planted_next_image,
    'rising_max': case_rising_max,
    'first_block_max': case_first_block_max,
}


def make_case(name, B, seq, heads, seed, device, **kw):
    gen = torch.Generator(device=device).manual_seed(seed)
    return CASES[name](B, seq, heads, gen, device, **kw)


def per_head(x):
    """[B, seq, heads, 64] -> [B, heads, seq, 64] bf16-rounded"""
    return rb(x).permute(0, 2, 1, 3)
