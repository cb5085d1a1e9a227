"""pf_gemm against the vendor GEMM (torch.matmul, bf16) on the linear layers of the step, and the phase timeline of
pf_gemm_kernel on the same shapes.

    python tools/linear_vs_vendor.py [--json FILE]
    python tools/linear_vs_vendor.py --timeline [--json FILE]

Each shape runs with the epilogue the model gives it (qkv: bias + V^T store of the last third, proj / fc2: fp32
residual update x += gamma * (acc + b), fc1: exact-erf GELU).  Timing: CUDA graph of REP launches, L2 flushed before
every window, median over windows.  The vendor column is `torch.matmul(x, w.t())` at the same M, K, N in bf16 with a
bf16 output (no epilogue): an upper bound on what a GEMM of that shape costs on this card.

--timeline loads libpf_b200_timeline.so (built with PF_B200_LIBNAME=libpf_b200_timeline.so
PF_B200_NVCC_EXTRA=-DPF_GEMM_TIMELINE python -m patchfusion_b200.build) and reports, per shape, the shares of a
consumer warpgroup's loop spent in the epilogue and waiting for a full stage, and the producer's share waiting for an
empty stage (clock64 stamps; the stamps themselves cost a little time, so the tiles/s of this build is not reported).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# name, M, K, N, epilogue.  D = 1024 (vitl); M = 9333 is one micro-batch of 9 tiles x 1037 tokens, 1037 the coarse image.
SHAPES = [
    ('qkv  M9333', 9333, 1024, 3072, 'vt'),
    ('proj M9333', 9333, 1024, 1024, 'gamma'),
    ('fc1  M9333', 9333, 1024, 4096, 'gelu'),
    ('fc2  M9333', 9333, 4096, 1024, 'gamma'),
    ('qkv  M1037', 1037, 1024, 3072, 'vt'),
    ('proj M1037', 1037, 1024, 1024, 'gamma'),
    ('fc1  M1037', 1037, 1024, 4096, 'gelu'),
    ('fc2  M1037', 1037, 4096, 1024, 'gamma'),
]


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, plim = [s.strip() for s in out.split(',')[:2]]
        return name, plim
    except Exception:
        return 'unknown', 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--timeline', action='store_true')
    ap.add_argument('--json', default=None)
    ap.add_argument('--windows', type=int, default=7)
    ap.add_argument('--rep', type=int, default=10)
    ap.add_argument('--only', nargs='*', default=None)
    args = ap.parse_args()
    if args.timeline:
        os.environ['PF_B200_LIBNAME'] = 'libpf_b200_timeline.so'
    import ctypes as C
    import torch
    from bench import ClockSampler
    from patchfusion_b200 import lib, ops

    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(args.rep):
                fn()
        ts = []
        for _ in range(args.windows):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / args.rep)
        return sorted(ts)[len(ts) // 2]

    tl_buf = (C.c_ulonglong * 8)()

    def timeline(fn):
        fn(); torch.cuda.synchronize()
        lib.call('pf_gemm_timeline', None, 1)
        for _ in range(args.rep):
            fn()
        lib.call('pf_gemm_timeline', tl_buf, 1)
        v = list(tl_buf)
        wg_loop = max(v[7], 1)
        return dict(epilogue=v[6] / wg_loop, mainloop=v[5] / wg_loop, full_wait=v[4] / wg_loop,
                    producer_empty_wait=v[1] / max(v[2], 1),
                    epilogue_kcycles_per_tile=v[6] / max(v[3], 1) / 1e3, mainloop_kcycles_per_tile=v[5] / max(v[3], 1) / 1e3)

    name, plim = gpu_info()
    sampler = ClockSampler(0)
    rows = []
    for label, M, K, N, epi in SHAPES:
        if args.only and not any(o in label for o in args.only):
            continue
        x = torch.randn(M, K, device=dev).to(torch.bfloat16)
        w = torch.randn(N, K, device=dev) / K ** 0.5
        pw = ops.pack_weight(w, torch.randn(N, device=dev))
        if epi == 'vt':
            D = N // 3
            seq = 1037
            B = (M + seq - 1) // seq
            seq_pad = (seq + 63) // 64 * 64
            qk = torch.empty(M, 2 * D, dtype=torch.bfloat16, device=dev)
            vt = torch.zeros(B * D * seq_pad, dtype=torch.bfloat16, device=dev)
            fn = lambda: ops.gemm(pw, [x], qk, vt=vt, vt_col0=2 * D, vt_seq=seq, vt_seq_pad=seq_pad)
        elif epi == 'gamma':
            out = torch.zeros(M, N, dtype=torch.float32, device=dev)
            gam = torch.rand(N, device=dev)
            fn = lambda: ops.gemm(pw, [x], out, gamma=gam)
        else:
            out = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
            fn = lambda: ops.gemm(pw, [x], out, act=ops.ACT_GELU)
        flops = 2.0 * M * K * N
        r = dict(shape=label, M=M, K=K, N=N, epilogue=epi, block_n=fn().block_n)
        if args.timeline:
            r.update(timeline(fn))
            print('%-11s BN %3d  epilogue %5.1f %%  mainloop %5.1f %%  full-stage wait %5.1f %%  producer empty-stage wait %5.1f %%'
                  '  (per tile: mainloop %.1f, epilogue %.1f kcycles)'
                  % (label, r['block_n'], 100 * r['epilogue'], 100 * r['mainloop'], 100 * r['full_wait'],
                     100 * r['producer_empty_wait'], r['mainloop_kcycles_per_tile'], r['epilogue_kcycles_per_tile']),
                  flush=True)
        else:
            ms = timed(fn)
            wb = w.to(torch.bfloat16)
            ms_v = timed(lambda: torch.matmul(x, wb.t()))
            r.update(ms=ms, tflops=flops / ms / 1e9, vendor_ms=ms_v, vendor_tflops=flops / ms_v / 1e9, ratio=ms_v / ms)
            print('%-11s K%5d N%5d BN %3d  ours %7.3f ms %6.1f TF/s   vendor %7.3f ms %6.1f TF/s   ours/vendor %.2f'
                  % (label, K, N, r['block_n'], ms, r['tflops'], ms_v, r['vendor_tflops'], r['ratio']), flush=True)
        rows.append(r)
    clocks = sampler.stop()
    print('card %s, power limit %s, median SM clock %s MHz (max %s)' % (name, plim, clocks.get('sm_mhz'), clocks.get('sm_max_mhz')))
    if args.json:
        json.dump(dict(card=name, power_limit=plim, clocks=clocks, rows=rows), open(args.json, 'w'), indent=1)


if __name__ == '__main__':
    main()
