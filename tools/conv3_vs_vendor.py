"""pf_conv3_halo_kernel against the vendor convolution (F.conv2d, bf16, channels_last) on the 3x3 convs that carry the
step's conv FLOPs, and the phase timeline of the halo kernel on the same shapes.

    python tools/conv3_vs_vendor.py [--json FILE]
    python tools/conv3_vs_vendor.py --timeline [--json FILE]

Each shape runs at micro-batch 9 (one micro-batch of the vitl 4K m2 step) with its real epilogue: bias + ReLU, bf16
NHWC out.  Timing as in linear_vs_vendor.py: CUDA graph of REP launches, L2 flushed before every window, median over
windows; TFLOP/s on true FLOPs (2 * pixels * 9 * Cin * Cout).  The vendor column is F.conv2d(x, w, b, padding=1) on
channels_last bf16 tensors: a reference point, not a bound.

--timeline loads libpf_b200_timeline.so (built with PF_B200_LIBNAME=libpf_b200_timeline.so
PF_B200_NVCC_EXTRA=-DPF_GEMM_TIMELINE python -m patchfusion_b200.build) and reports, per shape, the shares of a
consumer warpgroup's loop spent in the epilogue and waiting for a full halo slot or weight stage, and the producer's
share waiting for an empty one.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

NB = 9
# name, H, W, Cin, Cout (vitl, per tile)
SHAPES = [
    ('up_conv_list.4 conv0', 392, 518, 544, 544),
    ('up_conv_list.3 conv0', 224, 296, 768, 768),
    ('up_conv_list.3 conv2', 224, 296, 768, 256),
    ('up_conv_list.2 conv0', 112, 148, 768, 768),
    ('fusion_conv_list.4', 224, 296, 512, 256),
    ('up_conv_list.4 conv2', 392, 518, 544, 32),
    ('inc conv1', 392, 518, 32, 32),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--timeline', action='store_true')
    ap.add_argument('--json', default=None)
    ap.add_argument('--windows', type=int, default=7)
    ap.add_argument('--rep', type=int, default=5)
    ap.add_argument('--only', nargs='*', default=None)
    args = ap.parse_args()
    if args.timeline:
        os.environ['PF_B200_LIBNAME'] = 'libpf_b200_timeline.so'
    import ctypes as C
    import torch
    import torch.nn.functional as F
    from bench import ClockSampler
    from linear_vs_vendor import gpu_info
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
    for label, H, W, Cin, Cout in SHAPES:
        if args.only and not any(o in label for o in args.only):
            continue
        x = torch.randn(NB, H, W, Cin, device=dev).to(torch.bfloat16)
        w = torch.randn(Cout, Cin, 3, 3, device=dev) / (9 * Cin) ** 0.5
        b = torch.randn(Cout, device=dev)
        pw = ops.pack_weight(w, b)
        out = torch.empty(NB, H, W, Cout, dtype=torch.bfloat16, device=dev)
        fn = lambda: ops.gemm(pw, [x], out, image=(NB, H, W), act=ops.ACT_RELU)
        flops = 2.0 * NB * H * W * 9 * Cin * Cout
        d = fn()
        r = dict(shape=label, NB=NB, H=H, W=W, Cin=Cin, Cout=Cout, block_n=d.block_n, gflop=flops / 1e9)
        if args.timeline:
            r.update(timeline(fn))
            print('%-21s BN %3d  epilogue %5.1f %%  mainloop %5.1f %%  full wait %5.1f %%  producer empty wait %5.1f %%'
                  '  (per tile: mainloop %.1f, epilogue %.1f kcycles)'
                  % (label, r['block_n'], 100 * r['epilogue'], 100 * r['mainloop'], 100 * r['full_wait'],
                     100 * r['producer_empty_wait'], r['mainloop_kcycles_per_tile'], r['epilogue_kcycles_per_tile']),
                  flush=True)
        else:
            ms = timed(fn)
            xv = x.permute(0, 3, 1, 2)                      # NCHW view of the NHWC tensor: channels_last
            wv = w.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
            bv = b.to(torch.bfloat16)
            ms_v = timed(lambda: F.conv2d(xv, wv, bv, padding=1))
            r.update(ms=ms, tflops=flops / ms / 1e9, vendor_ms=ms_v, vendor_tflops=flops / ms_v / 1e9, ratio=ms_v / ms)
            print('%-21s %3dx%3d %3d->%3d BN %3d  ours %7.3f ms %6.1f TF/s   vendor %7.3f ms %6.1f TF/s   vendor/ours %.2f'
                  % (label, H, W, Cin, Cout, r['block_n'], ms, r['tflops'], ms_v, r['vendor_tflops'], r['ratio']), flush=True)
        rows.append(r)
        del x, out
    clocks = sampler.stop()
    print('card %s, power limit %s, median SM clock %s MHz (max %s)' % (name, plim, clocks.get('sm_mhz'), clocks.get('sm_max_mhz')))
    if args.json:
        json.dump(dict(card=name, power_limit=plim, clocks=clocks, rows=rows), open(args.json, 'w'), indent=1)


if __name__ == '__main__':
    main()
