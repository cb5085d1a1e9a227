"""The fragment-layout epilogue of pf_gemm_kernel: its SASS (stmatrix staging, bulk stores, next to no spills) and a
host-side model of its shared-memory addressing.

The TMA-store epilogue applies bias / activation / gamma on the wgmma accumulator fragment and stages each warp's 16
rows with stmatrix (bf16) or 8-byte stores (fp32).  The model replays the kernel's per-lane address arithmetic and the
stmatrix semantics in numpy and compares the staged tile with what the bulk copy expects: SWIZZLE_128B rows of 128 bytes.
Needs no GPU.
"""
import os
import re
import subprocess

import numpy as np
import pytest

GEMM_RE = re.compile(r'_ZN2pf14pf_gemm_kernelILb([01])ELi(\d+)EEEvNS_16GemmKernelParamsE')
WIDTHS = [32, 64, 96, 128, 192, 256]
# spill stores (STL instructions) per instantiation; the row-per-thread epilogue this one replaced had 25-70 at
# BN <= 128 and over 750 at BN = 256
STL_BOUND = {32: 0, 64: 8, 96: 8, 128: 8, 192: 200, 256: 400}


@pytest.fixture(scope='module')
def gemm_sass():
    from patchfusion_b200 import build
    path = build.build()
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    sass = subprocess.run([cuobjdump, '-sass', path], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in sass.split('Function : ')[1:]:
        name, _, body = part.partition('\n')
        m = GEMM_RE.match(name.strip())
        if m:
            funcs[(int(m.group(1)), int(m.group(2)))] = [l for l in body.split('\n') if re.search(r'/\*[0-9a-f]{4,}\*/', l)]
    return funcs


@pytest.mark.parametrize('mc', [0, 1])
@pytest.mark.parametrize('bn', WIDTHS)
def test_epilogue_sass(gemm_sass, mc, bn):
    lines = gemm_sass[(mc, bn)]
    count = lambda pat: sum(1 for l in lines if re.search(pat, l))
    # fp32 tiles: 8-byte staging stores and the bulk reduce-add, at every width
    assert count(r'\bSTS\.64\b') >= 8 and count(r'\bUTMAREDG\b') >= 1
    # bf16 tiles (widths of whole 64-column groups): stmatrix and bulk tensor stores
    if bn % 64 == 0:
        assert count(r'\bSTSM\.16\.M88\.4\b') >= 4 and count(r'\bUTMASTG\b') >= 2
    assert count(r'\bSTL\b') <= STL_BOUND[bn], count(r'\bSTL\b')
    # nothing is spilled while a block is staged: no STL between an stmatrix and the bulk store that follows it
    staging, bad = False, []
    for l in lines:
        if re.search(r'\bSTSM\b', l):
            staging = True
        elif re.search(r'\bUTMASTG\b', l):
            staging = False
        elif staging and re.search(r'\bSTL\b', l):
            bad.append(l.strip())
    assert not bad, bad[:4]


# ------------------------------------------------------------------------------------------------ addressing model
def swizzle_128b(row, byte):
    """byte offset, in a tile of 128-byte rows written or read by TMA with SWIZZLE_128B, of byte `byte` of row `row`"""
    return row * 128 + ((((byte >> 4) ^ (row & 7)) << 4) | (byte & 15))


def frag_elem(lane, i):
    """(row, column) within a 16 x 32 chunk of accumulator i of a lane's 16-value fragment slice"""
    j, e = divmod(i, 4)
    return lane // 4 + 8 * (e >> 1), 8 * j + 2 * (lane % 4) + (e & 1)


def stmatrix_x4(mem, addrs, regs):
    """stmatrix.sync.aligned.m8n8.x4.shared.b16: addrs[l] = row address of matrix l // 8, row l % 8;
    regs[l][m] = the two 16-bit elements lane l holds of matrix m (row l // 4, columns 2 (l % 4) + {0, 1})"""
    for m in range(4):
        mat = np.empty((8, 8), dtype=mem.dtype)
        for l in range(32):
            mat[l // 4, 2 * (l % 4)], mat[l // 4, 2 * (l % 4) + 1] = regs[l][m]
        for i in range(8):
            a = addrs[8 * m + i]
            assert a % 16 == 0
            mem[a // 2:a // 2 + 8] = mat[i]


def _stage_bf16():
    """a warp's 16 rows x 64 columns staged as the kernel does; element value = 64 * row + column"""
    mem = np.full(1024, -1, dtype=np.int32)       # 2 KB of 16-bit elements
    for h in range(2):
        for p in range(2):
            o = 4 * h + 2 * p
            addrs, regs = [], []
            for lane in range(32):
                oct_ = lane >> 4
                addrs.append((lane & 15) * 128 + (((o + oct_) ^ (lane & 7)) << 4))
                val = lambda i: (lambda rc: 64 * rc[0] + 32 * h + rc[1])(frag_elem(lane, i))
                regs.append([(val(8 * p + 2 * m), val(8 * p + 2 * m + 1)) for m in range(4)])
            stmatrix_x4(mem, addrs, regs)
    return mem


def test_bf16_staging_matches_swizzle_128b():
    mem = _stage_bf16()
    want = np.empty(1024, dtype=np.int32)
    for r in range(16):
        for c in range(64):
            want[swizzle_128b(r, 2 * c) // 2] = 64 * r + c
    assert (mem == want).all()


def test_f32_staging_matches_swizzle_128b():
    mem = np.full(512, -1, dtype=np.int32)        # 2 KB of 32-bit elements
    for lane in range(32):
        r, q = lane >> 2, lane & 3
        lane_off = r * 128 + (q & 1) * 8
        for j in range(4):
            addr = lane_off + (((2 * j + (q >> 1)) ^ r) << 4)
            for half, a in ((0, addr), (1, addr + 8 * 128)):
                for e in range(2):
                    row, col = frag_elem(lane, 4 * j + 2 * half + e)
                    mem[a // 4 + e] = 32 * row + col
    want = np.empty(512, dtype=np.int32)
    for r in range(16):
        for c in range(32):
            want[swizzle_128b(r, 4 * c) // 4] = 32 * r + c
    assert (mem == want).all()
