"""The bulk-store epilogue of pf_conv3_halo_kernel: its SASS (stmatrix staging, bulk tensor stores, no spill while a
block is staged) and a host-side model of its staging addresses for both group widths.

Plain bf16 outputs are staged per warp as 16 rows of 64 columns (128-byte rows, SWIZZLE_128B) or, at BN = 32, of 32
columns (64-byte rows, SWIZZLE_64B).  The model replays the kernel's per-lane address arithmetic and the stmatrix
semantics in numpy and compares the staged tile with where the bulk copy reads each element: the swizzle XORs address
bits 4-6 with bits 7-9 (128B) or bits 4-5 with bits 7-8 (64B).  Needs no GPU.
"""
import os
import re
import subprocess

import numpy as np
import pytest

from test_gemm_epilogue_sass import frag_elem, stmatrix_x4

HALO_RE = re.compile(r'_ZN2pf20pf_conv3_halo_kernelILi(\d)ELi(\d+)EEEvNS_16GemmKernelParamsE')
# spill stores (STL instructions) per width, all clusters (CUDA 12.9).  At BN = 192 they belong to the row-per-thread
# path the residual / ReLU-copy / fused-tail outputs still take (250-265 before the bulk-store path was added): the
# bound keeps them from growing and the staging check below keeps them out of the new path.
STL_BOUND = {32: 0, 64: 1, 128: 8, 192: 270}


@pytest.fixture(scope='module')
def halo_sass():
    from patchfusion_b200 import build
    path = build.build()
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    sass = subprocess.run([cuobjdump, '-sass', path], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in sass.split('Function : ')[1:]:
        name, _, body = part.partition('\n')
        m = HALO_RE.match(name.strip())
        if m:
            funcs[(int(m.group(1)), int(m.group(2)))] = [l for l in body.split('\n') if re.search(r'/\*[0-9a-f]{4,}\*/', l)]
    return funcs


@pytest.mark.parametrize('cl', [1, 2, 4])
@pytest.mark.parametrize('bn', [32, 64, 128, 192])
def test_halo_epilogue_sass(halo_sass, cl, bn):
    lines = halo_sass[(cl, bn)]
    count = lambda pat: sum(1 for l in lines if re.search(pat, l))
    assert count(r'\bSTSM\.16\.M88\.4\b') >= 2 and count(r'\bUTMASTG\b') >= 1
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
def swizzle(addr, row_bytes):
    """where TMA with SWIZZLE_128B (128-byte rows) or SWIZZLE_64B (64-byte rows) puts byte `addr` of the tile"""
    bits = 7 if row_bytes == 128 else 3
    return addr ^ (((addr >> 7) & bits) << 4)


def _stage_bf16(G):
    """a warp's 16 rows x G columns staged as epilogue_tile_tma_bf16<G> does; element value = G * row + column"""
    mem = np.full(16 * G, -1, dtype=np.int32)      # 16 rows of G 16-bit elements
    for h in range(G // 32):
        for p in range(2):
            o = 4 * h + 2 * p
            addrs, regs = [], []
            for lane in range(32):
                oct_ = lane >> 4
                swz = (lane & 7) if G == 64 else ((lane >> 1) & 3)
                addrs.append((lane & 15) * 2 * G + (((o + oct_) ^ swz) << 4))
                val = lambda i: (lambda rc: G * rc[0] + 32 * h + rc[1])(frag_elem(lane, i))
                regs.append([(val(8 * p + 2 * m), val(8 * p + 2 * m + 1)) for m in range(4)])
            stmatrix_x4(mem, addrs, regs)
    return mem


@pytest.mark.parametrize('G', [32, 64])
def test_bf16_staging_matches_swizzle(G):
    mem = _stage_bf16(G)
    want = np.empty(16 * G, dtype=np.int32)
    for r in range(16):
        for c in range(G):
            want[swizzle(r * 2 * G + 2 * c, 2 * G) // 2] = G * r + c
    assert (mem == want).all()


@pytest.mark.parametrize('G', [32, 64])
def test_stmatrix_rows_conflict_free(G):
    """each 8 x 8 matrix's eight 16-byte rows land in eight distinct 16-byte bank groups"""
    for o in range(G // 8):
        for half in range(2):
            rows = range(8 * half, 8 * half + 8)
            swz = [(r & 7) if G == 64 else ((r >> 1) & 3) for r in rows]
            banks = {((r * 2 * G + ((o ^ s) << 4)) % 128) // 16 for r, s in zip(rows, swz)}
            assert len(banks) == 8
