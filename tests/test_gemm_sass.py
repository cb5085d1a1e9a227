"""SASS of the implicit-GEMM kernel (pf_gemm_kernel): one fixed wgmma shape per instantiation, a pipelined mainloop and
no local-memory traffic while a K block's MMAs are issued.

ptxas serialises wgmma (a wait after every instruction) when a wgmma sits under a data-dependent branch or its registers
are touched while it may be in flight; that shows in the SASS as a `WARPGROUP.DEPBAR` after each HGMMA.  A spilled
accumulator shows as LDL / STL between the HGMMAs of one K block.  Needs no GPU.
"""
import os
import re
import subprocess

import pytest

GEMM_RE = re.compile(r'_ZN2pf14pf_gemm_kernelILb([01])ELi(\d+)EEEvNS_16GemmKernelParamsE')
HGMMA_RE = re.compile(r'\bHGMMA\.(\d+x\d+x\d+)\.')
LOCAL_RE = re.compile(r'\b(LDL|STL)\b')
WIDTHS = [32, 64, 96, 128, 192, 256]


@pytest.fixture(scope='module')
def gemm_functions():
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
            funcs[(int(m.group(1)), int(m.group(2)))] = body
    return funcs


def test_gemm_instantiations(gemm_functions):
    assert sorted(gemm_functions) == [(mc, bn) for mc in (0, 1) for bn in WIDTHS]


@pytest.mark.parametrize('mc', [0, 1])
@pytest.mark.parametrize('bn', WIDTHS)
def test_gemm_mainloop_sass(gemm_functions, mc, bn):
    body = gemm_functions[(mc, bn)]
    shapes = HGMMA_RE.findall(body)
    assert len(shapes) >= 4, len(shapes)
    assert set(shapes) == {'64x%dx16' % bn}, sorted(set(shapes))
    # HGMMAs between two warpgroup waits: the four k16 steps of a K block go out back to back, and no local-memory
    # access sits between the first and the last of them
    runs, n, local = [], 0, []
    for line in body.split('\n'):
        if HGMMA_RE.search(line):
            n += 1
        elif 'WARPGROUP.DEPBAR' in line:
            if n:
                runs.append(n)
            n = 0
        elif n and LOCAL_RE.search(line):
            local.append(line.strip())
    assert runs and min(runs) >= 4 and all(r % 4 == 0 for r in runs), runs
    assert not local, local[:4]
    # the mainloop keeps one K block's group in flight
    assert re.search(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x1 ;', body), 'no wait_group 1 in the mainloop'
