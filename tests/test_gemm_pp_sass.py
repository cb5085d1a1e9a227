"""SASS of the ping-pong GEMM kernel (pf_gemm_pp_kernel): one wgmma shape, the eight MMAs of a K block (two 64-row
halves x four k16 steps) issued back to back with one group in flight, no local memory anywhere, and no GPU-wide
fence in front of the multicast variant's remote stage release.  Needs no GPU.
"""
import os
import re
import subprocess

import pytest

PP_RE = re.compile(r'_ZN2pf17pf_gemm_pp_kernelILb([01])EEEvNS_16GemmKernelParamsE')
HGMMA_RE = re.compile(r'\bHGMMA\.(\d+x\d+x\d+)\.')
LOCAL_RE = re.compile(r'\b(LDL|STL)\b')
ARRIVE_RE = re.compile(r'\bSYNCS\.ARRIVE\.TRANS64\.RED\b')
FENCE_RE = re.compile(r'\bMEMBAR\.ALL\.GPU\b')


@pytest.fixture(scope='module')
def pp_functions():
    from patchfusion_b200 import build
    path = build.build()
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    sass = subprocess.run([cuobjdump, '-sass', path], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in sass.split('Function : ')[1:]:
        name, _, body = part.partition('\n')
        m = PP_RE.match(name.strip())
        if m:
            funcs[int(m.group(1))] = [l for l in body.split('\n') if re.search(r'/\*[0-9a-f]{4,}\*/', l)]
    return funcs


def test_pp_instantiations(pp_functions):
    assert sorted(pp_functions) == [0, 1]


@pytest.mark.parametrize('mc', [0, 1])
def test_pp_mainloop_sass(pp_functions, mc):
    lines = pp_functions[mc]
    shapes = [m.group(1) for m in (HGMMA_RE.search(l) for l in lines) if m]
    assert len(shapes) >= 8, len(shapes)
    assert set(shapes) == {'64x128x16'}, sorted(set(shapes))
    runs, n = [], 0
    for line in lines:
        if HGMMA_RE.search(line):
            n += 1
        elif 'WARPGROUP.DEPBAR' in line:
            if n:
                runs.append(n)
            n = 0
    assert runs and all(r == 8 for r in runs), runs
    assert any(re.search(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x1 ;', l) for l in lines), 'no wait_group 1 in the mainloop'


@pytest.mark.parametrize('mc', [0, 1])
def test_pp_no_local_memory(pp_functions, mc):
    local = [l.strip() for l in pp_functions[mc] if LOCAL_RE.search(l)]
    assert not local, local[:4]


def test_pp_remote_release_has_no_gpu_fence(pp_functions):
    lines = pp_functions[1]
    arrives = 0
    for i, line in enumerate(lines):
        if ARRIVE_RE.search(line):
            arrives += 1
            assert not any(FENCE_RE.search(l) for l in lines[max(0, i - 6):i]), lines[max(0, i - 6):i + 1]
    assert arrives > 0
