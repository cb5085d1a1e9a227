"""SASS of the operand-stage release in the multicast GEMM and halo-conv kernels: the consumers' arrive on a peer CTA's
empty barrier is not preceded by a GPU-wide fence.

A stage is released after wgmma.wait_group has retired every wgmma that read it, so the arrive has nothing to order;
with `.release.cluster` semantics ptxas put a MEMBAR.ALL.GPU in front of every such arrive, inside the mainloop.
Needs no GPU.
"""
import os
import re
import subprocess

import pytest

KERNEL_RE = re.compile(r'_ZN2pf(14pf_gemm_kernelILb1|20pf_conv3_halo_kernelILi[24])')
ARRIVE_RE = re.compile(r'\bSYNCS\.ARRIVE\.TRANS64\.RED\b')
FENCE_RE = re.compile(r'\bMEMBAR\.ALL\.GPU\b')


@pytest.fixture(scope='module')
def multicast_functions():
    from patchfusion_b200 import build
    path = build.build()
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    sass = subprocess.run([cuobjdump, '-sass', path], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in sass.split('Function : ')[1:]:
        name, _, body = part.partition('\n')
        if KERNEL_RE.match(name.strip()):
            funcs[name.strip()] = [l for l in body.split('\n') if re.search(r'/\*[0-9a-f]{4,}\*/', l)]
    return funcs


def test_multicast_instantiations_found(multicast_functions):
    # pf_gemm_kernel<true, BN> for six widths, pf_conv3_halo_kernel<2 | 4, BN> for four
    assert len(multicast_functions) == 6 + 8, sorted(multicast_functions)


def test_remote_release_has_no_gpu_fence(multicast_functions):
    bad = []
    for name, lines in multicast_functions.items():
        arrives = 0
        for i, line in enumerate(lines):
            if ARRIVE_RE.search(line):
                arrives += 1
                if any(FENCE_RE.search(l) for l in lines[max(0, i - 6):i]):
                    bad.append(name)
                    break
        assert arrives > 0, name
    assert not bad, bad
