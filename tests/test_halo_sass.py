"""SASS of the halo-tile 3x3 conv kernel: one fixed wgmma shape per instantiation and a pipelined mainloop.

The kernel's speed rests on the tensor cores seeing several k16 MMAs in flight.  ptxas serialises wgmma (a wait after
every instruction) when a wgmma sits under a data-dependent branch or its registers are touched while it may be in
flight; that shows in the SASS as a `WARPGROUP.DEPBAR` after each HGMMA.  Needs no GPU.
"""
import os
import re
import subprocess

import pytest

HALO_RE = re.compile(r'_ZN2pf20pf_conv3_halo_kernelILi(\d+)ELi(\d+)EEEv')
HGMMA_RE = re.compile(r'\bHGMMA\.(\d+x\d+x\d+)\.')


@pytest.fixture(scope='module')
def halo_functions():
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
            funcs[(int(m.group(1)), int(m.group(2)))] = body
    return funcs


def test_halo_instantiations(halo_functions):
    assert sorted(halo_functions) == [(cl, bn) for cl in (1, 2, 4) for bn in (32, 64, 128, 192)]


@pytest.mark.parametrize('cl', [1, 2, 4])
@pytest.mark.parametrize('bn', [32, 64, 128, 192])
def test_halo_mainloop_sass(halo_functions, cl, bn):
    body = halo_functions[(cl, bn)]
    shapes = HGMMA_RE.findall(body)
    # nine taps x four k16 steps per 64-channel chunk, fully unrolled
    assert len(shapes) >= 36, len(shapes)
    assert set(shapes) == {'64x%dx16' % bn}, sorted(set(shapes))
    # HGMMAs between two warpgroup waits: the four k16 steps of a tap (or more) go out back to back
    runs, n = [], 0
    for line in body.split('\n'):
        if HGMMA_RE.search(line):
            n += 1
        elif 'WARPGROUP.DEPBAR' in line:
            if n:
                runs.append(n)
            n = 0
    assert runs and min(runs) >= 4 and all(r % 4 == 0 for r in runs), runs
    # the mainloop keeps one tap's group in flight
    assert re.search(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x1 ;', body), 'no wait_group 1 in the mainloop'
