"""pf_gemm_timeline: the pf_gemm_kernel phase stamps exist only in a library built with -DPF_GEMM_TIMELINE; the default
build refuses the call with an error that names the switch (and launches nothing).  Needs no GPU."""
import ctypes as C

import pytest


def test_timeline_refused_without_the_build_switch():
    from patchfusion_b200 import build, lib
    build.build()
    buf = (C.c_ulonglong * 8)()
    with pytest.raises(lib.PFError, match='PF_GEMM_TIMELINE'):
        lib.call('pf_gemm_timeline', buf, 1)
