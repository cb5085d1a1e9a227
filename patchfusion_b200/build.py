"""Builds patchfusion_b200/libpf_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
SOURCES = ['pf_api.cu', 'pf_gemm.cu', 'pf_attn.cu', 'pf_elem.cu', 'pf_post.cu', 'pf_eval.cu', 'pf_stage.cu']
LIB = os.path.join(HERE, os.environ.get('PF_B200_LIBNAME', 'libpf_b200.so'))
EXTRA = os.environ.get('PF_B200_NVCC_EXTRA', '').split()
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
NVCC_FLAGS = ARCH + ['-lineinfo', '-O3', '-std=c++17', '-Xcompiler', '-fPIC']


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, '..', 'include', 'pf_b200.h')]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    objs = []
    os.makedirs(os.path.join(HERE, 'build'), exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, 'build', os.path.basename(LIB) + '.' + src.replace('.cu', '.o'))
        cmd = [nvcc] + NVCC_FLAGS + EXTRA + (['-Xptxas', '-v'] if verbose else []) + ['-c', os.path.join(CSRC, src), '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            raise RuntimeError('nvcc failed on %s' % src)
    cmd = [nvcc] + ARCH + ['-shared', '-o', LIB] + objs + ['-lcudart']
    subprocess.check_call(cmd)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
