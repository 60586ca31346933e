"""gem_b200/build.py -- compiles libgemb200.so IN-TREE with nvcc for sm_90a (H100; no torch, no JIT cache).

    python -m gem_b200.build [--force] [--verbose]

The .so and the objects under csrc/build/ are build products (git-ignored).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(HERE, 'csrc', 'build')
LIB = os.path.join(HERE, 'libgemb200.so')
SOURCES = ['core.cu', 'spmm.cu', 'dense.cu', 'gram_tc.cu', 'apply_tc.cu', 'hope.cu', 'halo.cu', 'n2v.cu', 'recon.cu', 'ingest.cu', 'synth.cu', 'gf.cu', 'nc.cu', 'cc.cu', 'tsne.cu']
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
CFLAGS = ['-O3', '-std=c++17', '-lineinfo', '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=default',
          '--expt-relaxed-constexpr']


def _newer(src, dst):
    return (not os.path.exists(dst)) or os.path.getmtime(src) > os.path.getmtime(dst)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    headers.append(os.path.join(os.path.dirname(HERE), 'include', 'gemb200.h'))
    hdr_time = max(os.path.getmtime(h) for h in headers)
    objs = []
    procs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        if not os.path.exists(src):
            continue
        obj = os.path.join(OBJ, s.replace('.cu', '.o'))
        objs.append(obj)
        if force or _newer(src, obj) or os.path.getmtime(obj) < hdr_time:
            cmd = [NVCC] + ARCH + CFLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', src, '-o', obj]
            if verbose:
                print(' '.join(cmd))
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            print('---- %s' % s)
            print(out)
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError('nvcc failed')
    if force or procs or not os.path.exists(LIB):
        cmd = [NVCC] + ARCH + ['-shared', '-cudart', 'static', '-o', LIB] + objs + ['-ldl']
        if verbose:
            print(' '.join(cmd))
        subprocess.check_call(cmd)
    return LIB


if __name__ == '__main__':
    build(force='--force' in sys.argv, verbose='--verbose' in sys.argv)
    print(LIB)
