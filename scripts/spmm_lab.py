"""Writes the BASELINE configs[1] SBM as raw int32 arrays for scripts/spmm_lab.cu and runs it."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from gem_b200 import synth
kind = sys.argv[1] if len(sys.argv) > 1 else 'sbm'
csr = synth.sbm(n=1_000_000, block=1000, seed=42) if kind == 'sbm' else synth.rmat(scale=20)
d = '/dev/shm' if os.path.isdir('/dev/shm') else '/tmp'
csr.indptr.astype(np.int32).tofile(d + '/lab_indptr.bin')
csr.indices.astype(np.int32).tofile(d + '/lab_indices.bin')
exe = '/tmp/spmm_lab'
subprocess.check_call(['nvcc', '-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-o', exe,
                       os.path.join(os.path.dirname(os.path.abspath(__file__)), 'spmm_lab.cu')])
mode = sys.argv[2:3]          # 'quick': row-major variants only
subprocess.check_call([exe, d + '/lab_indptr.bin', d + '/lab_indices.bin'] + mode)
