"""Developer probe for BASELINE configs[3] at reduced scale: HOPE d=128 on a Graph500 R-MAT graph,
beta = 0.5 / rho(A) with rho from 50 power iterations (SURVEY 8(d) config 4)."""
import argparse, json, sys, time, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from gem_b200 import _native, synth

ap = argparse.ArgumentParser()
ap.add_argument('--scale', type=int, default=22)
ap.add_argument('--d', type=int, default=128)
ap.add_argument('--tol', type=float, default=1e-3)
ap.add_argument('--reps', type=int, default=2)
a = ap.parse_args()
t = time.time()
csr = synth.rmat(scale=a.scale)
deg = np.diff(csr.indptr)
print('rmat scale', a.scale, 'n', csr.n, 'nnz', csr.nnz, 'max deg', int(deg.max()), 'isolated', int((deg == 0).sum()),
      'gen s', round(time.time() - t, 1), flush=True)
ctx = _native.Context(0)
g = _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, None)
# rho(A) by power iteration through the SpMM entry (4 columns: the narrowest block the ABI takes)
rng = np.random.default_rng(1)
x = rng.standard_normal((csr.n, 4)).astype(np.float32)
rho = 0.0
t = time.time()
for it in range(50):
    y = g.spmm(x)
    nrm = np.linalg.norm(y, axis=0)
    rho = float(nrm.max() / max(np.linalg.norm(x, axis=0).max(), 1e-30)) if it else 0.0
    x = (y / np.maximum(nrm, 1e-30)).astype(np.float32)
y = g.spmm(x)
rho = float(np.max(np.sum(x * y, axis=0)))          # Rayleigh quotient of the normalised iterate
beta = 0.5 / rho
print('rho(A) ~ %.4f (50 power iterations, %.1f s)  beta = %.6g' % (rho, time.time() - t, beta), flush=True)
for r in range(a.reps):
    last = r == a.reps - 1
    X, sig, st = g.hope(a.d, beta, tol=a.tol, max_iters=60, oversample=16, seed=1234, want_output=last,
                        compute_residual=int(last), verbose=int(r == 0))
    st['nodes_per_s_device'] = csr.n / (st['total_ms'] * 1e-3)
    st['spmm_GBps'] = st['spmm_bytes'] * st['spmm_count'] / (st['spmm_ms'] * 1e-3) / 1e9 if st['spmm_ms'] > 0 else 0
    print(json.dumps(st), flush=True)
print('sigma', sig[:3], sig[-3:], 'finite', bool(np.isfinite(X).all()))
out = {'scale': a.scale, 'n': csr.n, 'nnz': csr.nnz, 'rho': rho, 'beta': beta, 'stats': st,
       'sigma_top': [float(s) for s in sig[-5:]]}
print(json.dumps(out), flush=True)
