"""Developer probe: reconstruction + evaluation kernels at a size the reference cannot touch (n = 32768 by default)."""
import argparse, json, sys, time, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from gem_b200 import _native, synth

ap = argparse.ArgumentParser()
ap.add_argument('--n', type=int, default=32768)
ap.add_argument('--d', type=int, default=128)
a = ap.parse_args()
csr = synth.sbm(n=a.n, block=1024 if a.n % 1024 == 0 else 1000, seed=1)
ctx = _native.Context(0)
g = _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, None)
X, sig, st = g.hope(a.d, 0.01, tol=1e-4, max_iters=40)
out = {'n': a.n, 'd': a.d, 'nnz': csr.nnz, 'hope_ms': st['total_ms']}
lib = _native.lib()
for rep in range(2):
    l0 = lib.gemb_launch_count()
    t = time.perf_counter(); rec = _native.Reconstruction(ctx, X, True); out['create_ms'] = (time.perf_counter() - t) * 1e3
    t = time.perf_counter(); ranks, npr = rec.ranks(csr.indptr, csr.indices, True); out['ranks_ms'] = (time.perf_counter() - t) * 1e3
    t = time.perf_counter(); ti, tj, tw = rec.top(True, 1000); out['top1000_ms'] = (time.perf_counter() - t) * 1e3
    t = time.perf_counter(); ti2, tj2, tw2 = rec.top(True, 1000000); out['top1e6_ms'] = (time.perf_counter() - t) * 1e3
    out['launches'] = int(lib.gemb_launch_count() - l0)
    rec.free()
from gem_b200.evaluation import metrics
MAP, _, _ = metrics.map_from_ranks(csr.n, csr.indptr, ranks, True)
out['MAP'] = MAP
out['n_pred'] = int(npr.astype(np.int64).sum())
out['bytes_adj'] = 4.0 * a.n * ((a.n + 63) // 64 * 64)
out['create_GBps_written'] = out['bytes_adj'] / (out['create_ms'] * 1e-3) / 1e9
print(json.dumps(out))
