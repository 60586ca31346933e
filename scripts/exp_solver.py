"""Developer experiment (not the bench): the symmetric HOPE solver on the BASELINE configs[1] graph under a matrix of
settings -- filter degree, dynamic-range guard, oversampling, stopping rule -- each reported with its sweeps, device
time and the residual of the result against the fp32 Katz operator (a second, untimed call)."""
import itertools, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gem_b200 import _native, synth

n = int(os.environ.get('EXP_N', '1000000'))
csr = synth.sbm(n=n, block=1000, seed=42)
ctx = _native.Context(0)
g = _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, None)
base = dict(seed=1234, min_iters=2, max_iters=30)
grid = [dict(tol=1e-3, oversample=16, cheb_degree=8, cheb_range_log2=8, stop_rule=0)]
for deg, rng, osamp in itertools.product((8, 10, 12, 16), (8, 14, 20), (8, 16)):
    for stop, tol in ((0, 1e-3), (1, 4e-3), (1, 2e-3)):
        if deg == 8 and rng == 8 and osamp == 16 and stop == 0:
            continue
        grid.append(dict(tol=tol, oversample=osamp, cheb_degree=deg, cheb_range_log2=rng, stop_rule=stop))
for basis in (0, 128, 192):
    grid.append(dict(tol=1e-3, oversample=16, algorithm=3, algorithm3_basis=basis))
g.hope(128, 0.01, want_output=False, **base, **grid[0])           # warm-up
for cfg in grid:
    best = None
    for _ in range(2):
        _, _, st = g.hope(128, 0.01, want_output=False, **base, **cfg)
        if best is None or st['total_ms'] < best['total_ms']:
            best = st
    try:
        _, _, sr = g.hope(128, 0.01, want_output=False, compute_residual=1, **base, **cfg)
    except RuntimeError as exc:
        sr = {'resid_max': str(exc)}
    rec = dict(cfg, iters=best['iters'], converged=best['converged'], sweeps=best['spmm_count'], total_ms=round(best['total_ms'], 2),
               spmm_ms=round(best['spmm_ms'], 2), dense_ms=round(best['dense_ms'], 2), block=best['block'],
               ritz_change=best['ritz_change'], resid_est=best['resid_est'], resid_max=sr['resid_max'])
    print(json.dumps(rec), flush=True)
g.free(); ctx.close()
