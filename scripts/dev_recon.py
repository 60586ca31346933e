"""Developer probe: reconstruction + evaluation kernels at a size the reference cannot touch (n = 32768 by default).

--score split|dot|gaussian picks the gemb_recon_create kind (HOPE's embedding is the input in every case).
--profile adds the device time of the create's kernels from torch.profiler (a separate pass after the timed ones) and,
for gaussian, the distance kernel's achieved write bandwidth and FP32 instruction rate (n^2 d FADD + n^2 d FFMA)."""
import argparse, json, sys, time, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from gem_b200 import _native, synth

KINDS = {'dot': 0, 'split': 1, 'gaussian': 2}
ap = argparse.ArgumentParser()
ap.add_argument('--n', type=int, default=32768)
ap.add_argument('--d', type=int, default=128)
ap.add_argument('--score', default='split', choices=sorted(KINDS))
ap.add_argument('--reps', type=int, default=2)
ap.add_argument('--profile', action='store_true')
a = ap.parse_args()
kind = KINDS[a.score]
csr = synth.sbm(n=a.n, block=1024 if a.n % 1024 == 0 else 1000, seed=1)
ctx = _native.Context(0)
g = _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, None)
X, sig, st = g.hope(a.d, 0.01, tol=1e-4, max_iters=40)
out = {'n': a.n, 'd': a.d, 'score': a.score, 'nnz': csr.nnz, 'hope_ms': st['total_ms']}
lib = _native.lib()
runs = []
for rep in range(a.reps):
    r = {}
    l0 = lib.gemb_launch_count()
    t = time.perf_counter(); rec = _native.Reconstruction(ctx, X, kind); r['create_ms'] = (time.perf_counter() - t) * 1e3
    t = time.perf_counter(); ranks, npr = rec.ranks(csr.indptr, csr.indices, True); r['ranks_ms'] = (time.perf_counter() - t) * 1e3
    t = time.perf_counter(); ti, tj, tw = rec.top(True, 1000); r['top1000_ms'] = (time.perf_counter() - t) * 1e3
    t = time.perf_counter(); ti2, tj2, tw2 = rec.top(True, 1000000); r['top1e6_ms'] = (time.perf_counter() - t) * 1e3
    r['launches'] = int(lib.gemb_launch_count() - l0)
    rec.free()
    runs.append(r)
for key in runs[0]:
    out[key] = min(r[key] for r in runs[1:] or runs)          # first rep is the warm-up when reps > 1
from gem_b200.evaluation import metrics
MAP, _, _ = metrics.map_from_ranks(csr.n, csr.indptr, ranks, True)
out['MAP'] = MAP
out['n_pred'] = int(npr.astype(np.int64).sum())
n_pad = (a.n + 63) // 64 * 64
out['bytes_adj'] = 4.0 * a.n * n_pad
out['create_GBps_written'] = out['bytes_adj'] / (out['create_ms'] * 1e-3) / 1e9
if a.profile:
    import torch
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            _native.Reconstruction(ctx, X, kind).free()
    dev = {}
    for ev in prof.key_averages():
        t_us = getattr(ev, 'device_time_total', None)
        if t_us is None:
            t_us = ev.cuda_time_total
        if t_us and ('recon' in ev.key or 'apply' in ev.key):
            dev[ev.key] = t_us / max(ev.count, 1) / 1e3
    out['create_kernels_ms'] = dev
    sq = [v for k, v in dev.items() if 'recon_sqdist' in k]
    if sq:
        ms = sq[0]
        out['sqdist_ms'] = ms
        out['sqdist_write_TBps'] = out['bytes_adj'] / (ms * 1e-3) / 1e12
        out['sqdist_fp32_Tinstr_per_s'] = 2.0 * a.n * a.n * a.d / (ms * 1e-3) / 1e12
try:
    import subprocess
    out['gpu'] = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                                         text=True).strip()
except Exception:
    pass
print(json.dumps(out))
