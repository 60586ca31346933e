#!/usr/bin/env python
"""Compare two builds of libgemb200.so on the b x b fp64 factorizations (chol_inverse, eigh): outputs and kernel time.

    python scripts/dense_factor_compare.py --base OTHER/libgemb200.so [--reps 2]

Both libraries export the same symbols, so each run is a subprocess that loads one of them.  The runs alternate
base, this tree, base, this tree, ...  Each run
  * calls gemb_chol_inverse / gemb_eigh on the seeded inputs of tests/test_gpu_small_dense.py (every kind and size there)
    and keeps the outputs (first run of each library only);
  * times the factorization kernels with torch.profiler (device time per call, mean over the profiled calls):
    Cholesky at b in CHOL_TIMED, Jacobi at b in EIGH_TIMED (random symmetric input, rel_tol 1e-9);
  * runs HOPE d = 256, oversample 128 (b = 256) on the SBM-1024 fixture, algorithms 1 and 2, and keeps stats dense_ms.
Prints one JSON line: per size and output, whether the outputs are bit-identical and their largest difference (absolute, and
relative to the largest base entry of the same output), the kernel
times of both libraries (min over runs), and the card's name and power limit.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
CHOL_TIMED = [144, 160, 200, 256, 512]
EIGH_TIMED = [192, 256, 400]


def _inputs():
    """(name, kind of call, G, rel_tol) for every input the small-dense tests use."""
    sys.path.insert(0, os.path.join(REPO, 'tests'))
    import test_gpu_small_dense as t
    out = []
    for b in t.CHOL_SIZES:
        for kind in t.CHOL_KINDS:
            if b == 1 and kind.startswith('pivot'):
                continue
            out.append(('chol/%d/%s' % (b, kind), 'chol', t._chol_input(kind, b, np.random.default_rng(1000 + b))[0], 0.0))
    for b in t.EIGH_SIZES:
        for kind in t.EIGH_KINDS:
            out.append(('eigh/%d/%s' % (b, kind), 'eigh', t._eigh_input(kind, b, np.random.default_rng(2000 + b))[0], 1e-13))
        d = np.random.default_rng(3000 + b).integers(-3, 4, b).astype(np.float64)
        out.append(('eigh/%d/diagonal' % b, 'eigh', np.diag(d), 1e-13))
        for kind in ('random', 'sbm', 'graded'):
            G = t._eigh_input(kind, b, np.random.default_rng(4000 + b))[0]
            out.append(('eigh/%d/%s_tol1e-5' % (b, kind), 'eigh', G, 1e-5))
    return out


def _kernel_ms(prof, key):
    tot, n = 0.0, 0
    for ev in prof.key_averages():
        if key in ev.key:
            t_us = getattr(ev, 'device_time_total', None)
            tot += (ev.cuda_time_total if t_us is None else t_us) / 1e3
            n += ev.count
    return tot, n


def run_one(lib_path, out_path, dump):
    from gem_b200 import _native
    _native.LIB_PATH = lib_path
    import torch
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.init()
    ctx = _native.Context(0)
    res = {}
    if dump:
        arrays = {}
        for name, what, G, tol in _inputs():
            r = ctx.chol_inverse(G) if what == 'chol' else ctx.eigh(G, rel_tol=tol)
            for i, a in enumerate(r):
                arrays['%s/%d' % (name, i)] = np.asarray(a)
        np.savez(out_path + '.npz', **arrays)
    rng = np.random.default_rng(7)
    times = {}
    for what, sizes, calls in (('chol', CHOL_TIMED, 20), ('eigh', EIGH_TIMED, 4)):
        for b in sizes:
            P = rng.standard_normal((4 * b, b))
            G = P.T @ P if what == 'chol' else (P[:b] + P[:b].T) / 2
            call = (lambda: ctx.chol_inverse(G)) if what == 'chol' else (lambda: ctx.eigh(G, rel_tol=1e-9))
            call(); call()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(calls):
                    call()
            tot, n = _kernel_ms(prof, 'chol_inverse' if what == 'chol' else 'eigh_jacobi')
            assert n >= calls - 1, (what, b, n)      # the profiler may miss the last launch of the window
            times['%s/%d' % (what, b)] = tot / n
    ctx.close()
    sys.path.insert(0, os.path.join(REPO, 'tests'))
    from conftest import load_sbm1024_nx
    from gem_b200.embedding.hope import HOPE
    G, _ = load_sbm1024_nx()
    for alg in (1, 2):
        HOPE.hyper_params.clear(); HOPE.hyper_params.update({'method_name': 'hope_gsvd'})
        m = HOPE(d=256, beta=0.01, oversample=128, tol=1e-9, max_iters=400, min_iters=8, algorithm=alg)
        m.learn_embedding(graph=G, is_weighted=True, no_python=True)
        times['hope_d256_alg%d_dense_ms' % alg] = m.stats['dense_ms']
        times['hope_d256_alg%d_iters' % alg] = m.stats['iters']
    res['times'] = times
    with open(out_path + '.json', 'w') as f:
        json.dump(res, f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--base', help='libgemb200.so to compare against (required)')
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--run', nargs=3, metavar=('LIB', 'OUT', 'DUMP'), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.run:
        return run_one(a.run[0], a.run[1], a.run[2] == '1')
    if not a.base:
        ap.error('--base is required')
    tmp = tempfile.mkdtemp(prefix='dense_factor_compare_')      # the output dumps: ~300 MB per library
    libs = {'base': os.path.abspath(a.base), 'tree': os.path.join(REPO, 'gem_b200', 'libgemb200.so')}
    times = {k: [] for k in libs}
    for rep in range(a.reps):
        for k, lib in libs.items():
            o = os.path.join(tmp, '%s_%d' % (k, rep))
            subprocess.check_call([sys.executable, os.path.abspath(__file__), '--run', lib, o, '1' if rep == 0 else '0'])
            times[k].append(json.load(open(o + '.json'))['times'])
    zb, zt = np.load(os.path.join(tmp, 'base_0.npz')), np.load(os.path.join(tmp, 'tree_0.npz'))
    by_size = {}
    for key in zb.files:
        what, b, _, out = key.split('/')
        size = '%s/%s/%s' % (what, b, {'chol': ('Minv64', 'Minv32', 'rank'), 'eigh': ('w', 'Z')}[what][int(out)])
        x, y = zb[key], zt[key]
        e = by_size.setdefault(size, {'identical': True, 'max_abs_diff': 0.0, 'max_rel_diff': 0.0})
        e['identical'] &= bool(np.array_equal(x, y))
        d = float(np.abs(x.astype(np.float64) - y.astype(np.float64)).max())
        e['max_abs_diff'] = max(e['max_abs_diff'], d)
        e['max_rel_diff'] = max(e['max_rel_diff'], d / max(float(np.abs(x).max()), 1e-300))
    tmin = {k: {n: min(t[n] for t in v) for n in v[0]} for k, v in times.items()}
    try:
        gpu = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                                      text=True).strip().splitlines()[0]
    except Exception as e:      # noqa: BLE001
        gpu = 'unknown (%s)' % e
    print(json.dumps({'gpu': gpu, 'outputs': by_size, 'kernel_ms_min': tmin, 'runs': times}))
    shutil.rmtree(tmp)


if __name__ == '__main__':
    main()
