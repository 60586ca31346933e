"""scripts/bench_recon_blocks.py -- graph reconstruction and link prediction on graphs whose n x n reconstruction does
not fit in device memory (the handle regenerates it in column blocks, gemb_recon_create).

    python scripts/bench_recon_blocks.py --out DIR [--n 1000000] [--cmp-n 100000] [--max-k 1000]

Three workloads on one GPU:
  recon     the BASELINE SBM (--n nodes, 1000-node blocks, seed 42), HOPE d = 128 at bench.HOPE_SOLVER, then
            evaluateStaticGraphReconstruction(max_k) on every node
  linkpred  evaluateStaticLinkPrediction(train_ratio 0.8, n_sample_nodes None, max_k, seed 42) of the same graph
  compare   an SBM of --cmp-n nodes (HOPE d = 128), where the whole matrix fits: ranks, n_pred_row and top(max_k) of the
            kept matrix against 64 panels per block, bit for bit, and both times
For the public calls, every call on the reconstruction handle is timed on the host clock (each ends in a device
synchronise): create, exclude, ranks, top's count and top's entries, with its passes over the matrix (launches of
the call // panels: a pass issues one product launch per panel).  MAP is reported with its bits, with precision@100
and @max_k.  The card's name and power limit are read in the same run.  Writes DIR/bench_recon_blocks.json and prints
it as one line.  Needs a GPU; nothing falls back.
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'scripts'))

from bench_linkpred import card  # noqa: E402


def timed_handle(log):
    """A Reconstruction whose calls append {call, ms, passes} to log (installed as _native.Reconstruction)."""
    from gem_b200 import _native
    lib, base = _native.lib(), _native.Reconstruction

    def run(name, panels, f):
        l0 = lib.gemb_launch_count()
        t0 = time.perf_counter()
        out = f()
        log.append({'call': name, 'ms': (time.perf_counter() - t0) * 1e3,
                    'passes': int((lib.gemb_launch_count() - l0) // panels)})
        return out

    class Timed(base):
        def __init__(self, ctx, X, kind, panels_per_block=0):
            panels = (X.shape[0] + 63) // 64
            run('create', panels, lambda: base.__init__(self, ctx, X, kind, panels_per_block))
            log[-1].update(panels_per_block=self.panels_per_block, blocks=self.blocks)
            self._panels = panels

        def exclude(self, indptr, indices):
            return run('exclude', self._panels, lambda: super(Timed, self).exclude(indptr, indices))

        def ranks(self, indptr, indices, is_undirected):
            return run('ranks', self._panels, lambda: super(Timed, self).ranks(indptr, indices, is_undirected))

        def top(self, is_undirected, max_k=-1):
            m = ctypes.c_int64(0)
            run('top_count', self._panels, lambda: _native.check(lib.gemb_recon_top(
                self._h, int(bool(is_undirected)), int(max_k), 0, None, None, None, ctypes.byref(m))))
            return run('top_entries', self._panels, lambda: super(Timed, self).top(is_undirected, max_k))
    return Timed


def learn(csr, d, beta):
    from bench import HOPE_SOLVER
    from gem_b200.embedding.hope import HOPE
    HOPE.hyper_params.clear(); HOPE.hyper_params.update({'method_name': 'hope_gsvd'})
    model = HOPE(d=d, beta=beta, **HOPE_SOLVER)
    t0 = time.perf_counter()
    X = model.learn_embedding(graph=csr)
    return model, X, time.perf_counter() - t0


def with_timed(f):
    from gem_b200 import _native
    log, base = [], _native.Reconstruction
    _native.Reconstruction = timed_handle(log)
    try:
        t0 = time.perf_counter()
        out = f()
        return out, log, time.perf_counter() - t0
    finally:
        _native.Reconstruction = base


def curve(MAP, prec, max_k):
    return {'MAP': MAP, 'MAP_hex': float(MAP).hex(), 'prec_at_100': prec[99] if len(prec) >= 100 else None,
            'prec_at_max_k': prec[max_k - 1] if len(prec) >= max_k else None}


def compare(n, d, beta, max_k):
    from gem_b200 import _native, synth
    from gem_b200.evaluation.evaluate_graph_reconstruction import _true_csr
    csr = synth.sbm(n=n, block=1000, seed=42)
    _, X, _ = learn(csr, d, beta)
    indptr, indices = _true_csr(csr, n)
    out, res = [], {'n': n, 'nnz': csr.nnz}
    with _native.Context(0) as ctx:
        for tag, ppb in (('resident', 0), ('blocked', 64)):
            log = []
            rec = timed_handle(log)(ctx, X, _native.RECON_SPLIT, ppb)
            ranks, npr = rec.ranks(indptr, indices, True)
            i, j, w = rec.top(True, max_k)
            rec.free()
            o = np.argsort(i.astype(np.int64) * n + j)
            out.append((ranks, npr, i[o], j[o], w[o].view(np.uint32)))
            res[tag] = log
    res['identical'] = {k: bool(np.array_equal(a, b)) for k, a, b in zip(('ranks', 'n_pred_row', 'top_i', 'top_j', 'top_w'),
                                                                          *out)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--n', type=int, default=1_000_000)
    ap.add_argument('--cmp-n', type=int, default=100_000)
    ap.add_argument('--max-k', type=int, default=1000)
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--beta', type=float, default=0.01)
    args = ap.parse_args()
    from gem_b200 import synth
    from gem_b200.evaluation.evaluate_graph_reconstruction import evaluateStaticGraphReconstruction
    from gem_b200.evaluation.evaluate_link_prediction import evaluateStaticLinkPrediction
    os.makedirs(args.out, exist_ok=True)
    res = {'metric': 'reconstruction_in_blocks', 'card': card()}
    res['compare'] = compare(args.cmp_n, args.d, args.beta, args.max_k)
    csr = synth.sbm(n=args.n, block=1000, seed=42)
    model, X, learn_s = learn(csr, args.d, args.beta)
    (MAP, prec, _, _), log, wall = with_timed(lambda: evaluateStaticGraphReconstruction(csr, model, X, None,
                                                                                        max_k=args.max_k))
    res['recon'] = dict(n=csr.n, nnz=csr.nnz, learn_s=learn_s, eval_s=wall, calls=log, **curve(MAP, prec, args.max_k))
    (MAP, prec), log, wall = with_timed(lambda: evaluateStaticLinkPrediction(csr, model, train_ratio=0.8, n_sample_nodes=None,
                                                                             max_k=args.max_k, seed=42))
    res['linkpred'] = dict(n=csr.n, eval_s=wall, calls=log, **curve(MAP, prec, args.max_k))
    with open(os.path.join(args.out, 'bench_recon_blocks.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
