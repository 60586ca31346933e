"""Records tests/golden/hope_setup.npz: what gemb_hope, gemb_hope_apply and gemb_hope_svd_error return on every path of
HOPE's set-up (the beta a solve runs with, its Katz terms and what bounds A's spectrum), for tests/test_gpu_hope_setup.py.
Each case stores a row sample of X, sigma, the stats fields that are not timings and the gemb_launch_count() delta of
the call; each refusal its status, message and launch delta.  Needs an H100; the file in the repository was recorded on
an H100 80GB HBM3 (700 W power limit) from the build that decided the set-up inline in gemb_hope, before hope_setup
existed.

    python tests/golden/make_golden_hope_setup.py [OUT.npz]
"""
import os
import re
import sys

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'oracle'))

STATS = ['iters', 'converged', 'algorithm', 'katz_terms', 'spmm_count', 'norm2_A', 'beta_used', 'resid_est', 'resid_max',
         'ritz_change']
ROWS = 64
FAST = dict(tol=1e-6, max_iters=6, oversample=8)


def _f32(A):
    A = sp.csr_matrix(A, dtype=np.float32).astype(np.float64)
    A.sort_indices()
    return A


_GRAPHS = {}


def graph(name):
    """(A in fp64, symmetric upload?) -- cached."""
    if name in _GRAPHS:
        return _GRAPHS[name]
    import proximity_oracle as po
    if name == 'digraph':                 # po.random_digraph: rho(A) = 13.47, ||A||_2 = 15.22
        out = (_f32(po.random_digraph()), False)
    elif name == 'digraph_P':
        out = (_f32(po.transition(po.random_digraph())), False)
    elif name in ('sbm1024', 'sbm1024_signed'):
        z = np.load(os.path.join(HERE, 'sbm1024.npz'))
        n = z['nodes'].shape[0]
        A = sp.csr_matrix((np.ones(z['src'].shape[0]), (z['src'], z['dst'])), shape=(n, n))
        A = ((A + A.T) > 0).astype(np.float64)
        A.setdiag(0)
        A.eliminate_zeros()
        if name == 'sbm1024_signed':      # weights +-U[0.5, 1.5], w_ij = w_ji: rowsum_bound sees negative weights
            U = sp.triu(A, 1).tocoo()
            rng = np.random.default_rng(5)
            w = rng.uniform(0.5, 1.5, U.nnz) * rng.choice([-1.0, 1.0], U.nnz)
            U = sp.csr_matrix((w, (U.row, U.col)), shape=A.shape)
            A = U + U.T
        out = (_f32(A), True)
    elif name == 'rmat12':
        from gem_b200 import synth
        out = (_f32(synth.rmat(scale=12, edge_factor=8, seed=3).to_scipy()), True)
    elif name == 'randw120_P':            # LLE's P = D^-1 W of the randw120 fixture, uploaded with its transpose
        import proximity_oracle as po
        z = np.load(os.path.join(HERE, 'ref_lle_randw120_d8.npz'))
        e, n = z['edges'], int(z['n'])
        W = sp.csr_matrix((e[:, 2], (e[:, 0].astype(int), e[:, 1].astype(int))), shape=(n, n))
        out = (_f32(po.transition(W)), False)
    elif name == 'empty':
        out = (sp.csr_matrix((300, 300)), True)
    else:
        raise ValueError(name)
    _GRAPHS[name] = out
    return out


def upload(ctx, name):
    from gem_b200 import _native
    A, sym = graph(name)
    data = None if np.all(A.data == 1.0) else A.data.astype(np.float32)
    if sym:
        return _native.DeviceGraph(ctx, A.shape[0], A.indptr, A.indices, data)
    T = A.T.tocsr()
    T.sort_indices()
    tdata = None if data is None else T.data.astype(np.float32)
    return _native.DeviceGraph(ctx, A.shape[0], A.indptr, A.indices, data, T.indptr, T.indices, tdata)


def _launches():
    from gem_b200 import _native
    return int(_native.lib().gemb_launch_count())


# name -> (graph, d, beta, opts) of one gemb_hope call
SOLVES = {
    # spectral_mode 0, beta > 0
    'a1_norm': ('digraph', 8, 0.02, dict(algorithm=1)),
    'a1_katz_terms': ('digraph', 8, 0.02, dict(algorithm=1, katz_terms=7)),
    'a1_probe': ('digraph', 8, 0.07, dict(algorithm=1)),                 # beta ||A||_2 = 1.07, beta rho = 0.94
    'a1_residual': ('digraph', 8, 0.02, dict(algorithm=1, compute_residual=1)),
    'a1_stop_rule1': ('digraph', 8, 0.02, dict(algorithm=1, stop_rule=1)),
    'a2_ritz': ('sbm1024', 16, 0.01, dict(algorithm=2)),
    'a2_ritz_residual': ('sbm1024', 16, 0.01, dict(algorithm=2, compute_residual=1)),
    'a2_ritz_stop_rule1': ('sbm1024', 16, 0.01, dict(algorithm=2, stop_rule=1)),
    'a2_power': ('sbm1024_signed', 16, 0.02, dict(algorithm=2)),
    'a2_power_residual': ('sbm1024_signed', 16, 0.02, dict(algorithm=2, compute_residual=1)),
    'a3_ritz': ('rmat12', 16, 0.001, dict(algorithm=3)),                  # beta ||A||_inf = 0.93
    'a0_lanczos_switch': ('rmat12', 16, 0.005, dict(algorithm=0)),        # beta ||A||_2 = 0.48, beta ||A||_inf = 4.6
    # spectral_mode 0, beta < 0: |beta| / ||A||_2
    'neg_a1': ('digraph', 8, -0.5, dict(algorithm=1)),
    'neg_a1_katz_terms': ('digraph', 8, -0.5, dict(algorithm=1, katz_terms=9)),
    'neg_a2_ritz': ('sbm1024', 16, -0.5, dict(algorithm=2)),
    'neg_a2_power': ('sbm1024_signed', 16, -0.5, dict(algorithm=2, compute_residual=1)),
    'neg_a3': ('rmat12', 16, -0.5, dict(algorithm=3)),
    # spectral_modes 1-5
    'm1_ritz': ('sbm1024', 8, 0.0, dict(spectral_mode=1)),
    'm1_power': ('sbm1024_signed', 8, 0.0, dict(spectral_mode=1, stop_rule=1)),
    'm2_randw120': ('randw120_P', 8, 0.0, dict(spectral_mode=2)),
    'm3': ('digraph', 8, 0.0, dict(spectral_mode=3, compute_residual=1)),
    'm4': ('digraph', 8, 0.0, dict(spectral_mode=4)),
    'm5': ('digraph_P', 8, 0.5, dict(spectral_mode=5, compute_residual=1)),
    'm5_katz_terms': ('digraph_P', 8, 0.5, dict(spectral_mode=5, katz_terms=6)),
}

# name -> (graph, d, beta, opts, expected text of the refusal)
REFUSALS = {
    'divergent_symmetric': ('sbm1024', 16, 1.0, dict(algorithm=2), 'does not converge'),
    'divergent_directed': ('digraph', 8, 0.1, dict(algorithm=1), 'does not converge'),   # beta rho = 1.35: the probe
    'relative_beta_098': ('digraph', 8, -0.99, dict(algorithm=1), 'outside the Katz convergence radius'),
    'relative_beta_empty': ('empty', 8, -0.5, dict(algorithm=2), 'empty graph'),
}

# name -> (graph, d, beta)
SVD_ERRORS = {'svd_symmetric': ('sbm1024', 8, 0.01), 'svd_directed': ('digraph', 8, 0.07)}

# spectral_mode -> (graph, beta, opts) of one gemb_hope_apply call, S X and S^T X
APPLIES = {0: ('digraph', 0.02, dict(katz_terms=5)), 1: ('sbm1024', 0.0, {}), 2: ('randw120_P', 0.0, {}),
           3: ('digraph', 0.0, {}), 4: ('digraph', 0.0, {}), 5: ('digraph_P', 0.5, {})}


def solve_case(ctx, name):
    gname, d, beta, opts = SOLVES[name]
    n = graph(gname)[0].shape[0]
    with upload(ctx, gname) as g:
        l0 = _launches()
        X, sig, st = g.hope(d, beta, **dict(FAST, **opts))
        launches = _launches() - l0
    rows = np.sort(np.random.default_rng(11).choice(n, min(n, ROWS), replace=False))
    out = dict(X=X[rows], sigma=sig, launches=np.int64(launches))
    for f in STATS:
        out[f] = np.asarray(st[f], dtype=np.float32 if isinstance(st[f], float) else np.int64)
    return out


def refusal_case(ctx, name):
    gname, d, beta, opts, _ = REFUSALS[name]
    with upload(ctx, gname) as g:
        l0 = _launches()
        try:
            g.hope(d, beta, **dict(FAST, **opts))
            msg = 'accepted'
        except RuntimeError as e:
            msg = str(e)
        launches = _launches() - l0
    m = re.match(r'libgemb200 error (-?\d+): (.*)', msg, re.S)
    status, text = (int(m.group(1)), m.group(2)) if m else (0, msg)
    return dict(status=np.int64(status), message=np.array(text), launches=np.int64(launches))


def svd_error_case(ctx, name):
    gname, d, beta = SVD_ERRORS[name]
    n = graph(gname)[0].shape[0]
    X = np.random.default_rng(d).standard_normal((n, d)).astype(np.float32)
    with upload(ctx, gname) as g:
        l0 = _launches()
        err = g.hope_svd_error(d, beta, X)
        launches = _launches() - l0
    return dict(err=np.float64(err), launches=np.int64(launches))


def apply_case(ctx, mode):
    gname, beta, opts = APPLIES[mode]
    n = graph(gname)[0].shape[0]
    X = np.random.default_rng(mode).standard_normal((n, 8)).astype(np.float32)
    out = {}
    with upload(ctx, gname) as g:
        for t in (False, True):
            l0 = _launches()
            Y, J = g.hope_apply(X, beta, transpose=t, spectral_mode=mode, **opts)
            out.update({'Y%d' % t: Y, 'J%d' % t: np.int64(J), 'launches%d' % t: np.int64(_launches() - l0)})
    return out


def all_cases():
    """(kind, name) of every case, in recording order."""
    return ([('solve', k) for k in SOLVES] + [('refusal', k) for k in REFUSALS] + [('svd_error', k) for k in SVD_ERRORS] +
            [('apply', k) for k in APPLIES])


def run(ctx, kind, name):
    return {'solve': solve_case, 'refusal': refusal_case, 'svd_error': svd_error_case, 'apply': apply_case}[kind](ctx, name)


def main():
    from gem_b200 import _native
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, 'hope_setup.npz')
    ctx = _native.Context(0)
    rec = {}
    for kind, name in all_cases():
        r = run(ctx, kind, name)
        rec.update({'%s/%s/%s' % (kind, name, k): v for k, v in r.items()})
        brief = {k: (v.item() if np.ndim(v) == 0 else np.shape(v)) for k, v in r.items()}
        print('%-9s %-20s %s' % (kind, name, brief))
    ctx.close()
    np.savez_compressed(out, **rec)
    print('wrote %s: %d cases' % (out, len(all_cases())))


if __name__ == '__main__':
    main()
