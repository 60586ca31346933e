"""HOPE on an H100 -- drop-in for reference gem/embedding/hope.py:8-44.

Same class name, hyper-parameters (d, beta), method name ('hope_gsvd'), call signature
(learn_embedding(graph=None, is_weighted=False, no_python=False)), error behaviour
(ValueError('graph needed')), row order (list(graph.nodes), SURVEY F6), column layout
([U sqrt(S) | V sqrt(S)], sigma ascending) and get_edge_weight.  The arithmetic runs in
libgemb200.so (CUDA, sm_90a); there is no CPU path -- without a GPU learn_embedding raises
RuntimeError.

Extra, optional hyper-parameters (defaults keep reference call sites working unchanged):
    tol, max_iters, min_iters, oversample, katz_terms, katz_tol, seed, compute_residual, verbose,
    algorithm (0 auto / 1 general / 2 symmetric-Chebyshev), cheb_degree
        -> gemb_hope_opts (include/gemb200.h)
    device (int), dtype (np.float32 default | np.float64), strict (raise instead of warn when the solver
    stops unconverged), svd_error_probes (False: never print hope.py:38-40's 'SVD error' line; int: Hutchinson
    estimate with that many probes on graphs above 4096 nodes; default: exact, printed for n <= 4096 only)
proximity (default 'katz'), alpha: the proximity S whose top-d/2 SVD is embedded (Ou et al., KDD 2016, Table 1), with A the
    weighted adjacency in list(graph.nodes) order:
        'katz'              (I - beta A)^-1 beta A  (the reference's; beta_over_rho and multi-GPU apply to it only)
        'common_neighbors'  A A
        'adamic_adar'       A D A, D_ii = 1 / sum_j (A_ij + A_ji) (0 where that sum is 0); non-negative weights
        'rooted_pagerank'   (1 - alpha) (I - alpha P)^-1, P = D_out^-1 A (a row with out-degree 0 stays 0), 0 < alpha < 1,
                            computed as (1 - alpha) sum_{j=0..J} (alpha P)^j, J = ceil(log(katz_tol) / log(alpha)) unless
                            katz_terms is given; non-negative weights
    beta is accepted and unused outside 'katz'.  The 'SVD error' line is printed for 'katz' only.  model.stats['proximity']
    records which proximity ran.  The non-Katz proximities run on the general solver (algorithm 0 or 1), single GPU.
Multi-GPU (SPMD, one process per GPU under torchrun with torch.distributed initialised): every rank calls
learn_embedding with the same graph and receives ITS row shard of X (rows [rank*ceil(n/P), ...)); see INTEGRATION.md.
`graph` may also be a scipy.sparse matrix or a gem_b200.graph.HostCSR (rows = 0..n-1) so that
million-node inputs need not go through networkx.
"""
import contextlib

import numpy as np

from gem_b200 import _native
from gem_b200 import dist as _gd
from gem_b200.embedding.static_graph_embedding import StaticGraphEmbedding

_OPT_KEYS = ('tol', 'max_iters', 'min_iters', 'oversample', 'katz_terms', 'katz_tol', 'seed',
             'compute_residual', 'verbose', 'algorithm', 'cheb_degree', 'cheb_range_log2', 'stop_rule',
             'algorithm3_basis')


# proximity -> gemb_hope_opts.spectral_mode
PROXIMITIES = {'katz': 0, 'common_neighbors': 3, 'adamic_adar': 4, 'rooted_pagerank': 5}


def check_proximity(proximity, alpha, beta_over_rho=None, world=1, csr=None):
    """ValueError for a proximity the solver cannot run, before any device call: an unknown name; alpha missing or outside
    (0, 1) for 'rooted_pagerank', or given for another proximity; beta_over_rho or world > 1 with a proximity other than
    'katz'; a negative weight in csr for 'adamic_adar' or 'rooted_pagerank'."""
    if proximity not in PROXIMITIES:
        raise ValueError('proximity must be one of %s, not %r' % (', '.join(map(repr, PROXIMITIES)), proximity))
    if proximity == 'rooted_pagerank':
        if alpha is None or not 0.0 < float(alpha) < 1.0:
            raise ValueError("proximity='rooted_pagerank' needs alpha with 0 < alpha < 1, not %r" % (alpha,))
    elif alpha is not None:
        raise ValueError("alpha is the rooted PageRank coefficient; proximity=%r takes none" % (proximity,))
    if proximity != 'katz':
        if beta_over_rho is not None:
            raise ValueError("beta_over_rho sets the Katz beta; proximity=%r has no beta" % (proximity,))
        if world > 1:
            raise ValueError("proximity=%r is single-GPU; multi-GPU HOPE runs proximity='katz' only" % (proximity,))
        if proximity in ('adamic_adar', 'rooted_pagerank') and csr is not None and csr.data is not None \
                and bool(np.any(csr.data < 0)):
            raise ValueError('proximity=%r needs non-negative edge weights' % (proximity,))


def rooted_pagerank_operator(csr):
    """HostCSR of P = D_out^-1 A: every row divided by its weighted out-degree, a row with out-degree 0 stays zero."""
    from gem_b200 import graph as _graph
    w = np.ones(csr.nnz) if csr.data is None else csr.data
    rows = np.repeat(np.arange(csr.n, dtype=np.int64), np.diff(csr.indptr).astype(np.int64))
    out = np.bincount(rows, weights=w, minlength=csr.n)
    inv = np.where(out > 0, 1.0 / np.where(out > 0, out, 1.0), 0.0)
    return _graph.HostCSR(csr.n, csr.indptr, csr.indices, w * inv[rows], nodes=csr.nodes, symmetric=False)


_SPMD_CTX = {}     # (device, rank, world) -> _native.Context holding the process's NCCL communicator


class HOPE(StaticGraphEmbedding):

    _recon_split = True      # get_edge_weight form, for the GPU reconstruction (gemb_recon_create)

    hyper_params = {
        'method_name': 'hope_gsvd'
    }

    def __init__(self, *args, **kwargs):
        """ Initialize the HOPE class

        Args:
            d: dimension of the embedding
            beta: higher order coefficient
        """
        super(HOPE, self).__init__(*args, **kwargs)
        self.stats = None
        self._sigma = None

    def learn_embedding(self, graph=None, is_weighted=False, no_python=False, out=None, **ignored):
        csr = self._to_csr(graph)
        opts = {k: getattr(self, '_' + k) for k in _OPT_KEYS if hasattr(self, '_' + k)}
        proximity = getattr(self, '_proximity', 'katz')
        alpha = getattr(self, '_alpha', None)
        bor = getattr(self, '_beta_over_rho', None)
        dist_mod, rank, world, device = _gd.spmd(getattr(self, '_device', None))
        check_proximity(proximity, alpha, bor, world, csr)
        katz = proximity == 'katz'
        if not katz:
            opts['spectral_mode'] = PROXIMITIES[proximity]
        if world > 1:
            # SPMD: the context and its NCCL communicator are created once per process and kept (communicator set-up
            # costs 0.5-1 s -- ten times the solve); single GPU: a context is a stream + a few small buffers, made per call
            ctx = _SPMD_CTX.get((device, rank, world))
            if ctx is None:
                ctx = _native.Context(device)
                _gd.init_comm_from_torch(ctx, dist_mod, rank, world)
                _SPMD_CTX[(device, rank, world)] = ctx
            ctx_scope = contextlib.nullcontext(ctx)
        else:
            ctx_scope = _native.Context(device)
        op = rooted_pagerank_operator(csr) if proximity == 'rooted_pagerank' else csr
        with ctx_scope as ctx, self._upload(ctx, op, rank, world) as g:
            # beta_over_rho=c (extra hyper-parameter): beta = c / rho_hat(A), estimated on the device (BASELINE configs[3])
            if proximity == 'rooted_pagerank':
                beta_arg = float(alpha)                  # gemb_hope's beta carries alpha in spectral_mode 5
            else:
                beta_arg = float(self._beta) if bor is None else -float(bor)
            X, sigma, st = g.hope(int(self._d), beta_arg, out=out, **opts)
            if bor is not None:
                self._beta = float(st['beta_used'])
            self._svd_error = None
            want_err = getattr(self, '_svd_error_probes', None)
            if katz and world == 1 and (csr.n <= 4096 if want_err is None else want_err is not False):
                # hope.py:38-40.  Exact up to 4096 nodes (where the reference itself is practical); beyond that
                # only on request, as a Hutchinson estimate with svd_error_probes Rademacher vectors (SURVEY H8).
                probes = 0 if (want_err is None or want_err is True or csr.n <= 4096) else int(want_err)
                try:
                    self._svd_error = g.hope_svd_error(int(self._d), float(self._beta), X, probes)
                    print('SVD error (low rank): %f' % self._svd_error)
                except RuntimeError as exc:        # e.g. beta*||A||_2 >= 1: the reference would print inv()'s answer
                    print('SVD error (low rank): unavailable (%s)' % exc)
        st['proximity'] = proximity
        self.stats = st
        self._sigma = sigma
        # the measure the solver stopped on: algorithm 3 always stops on its residual estimate
        measure = ('residual estimate %.3g' % st['resid_est'] if opts.get('stop_rule', 0) == 1 or st.get('algorithm') == 3 else
                   'singular values still moving by %.3g relative per round' % st['ritz_change'])
        self._check_converged(st, 'HOPE: the solver stopped at max_iters=%d without meeting tol=%g (%s); the embedding is '
                              'less accurate than requested -- raise max_iters / oversample%s'
                              % (st['iters'], opts.get('tol', 1e-6), measure,
                                 ' or use algorithm=3 on power-law graphs' if katz else ''))
        self._result(X, csr.n)
        if getattr(self, '_verbose', 0):
            print('HOPE: algorithm %d, %d iterations, J=%d Katz terms, block %d, ritz change %.3g, converged %d' %
                  (st['algorithm'], st['iters'], st['katz_terms'], st['block'], st['ritz_change'], st['converged']))
        return self._X

    def _upload(self, ctx, csr, rank, world):
        """The graph on the device: under SPMD (INTEGRATION.md C) every rank is called with the same graph, uploads
        its row shard and returns THIS rank's rows of X; a general (non-symmetric) graph also uploads its transpose, and
        so does rooted PageRank's P (symmetric=False) always."""
        if world == 1:
            if csr.is_symmetric():
                return _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, csr.data_f32())
            t = csr.transpose()
            return _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, csr.data_f32(),
                                       t.indptr, t.indices, t.data_f32())
        r0, ip, ix, dat = csr.row_shard(rank, world)
        self._row0 = r0
        dat = None if dat is None else dat.astype(np.float32)
        if csr.is_symmetric():
            return _native.DeviceGraph(ctx, csr.n, ip, ix, dat, row0=r0)
        _, tp, tx, tdat = csr.transpose().row_shard(rank, world)
        return _native.DeviceGraph(ctx, csr.n, ip, ix, dat, tp, tx, None if tdat is None else tdat.astype(np.float32),
                                   row0=r0)

    def get_edge_weight(self, i, j):
        return np.dot(self._X[i, :self._d // 2], self._X[j, self._d // 2:])
