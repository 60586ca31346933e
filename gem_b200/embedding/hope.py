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
        dist_mod, rank, world, device = _gd.spmd(getattr(self, '_device', None))
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
        with ctx_scope as ctx, self._upload(ctx, csr, rank, world) as g:
            # beta_over_rho=c (extra hyper-parameter): beta = c / rho_hat(A), estimated on the device (BASELINE configs[3])
            bor = getattr(self, '_beta_over_rho', None)
            beta_arg = float(self._beta) if bor is None else -float(bor)
            X, sigma, st = g.hope(int(self._d), beta_arg, out=out, **opts)
            if bor is not None:
                self._beta = float(st['beta_used'])
            self._svd_error = None
            want_err = getattr(self, '_svd_error_probes', None)
            if world == 1 and (csr.n <= 4096 if want_err is None else want_err is not False):
                # hope.py:38-40.  Exact up to 4096 nodes (where the reference itself is practical); beyond that
                # only on request, as a Hutchinson estimate with svd_error_probes Rademacher vectors (SURVEY H8).
                probes = 0 if (want_err is None or want_err is True or csr.n <= 4096) else int(want_err)
                try:
                    self._svd_error = g.hope_svd_error(int(self._d), float(self._beta), X, probes)
                    print('SVD error (low rank): %f' % self._svd_error)
                except RuntimeError as exc:        # e.g. beta*||A||_2 >= 1: the reference would print inv()'s answer
                    print('SVD error (low rank): unavailable (%s)' % exc)
        self.stats = st
        self._sigma = sigma
        self._check_converged(st, 'HOPE: the solver stopped at max_iters=%d without meeting tol=%g (singular values still '
                              'moving by %.3g per round); the embedding is less accurate than requested -- raise max_iters / '
                              'oversample or use algorithm=3 on power-law graphs'
                              % (st['iters'], opts.get('tol', 1e-6), st['ritz_change']))
        self._result(X, csr.n)
        if getattr(self, '_verbose', 0):
            print('HOPE: algorithm %d, %d iterations, J=%d Katz terms, block %d, ritz change %.3g, converged %d' %
                  (st['algorithm'], st['iters'], st['katz_terms'], st['block'], st['ritz_change'], st['converged']))
        return self._X

    def _upload(self, ctx, csr, rank, world):
        """The graph on the device: under SPMD (INTEGRATION.md C) every rank is called with the same graph, uploads
        its row shard and returns THIS rank's rows of X; a general (non-symmetric) graph also uploads its transpose."""
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
