"""gem_b200/_native.py -- ctypes binding of libgemb200.so (the C ABI in include/gemb200.h).

There is no CPU fallback: if the shared object is missing or no CUDA device is visible, every
compute call raises RuntimeError.  Nothing here imports oracle/.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libgemb200.so')
_lib = None

UNIQUE_ID_BYTES = 128

EXPORTS = [
    'gemb_version', 'gemb_last_error', 'gemb_device_count', 'gemb_launch_count', 'gemb_ctx_create', 'gemb_ctx_destroy',
    'gemb_host_alloc', 'gemb_host_free', 'gemb_mem_trim', 'gemb_mem_cached_bytes', 'gemb_mem_live_blocks', 'gemb_comm_unique_id', 'gemb_comm_init', 'gemb_graph_upload',
    'gemb_graph_free', 'gemb_spmm', 'gemb_spmm4', 'gemb_gram', 'gemb_apply', 'gemb_chol_inverse', 'gemb_eigh', 'gemb_hope', 'gemb_hope_svd_error', 'gemb_n2v_alias', 'gemb_n2v_walks', 'gemb_node2vec',
    'gemb_edge_list_scan', 'gemb_edge_list_parse', 'gemb_edge_list_write', 'gemb_emb_read', 'gemb_emb_write',
    'gemb_synth_rmat', 'gemb_gf', 'gemb_recon_create', 'gemb_recon_free', 'gemb_recon_dense', 'gemb_recon_pairs', 'gemb_recon_ranks', 'gemb_recon_top',
    'gemb_recon_exclude', 'gemb_nc_fit', 'gemb_nc_topk', 'gemb_cc_create', 'gemb_cc_info', 'gemb_cc_labels', 'gemb_cc_lcc',
    'gemb_cc_times', 'gemb_cc_free',
]


class _Stats(ctypes.Structure):
    """Base of the statistics structs the library fills in."""

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if k != 'struct_size'}


class HopeOpts(ctypes.Structure):
    _fields_ = [('struct_size', ctypes.c_uint32), ('oversample', ctypes.c_int32),
                ('max_iters', ctypes.c_int32), ('min_iters', ctypes.c_int32), ('tol', ctypes.c_float),
                ('katz_terms', ctypes.c_int32), ('katz_tol', ctypes.c_float), ('seed', ctypes.c_uint64),
                ('compute_residual', ctypes.c_int32), ('verbose', ctypes.c_int32),
                ('algorithm', ctypes.c_int32), ('cheb_degree', ctypes.c_int32), ('cheb_range_log2', ctypes.c_float),
                ('stop_rule', ctypes.c_int32), ('algorithm3_basis', ctypes.c_int32), ('spectral_mode', ctypes.c_int32)]


class HopeStats(_Stats):
    _fields_ = [('struct_size', ctypes.c_uint32), ('iters', ctypes.c_int32), ('katz_terms', ctypes.c_int32),
                ('block', ctypes.c_int32), ('converged', ctypes.c_int32), ('algorithm', ctypes.c_int32),
                ('spmm_count', ctypes.c_int64),
                ('spmm_ms', ctypes.c_double), ('spmm_bytes', ctypes.c_double), ('dense_ms', ctypes.c_double),
                ('comm_ms', ctypes.c_double), ('total_ms', ctypes.c_double), ('h2d_ms', ctypes.c_double),
                ('d2h_ms', ctypes.c_double), ('norm2_A', ctypes.c_float), ('ritz_change', ctypes.c_float),
                ('resid_max', ctypes.c_float), ('resid_est', ctypes.c_float), ('mg_mode', ctypes.c_int32),
                ('halo_rows', ctypes.c_int64), ('push_rows', ctypes.c_int64), ('pushes', ctypes.c_int64),
                ('beta_used', ctypes.c_float), ('push_bytes', ctypes.c_double)]


class N2VStats(_Stats):
    _fields_ = [('struct_size', ctypes.c_uint32), ('alias_ms', ctypes.c_double), ('shuffle_ms', ctypes.c_double),
                ('walk_ms', ctypes.c_double), ('vocab_ms', ctypes.c_double), ('sgns_ms', ctypes.c_double),
                ('total_ms', ctypes.c_double), ('h2d_ms', ctypes.c_double), ('d2h_ms', ctypes.c_double),
                ('comm_ms', ctypes.c_double), ('n_tokens', ctypes.c_int64), ('n_walks', ctypes.c_int64),
                ('pairs', ctypes.c_int64), ('sgns_bytes', ctypes.c_double), ('walk_bytes', ctypes.c_double)]


class NCStats(_Stats):
    _fields_ = [('struct_size', ctypes.c_uint32), ('panels', ctypes.c_int32), ('evaluations', ctypes.c_int64),
                ('max_iters', ctypes.c_int32), ('unconverged', ctypes.c_int64), ('constant', ctypes.c_int64),
                ('eval_bytes', ctypes.c_double), ('total_ms', ctypes.c_double)]


NC_CONVERGED, NC_CONSTANT, NC_MAXITER, NC_STALLED = 1, 2, 3, 4


def lib():
    """Load libgemb200.so (once).  Raises RuntimeError loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError('gem_b200: %s is missing -- build it with `python -m gem_b200.build` '
                           '(there is no CPU fallback)' % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    vp, i32, i64, f32, f64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_double
    L.gemb_version.restype = ctypes.c_int
    L.gemb_last_error.restype = ctypes.c_char_p
    L.gemb_device_count.restype = ctypes.c_int
    L.gemb_launch_count.restype = ctypes.c_int64
    L.gemb_ctx_create.argtypes = [ctypes.c_int, ctypes.POINTER(vp)]
    L.gemb_ctx_destroy.argtypes = [vp]
    L.gemb_host_alloc.argtypes = [ctypes.c_size_t, ctypes.POINTER(vp)]
    L.gemb_host_free.argtypes = [vp]
    L.gemb_mem_trim.argtypes = []
    L.gemb_mem_cached_bytes.argtypes = []
    L.gemb_mem_cached_bytes.restype = ctypes.c_size_t
    L.gemb_mem_live_blocks.argtypes = []
    L.gemb_mem_live_blocks.restype = ctypes.c_size_t
    L.gemb_comm_unique_id.argtypes = [vp]
    L.gemb_comm_init.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp]
    L.gemb_graph_upload.argtypes = [vp, i64, i64, i64, vp, vp, vp, vp, vp, vp, ctypes.POINTER(vp)]
    L.gemb_graph_free.argtypes = [vp]
    L.gemb_spmm.argtypes = [vp, ctypes.c_int, ctypes.c_int, f32, vp, f32, vp, f32, vp, vp]
    L.gemb_spmm4.argtypes = [vp, ctypes.c_int, ctypes.c_int, f32, vp, f32, vp, f32, vp, f32, vp, vp]
    L.gemb_gram.argtypes = [vp, i64, vp, ctypes.c_int, vp, ctypes.c_int, ctypes.c_int, vp]
    L.gemb_apply.argtypes = [vp, i64, vp, ctypes.c_int, vp, ctypes.c_int, ctypes.c_int, vp]
    L.gemb_chol_inverse.argtypes = [vp, ctypes.c_int, vp, vp, vp, ctypes.POINTER(ctypes.c_int)]
    L.gemb_eigh.argtypes = [vp, ctypes.c_int, vp, f64, vp, vp]
    L.gemb_hope.argtypes = [vp, ctypes.c_int, f32, ctypes.POINTER(HopeOpts), vp, vp, ctypes.POINTER(HopeStats)]
    L.gemb_hope_svd_error.argtypes = [vp, ctypes.c_int, f32, vp, ctypes.c_int, ctypes.c_uint64, ctypes.POINTER(f64)]
    L.gemb_n2v_alias.argtypes = [vp, vp, vp, vp]
    L.gemb_n2v_walks.argtypes = [vp, vp, vp, i64, ctypes.c_int, ctypes.c_int, f64, f64, i32, i64, i64, vp,
                                 ctypes.POINTER(N2VStats)]
    L.gemb_node2vec.argtypes = [vp, vp, vp, i64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                ctypes.c_int, f64, f64, i32, ctypes.c_int, i64, vp, ctypes.POINTER(N2VStats)]
    for name in EXPORTS:
        getattr(L, name)  # AttributeError here = header/library mismatch
    cp = ctypes.c_char_p
    L.gemb_edge_list_scan.argtypes = [cp, i64, ctypes.POINTER(i64)]
    L.gemb_edge_list_parse.argtypes = [cp, i64, i64, vp, vp, vp, ctypes.POINTER(i32)]
    L.gemb_edge_list_write.argtypes = [cp, i64, vp, vp, vp, i64]
    L.gemb_emb_read.argtypes = [cp, ctypes.POINTER(i64), ctypes.POINTER(i32), vp]
    L.gemb_emb_write.argtypes = [cp, i64, vp, i32, vp, i64]
    L.gemb_synth_rmat.argtypes = [vp, ctypes.c_int, ctypes.c_int, f64, f64, f64, ctypes.c_uint64, ctypes.c_int, i64, i64,
                                  ctypes.POINTER(i64), ctypes.POINTER(i64), vp, vp, i64]
    L.gemb_gf.argtypes = [vp, i64, i64, vp, vp, vp, ctypes.c_int, f32, f32, ctypes.c_int, ctypes.c_int, vp, vp, ctypes.POINTER(f64)]
    L.gemb_recon_create.argtypes = [vp, vp, i64, ctypes.c_int, ctypes.c_int, ctypes.POINTER(vp)]
    L.gemb_recon_free.argtypes = [vp]
    L.gemb_recon_dense.argtypes = [vp, vp]
    L.gemb_recon_pairs.argtypes = [vp, vp, vp, i64, vp]
    L.gemb_recon_ranks.argtypes = [vp, vp, vp, ctypes.c_int, vp, vp]
    L.gemb_recon_top.argtypes = [vp, ctypes.c_int, i64, i64, vp, vp, vp, ctypes.POINTER(i64)]
    L.gemb_recon_exclude.argtypes = [vp, vp, vp]
    L.gemb_nc_fit.argtypes = [vp, i64, ctypes.c_int, vp, vp, vp, ctypes.c_int, f64, f64, ctypes.c_int, vp, vp, vp,
                              ctypes.POINTER(NCStats)]
    L.gemb_nc_topk.argtypes = [vp, i64, ctypes.c_int, vp, ctypes.c_int, vp, vp, vp]
    L.gemb_cc_create.argtypes = [vp, i64, vp, vp, ctypes.POINTER(vp)]
    L.gemb_cc_info.argtypes = [vp] + [ctypes.POINTER(i64)] * 4
    L.gemb_cc_labels.argtypes = [vp, vp]
    L.gemb_cc_lcc.argtypes = [vp, vp, vp, vp, vp, vp]
    L.gemb_cc_times.argtypes = [vp, ctypes.POINTER(f64), ctypes.POINTER(f64)]
    L.gemb_cc_free.argtypes = [vp]
    _lib = L
    return L


def check(status):
    if status != 0:
        msg = lib().gemb_last_error().decode('utf-8', 'replace')
        raise RuntimeError('libgemb200 error %d: %s' % (status, msg))


def _ptr(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


class PinnedArray(np.ndarray):
    """numpy view over cudaHostAlloc memory (freed when the owner dies)."""


class _PinnedOwner:
    def __init__(self, nbytes):
        p = ctypes.c_void_p()
        check(lib().gemb_host_alloc(nbytes, ctypes.byref(p)))
        self.ptr = p.value
        self.nbytes = nbytes

    def __del__(self):
        try:
            if self.ptr:
                lib().gemb_host_free(ctypes.c_void_p(self.ptr))
        except Exception:
            pass


def pinned_empty(shape, dtype):
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) if np.ndim(shape) else int(shape)
    owner = _PinnedOwner(max(1, n * dtype.itemsize))
    buf = (ctypes.c_char * owner.nbytes).from_address(owner.ptr)
    buf._owner = owner          # `buf` is the ultimate .base of every view: the allocation lives as long as any of them
    arr = np.frombuffer(buf, dtype=dtype, count=n).reshape(shape)
    return arr.view(PinnedArray)


def mem_trim():
    """Return the cached device work buffers to the driver (gemb_mem_trim)."""
    check(lib().gemb_mem_trim())


def mem_cached_bytes():
    return int(lib().gemb_mem_cached_bytes())


def mem_live_blocks():
    """Device blocks handed out by the block cache and not yet released (gemb_mem_live_blocks)."""
    return int(lib().gemb_mem_live_blocks())


class _Handle:
    """An opaque library handle `_h`, released once by `_destroy` (the gemb_* function that frees it): explicitly, at
    the end of a `with` block, or when the object is collected."""

    def _release(self):
        if self._h:
            getattr(lib(), self._destroy)(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self._release()

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass


class Context(_Handle):
    """One CUDA device (+ optional NCCL communicator)."""
    _destroy = 'gemb_ctx_destroy'

    def __init__(self, device=0):
        self._h = ctypes.c_void_p()
        check(lib().gemb_ctx_create(int(device), ctypes.byref(self._h)))
        self.device = int(device)
        self.rank, self.nranks = 0, 1

    def comm_init(self, rank, nranks, unique_id):
        buf = ctypes.create_string_buffer(bytes(unique_id), UNIQUE_ID_BYTES)
        check(lib().gemb_comm_init(self._h, int(rank), int(nranks), buf))
        self.rank, self.nranks = int(rank), int(nranks)

    def gram(self, P, Q=None, tensor_cores=True):
        """G = P^T Q (fp64) through the device kernels (test hook)."""
        P = np.ascontiguousarray(P, dtype=np.float32)
        Qc = None if Q is None else np.ascontiguousarray(Q, dtype=np.float32)
        b1, b2 = P.shape[1], (P.shape[1] if Qc is None else Qc.shape[1])
        G = np.empty((b1, b2), dtype=np.float64)
        check(lib().gemb_gram(self._h, P.shape[0], _ptr(P), b1, _ptr(Qc), b2, int(bool(tensor_cores)), _ptr(G)))
        return G

    def apply(self, Q, M, tensor_cores=True):
        """Out = Q @ M through the device kernels (test hook)."""
        Q = np.ascontiguousarray(Q, dtype=np.float32)
        M = np.ascontiguousarray(M, dtype=np.float32)
        out = np.empty((Q.shape[0], M.shape[1]), dtype=np.float32)
        check(lib().gemb_apply(self._h, Q.shape[0], _ptr(Q), Q.shape[1], _ptr(M), M.shape[1], int(bool(tensor_cores)), _ptr(out)))
        return out

    def chol_inverse(self, G):
        """(Minv fp64, Minv fp32, rank): R^-1 of G = R^T R with the rank test of CholeskyQR (test hook)."""
        G = np.ascontiguousarray(G, dtype=np.float64)
        b = G.shape[0]
        assert G.shape == (b, b)
        M64 = np.empty((b, b), dtype=np.float64)
        M32 = np.empty((b, b), dtype=np.float32)
        rank = ctypes.c_int(-1)
        check(lib().gemb_chol_inverse(self._h, b, _ptr(G), _ptr(M64), _ptr(M32), ctypes.byref(rank)))
        return M64, M32, int(rank.value)

    def eigh(self, G, rel_tol=1e-13):
        """(w ascending, Z) of the symmetric G by the device Jacobi solver (test hook)."""
        G = np.ascontiguousarray(G, dtype=np.float64)
        b = G.shape[0]
        assert G.shape == (b, b)
        w = np.empty(b, dtype=np.float64)
        Z = np.empty((b, b), dtype=np.float64)
        check(lib().gemb_eigh(self._h, b, _ptr(G), float(rel_tol), _ptr(w), _ptr(Z)))
        return w, Z

    close = _Handle._release


def synth_rmat(ctx, scale, edge_factor=8, a=0.57, b=0.19, c=0.19, seed=42, permute=True, row0=0, n_rows=-1):
    """Device R-MAT generator (gemb_synth_rmat): (indptr int64 shard-local, indices int32 global ids, nnz of the whole graph)
    of rows [row0, row0 + n_rows) -- all rows when n_rows < 0."""
    nnz, tot = ctypes.c_int64(0), ctypes.c_int64(0)
    args = (ctx._h, int(scale), int(edge_factor), float(a), float(b), float(c), int(seed), int(bool(permute)), int(row0), int(n_rows))
    check(lib().gemb_synth_rmat(*args, ctypes.byref(nnz), ctypes.byref(tot), None, None, 0))
    rows = (1 << scale) if n_rows < 0 else int(n_rows)
    indptr = np.empty(rows + 1, dtype=np.int64)
    indices = np.empty(max(int(nnz.value), 1), dtype=np.int32)
    check(lib().gemb_synth_rmat(*args, ctypes.byref(nnz), ctypes.byref(tot), _ptr(indptr), _ptr(indices), int(indices.shape[0])))
    return indptr, indices[:int(nnz.value)], int(tot.value)


def graph_factorization(ctx, n, src, dst, w, d, eta, regu, max_iter, X0, mode=0):
    """gemb_gf: the edge SGD of gf.py:94-104 on the device.  Returns (X n x d float32, device ms)."""
    src = np.ascontiguousarray(src, dtype=np.int32)
    dst = np.ascontiguousarray(dst, dtype=np.int32)
    w = None if w is None else np.ascontiguousarray(w, dtype=np.float32)
    X0 = np.ascontiguousarray(X0, dtype=np.float32)
    assert X0.shape == (int(n), int(d)) and src.shape == dst.shape
    X = np.empty_like(X0)
    ms = ctypes.c_double(0.0)
    check(lib().gemb_gf(ctx._h, int(n), int(src.shape[0]), _ptr(src), _ptr(dst), _ptr(w), int(d), float(eta), float(regu),
                        int(max_iter), int(mode), _ptr(X0), _ptr(X), ctypes.byref(ms)))
    return X, float(ms.value)


def comm_unique_id():
    buf = ctypes.create_string_buffer(UNIQUE_ID_BYTES)
    check(lib().gemb_comm_unique_id(buf))
    return buf.raw


class DeviceGraph(_Handle):
    """A CSR row shard (and its transpose) resident in HBM."""
    _destroy = 'gemb_graph_free'

    def __init__(self, ctx, n, indptr, indices, data=None, indptr_t=None, indices_t=None, data_t=None,
                 row0=0):
        self.ctx = ctx
        if len(indptr) and int(indptr[-1]) >= 2 ** 31:
            raise ValueError('a CSR shard holds %d nonzeros; gemb_graph_upload takes int32 offsets (< 2^31 per shard): '
                             'shard the rows over more GPUs' % int(indptr[-1]))
        if indptr_t is not None and len(indptr_t) and int(indptr_t[-1]) >= 2 ** 31:
            raise ValueError('the transposed shard holds >= 2^31 nonzeros')
        indptr = np.ascontiguousarray(indptr, dtype=np.int32)
        indices = np.ascontiguousarray(indices, dtype=np.int32)
        data = None if data is None else np.ascontiguousarray(data, dtype=np.float32)
        if indptr_t is not None:
            indptr_t = np.ascontiguousarray(indptr_t, dtype=np.int32)
            indices_t = np.ascontiguousarray(indices_t, dtype=np.int32)
            data_t = None if data_t is None else np.ascontiguousarray(data_t, dtype=np.float32)
        self.n = int(n)
        self.row0 = int(row0)
        self.n_local = int(indptr.shape[0] - 1)
        self.nnz = int(indptr[-1])
        self.weighted = data is not None
        self._h = ctypes.c_void_p()
        check(lib().gemb_graph_upload(ctx._h, self.n, self.row0, self.n_local, _ptr(indptr), _ptr(indices),
                                      _ptr(data), _ptr(indptr_t), _ptr(indices_t), _ptr(data_t),
                                      ctypes.byref(self._h)))

    def spmm(self, X, alpha=1.0, X0=None, transpose=False, gamma=0.0, Xself=None, delta=1.0):
        """Y = alpha op(A) X + gamma Xself + delta X0 (Xself, X0: n_local x b row shards or None; test hook)."""
        X = np.ascontiguousarray(X, dtype=np.float32)
        b = X.shape[1]
        X0 = None if X0 is None else np.ascontiguousarray(X0, dtype=np.float32)
        Xself = None if Xself is None else np.ascontiguousarray(Xself, dtype=np.float32)
        for a in (X0, Xself):
            assert a is None or a.shape == (self.n_local, b)
        Y = np.empty((self.n_local, b), dtype=np.float32)
        check(lib().gemb_spmm(self._h, int(bool(transpose)), b, float(alpha), _ptr(X), float(gamma), _ptr(Xself),
                              float(delta), _ptr(X0), _ptr(Y)))
        return Y

    def spmm4(self, X, alpha, gamma, Xself, delta, X0, eps, X1, transpose=False):
        """Y = alpha op(A) X + gamma Xself + delta X0 + eps X1 (the composite operator's epilogue; test hook)."""
        X = np.ascontiguousarray(X, dtype=np.float32)
        b = X.shape[1]
        ops = [np.ascontiguousarray(a, dtype=np.float32) for a in (Xself, X0, X1)]
        for a in ops:
            assert a.shape == (self.n_local, b)
        Y = np.empty((self.n_local, b), dtype=np.float32)
        check(lib().gemb_spmm4(self._h, int(bool(transpose)), b, float(alpha), _ptr(X), float(gamma), _ptr(ops[0]),
                               float(delta), _ptr(ops[1]), float(eps), _ptr(ops[2]), _ptr(Y)))
        return Y

    def hope(self, d, beta, out=None, want_output=True, **opts):
        o = HopeOpts(struct_size=ctypes.sizeof(HopeOpts), oversample=int(opts.get('oversample', -1)),
                     max_iters=int(opts.get('max_iters', 0)), min_iters=int(opts.get('min_iters', 0)),
                     tol=float(opts.get('tol', 0.0)), katz_terms=int(opts.get('katz_terms', 0)),
                     katz_tol=float(opts.get('katz_tol', 0.0)), seed=int(opts.get('seed', 0)),
                     compute_residual=int(opts.get('compute_residual', 0)), verbose=int(opts.get('verbose', 0)),
                     algorithm=int(opts.get('algorithm', 0)), cheb_degree=int(opts.get('cheb_degree', 0)),
                     cheb_range_log2=float(opts.get('cheb_range_log2', 0.0)), stop_rule=int(opts.get('stop_rule', 0)),
                     algorithm3_basis=int(opts.get('algorithm3_basis', 0)), spectral_mode=int(opts.get('spectral_mode', 0)))
        st = HopeStats(struct_size=ctypes.sizeof(HopeStats))
        X = sig = None
        if want_output:
            X = out if out is not None else np.empty((self.n_local, d), dtype=np.float32)
            assert X.dtype == np.float32 and X.shape == (self.n_local, d) and X.flags.c_contiguous
            sig = np.empty(d if o.spectral_mode in (1, 2) else d // 2, dtype=np.float32)
        check(lib().gemb_hope(self._h, int(d), float(beta), ctypes.byref(o), _ptr(X), _ptr(sig), ctypes.byref(st)))
        return X, sig, st.as_dict()

    def hope_svd_error(self, d, beta, X, n_probe=0, seed=1):
        """|| X1 X2^T - S ||_F (hope.py:38-40): exact (n_probe = 0) or a Hutchinson estimate."""
        X = np.ascontiguousarray(X, dtype=np.float32)
        assert X.shape == (self.n, d)
        err = ctypes.c_double(0.0)
        check(lib().gemb_hope_svd_error(self._h, int(d), float(beta), _ptr(X), int(n_probe), int(seed), ctypes.byref(err)))
        return float(err.value)

    def n2v_alias(self, weights64=None):
        w = None if weights64 is None else np.ascontiguousarray(weights64, dtype=np.float64)
        K = np.empty(self.nnz, dtype=np.int32)
        U = np.empty(self.nnz, dtype=np.float64)
        check(lib().gemb_n2v_alias(self._h, _ptr(w), _ptr(K), _ptr(U)))
        return K, U

    def n2v_walks(self, nids, walk_len, num_walks, p=1.0, q=1.0, seed=1, weights64=None, w_begin=0, w_end=None):
        nids = np.ascontiguousarray(nids, dtype=np.int32)
        N = nids.shape[0]
        w_end = N * num_walks if w_end is None else w_end
        w = None if weights64 is None else np.ascontiguousarray(weights64, dtype=np.float64)
        out = np.empty((w_end - w_begin, walk_len), dtype=np.int32)
        st = N2VStats(struct_size=ctypes.sizeof(N2VStats))
        check(lib().gemb_n2v_walks(self._h, _ptr(w), _ptr(nids), N, int(walk_len), int(num_walks), float(p),
                                   float(q), int(seed), int(w_begin), int(w_end), _ptr(out), ctypes.byref(st)))
        return out, st.as_dict()

    def node2vec(self, nids, d, walk_len, num_walks, con_size, max_iter, p=1.0, q=1.0, seed=1, sequential=False,
                 n_rows=None, weights64=None, out=None, want_output=True):
        nids = np.ascontiguousarray(nids, dtype=np.int32)
        N = nids.shape[0]
        n_rows = self.n if n_rows is None else int(n_rows)
        w = None if weights64 is None else np.ascontiguousarray(weights64, dtype=np.float64)
        X = None
        if want_output:
            X = out if out is not None else np.empty((n_rows, d), dtype=np.float32)
            assert X.dtype == np.float32 and X.shape == (n_rows, d) and X.flags.c_contiguous
        st = N2VStats(struct_size=ctypes.sizeof(N2VStats))
        check(lib().gemb_node2vec(self._h, _ptr(w), _ptr(nids), N, int(d), int(walk_len), int(num_walks),
                                  int(con_size), int(max_iter), float(p), float(q), int(seed), int(bool(sequential)),
                                  n_rows, _ptr(X), ctypes.byref(st)))
        return X, st.as_dict()

    free = _Handle._release


RECON_DOT, RECON_SPLIT, RECON_GAUSS = 0, 1, 2


class Reconstruction(_Handle):
    """The reconstruction of an embedding X resident on the device: gemb_recon_* (include/gemb200.h).

    kind 0 (or False): A_hat = X X^T; kind 1 (or True, or any other value but 2): A_hat = L R^T with L, R the two
    halves of the columns.  For both, dense / pairs / the w of top return A_hat (0 on the diagonal).
    kind 2: score exp(-delta) with delta = |x_i - x_j|^2 (fp32).  dense / pairs / the w of top return delta itself,
    +inf on the diagonal and where the fp64 score underflows to 0 (delta > 745.1332), so exp(-out) is the score
    everywhere; ranks / top order by delta ascending.  A non-finite X raises."""
    _destroy = 'gemb_recon_free'

    def __init__(self, ctx, X, kind):
        X = np.ascontiguousarray(X, dtype=np.float32)
        assert X.ndim == 2
        self.ctx = ctx
        self.n, self.d = int(X.shape[0]), int(X.shape[1])
        kind = int(kind)
        self.kind = kind if kind in (RECON_DOT, RECON_GAUSS) else RECON_SPLIT
        self._h = ctypes.c_void_p()
        check(lib().gemb_recon_create(ctx._h, _ptr(X), self.n, self.d, self.kind, ctypes.byref(self._h)))

    def dense(self, out=None):
        A = out if out is not None else np.empty((self.n, self.n), dtype=np.float32)
        assert A.dtype == np.float32 and A.shape == (self.n, self.n) and A.flags.c_contiguous
        check(lib().gemb_recon_dense(self._h, _ptr(A)))
        return A

    def pairs(self, i, j):
        i = np.ascontiguousarray(i, dtype=np.int32)
        j = np.ascontiguousarray(j, dtype=np.int32)
        assert i.shape == j.shape and i.ndim == 1
        out = np.empty(i.shape[0], dtype=np.float32)
        check(lib().gemb_recon_pairs(self._h, _ptr(i), _ptr(j), int(i.shape[0]), _ptr(out)))
        return out

    def ranks(self, indptr, indices, is_undirected):
        indptr = np.ascontiguousarray(indptr, dtype=np.int32)
        indices = np.ascontiguousarray(indices, dtype=np.int32)
        assert indptr.shape[0] == self.n + 1
        rank = np.zeros(max(int(indptr[-1]), 1), dtype=np.int32)
        n_pred_row = np.zeros(self.n, dtype=np.int32)
        check(lib().gemb_recon_ranks(self._h, _ptr(indptr), _ptr(indices), int(bool(is_undirected)), _ptr(rank),
                                     _ptr(n_pred_row)))
        return rank[:int(indptr[-1])], n_pred_row

    def top(self, is_undirected, max_k=-1):
        m = ctypes.c_int64(0)
        check(lib().gemb_recon_top(self._h, int(bool(is_undirected)), int(max_k), 0, None, None, None, ctypes.byref(m)))
        cnt = int(m.value)
        i = np.empty(cnt, dtype=np.int32)
        j = np.empty(cnt, dtype=np.int32)
        w = np.empty(cnt, dtype=np.float32)
        if cnt:
            check(lib().gemb_recon_top(self._h, int(bool(is_undirected)), int(max_k), cnt, _ptr(i), _ptr(j), _ptr(w),
                                       ctypes.byref(m)))
        return i, j, w

    def exclude(self, indptr, indices):
        """gemb_recon_exclude: from now on ranks / top see only the candidates outside this CSR (n + 1 offsets,
        strictly ascending column ids per row) -- the training edges of a link-prediction split.
        indptr None clears it."""
        if indptr is None:
            check(lib().gemb_recon_exclude(self._h, None, None))
            return
        indptr = np.ascontiguousarray(indptr, dtype=np.int32)
        indices = np.ascontiguousarray(indices, dtype=np.int32)
        assert indptr.shape[0] == self.n + 1 and indices.shape[0] >= int(indptr[-1])
        check(lib().gemb_recon_exclude(self._h, _ptr(indptr), _ptr(indices)))

    free = _Handle._release


def nc_fit(ctx, X, indptr, labels, L, C=1.0, tol=1e-5, max_iter=1000):
    """gemb_nc_fit: one-vs-rest logistic regression of the n x d rows X against the label CSR (indptr n + 1, strictly
    ascending label ids per row).  -> (W L x (d + 1) fp64 with rows (w_c, b_c), iters, status, stats dict)"""
    X = np.ascontiguousarray(X, dtype=np.float32)
    indptr = np.ascontiguousarray(indptr, dtype=np.int64)
    labels = np.ascontiguousarray(labels, dtype=np.int32)
    n, d = X.shape
    assert indptr.shape == (n + 1,) and labels.shape[0] >= int(indptr[-1])
    W = np.empty((int(L), d + 1), dtype=np.float64)
    iters = np.empty(int(L), dtype=np.int32)
    status = np.empty(int(L), dtype=np.int32)
    st = NCStats(struct_size=ctypes.sizeof(NCStats))
    check(lib().gemb_nc_fit(ctx._h, n, d, _ptr(X), _ptr(indptr), _ptr(labels), int(L), float(C), float(tol),
                            int(max_iter), _ptr(W), _ptr(iters), _ptr(status), ctypes.byref(st)))
    return W, iters, status, st.as_dict()


def nc_topk(ctx, X, W, koff):
    """gemb_nc_topk: row i of X gets the koff[i + 1] - koff[i] labels of largest probability (ties to the larger
    label), highest first, in CSR order.  Rows with k = 0 get nothing."""
    X = np.ascontiguousarray(X, dtype=np.float32)
    W = np.ascontiguousarray(W, dtype=np.float64)
    koff = np.ascontiguousarray(koff, dtype=np.int64)
    m, d = X.shape
    assert W.ndim == 2 and W.shape[1] == d + 1 and koff.shape == (m + 1,)
    out = np.empty(max(int(koff[-1]), 1), dtype=np.int32)
    check(lib().gemb_nc_topk(ctx._h, m, d, _ptr(X), W.shape[0], _ptr(W), _ptr(koff), _ptr(out)))
    return out[:int(koff[-1])]


class Components(_Handle):
    """The weakly connected components of an n x n CSR resident on the device: gemb_cc_* (include/gemb200.h).
    indptr int64 (n + 1), indices int32.  n_comp, lcc_root (smallest vertex id of the largest component, -1 when
    n = 0), lcc_size and lcc_nnz are read once at creation."""
    _destroy = 'gemb_cc_free'

    def __init__(self, ctx, n, indptr, indices):
        indptr = np.ascontiguousarray(indptr, dtype=np.int64)
        indices = np.ascontiguousarray(indices, dtype=np.int32)
        assert indptr.shape == (int(n) + 1,)
        self.ctx = ctx
        self.n = int(n)
        self._h = ctypes.c_void_p()
        check(lib().gemb_cc_create(ctx._h, self.n, _ptr(indptr), _ptr(indices), ctypes.byref(self._h)))
        v = [ctypes.c_int64(0) for _ in range(4)]
        check(lib().gemb_cc_info(self._h, *(ctypes.byref(x) for x in v)))
        self.n_comp, self.lcc_root, self.lcc_size, self.lcc_nnz = (int(x.value) for x in v)

    def labels(self):
        """Component number of every vertex, 0..n_comp - 1 in the order of each component's smallest vertex."""
        out = np.empty(self.n, dtype=np.int32)
        check(lib().gemb_cc_labels(self._h, _ptr(out)))
        return out

    def lcc(self, data=None):
        """The largest component as a CSR: (node_l int64 ascending old rows, indptr int64, indices int32, weights
        fp64 or None).  data: the nnz fp64 weights of the graph, or None (unit)."""
        data = None if data is None else np.ascontiguousarray(data, dtype=np.float64)
        k, m = self.lcc_size, self.lcc_nnz
        node_l = np.empty(k, dtype=np.int64)
        indptr = np.empty(k + 1, dtype=np.int64)
        indices = np.empty(max(m, 1), dtype=np.int32)
        w = None if data is None else np.empty(max(m, 1), dtype=np.float64)
        check(lib().gemb_cc_lcc(self._h, _ptr(data), _ptr(node_l), _ptr(indptr), _ptr(indices), _ptr(w)))
        return node_l, indptr, indices[:m], (None if w is None else w[:m])

    def times(self):
        """(device ms of the labelling, device ms of the last lcc extraction)"""
        a, b = ctypes.c_double(0.0), ctypes.c_double(0.0)
        check(lib().gemb_cc_times(self._h, ctypes.byref(a), ctypes.byref(b)))
        return float(a.value), float(b.value)

    free = _Handle._release
