"""oracle/n2v_oracle_py.py -- TEST INFRASTRUCTURE: ctypes front end of oracle/n2v_oracle.c
(our CPU restatement of the SNAP node2vec binary GEM shells out to, node2vec.py:31-48).
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import it."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, 'build', 'libn2v_oracle.so')
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, 'n2v_oracle.c')
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
            subprocess.check_call(['make', '-C', _HERE, 'all'], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(_SO)
        i64p = np.ctypeslib.ndpointer(np.int64, flags='C')
        i32p = np.ctypeslib.ndpointer(np.int32, flags='C')
        f64p = np.ctypeslib.ndpointer(np.float64, flags='C')
        L.n2v_oracle_alias_first_order.argtypes = [ctypes.c_int64, i64p, f64p, i32p, f64p]
        L.n2v_oracle_walks.argtypes = [ctypes.c_int64, i64p, i32p, f64p, i32p, ctypes.c_int64, ctypes.c_int,
                                       ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_int32,
                                       ctypes.c_int, i32p, ctypes.c_void_p]
        L.n2v_oracle_learn.argtypes = [i32p, ctypes.c_int64, ctypes.c_int, ctypes.c_int64, ctypes.c_int,
                                       ctypes.c_int, ctypes.c_int, ctypes.c_int32, ctypes.c_int,
                                       ctypes.POINTER(ctypes.c_int64), i32p, f64p, ctypes.c_void_p]
        L.n2v_oracle_rng_skip.argtypes = [ctypes.c_int32, ctypes.c_uint64]
        L.n2v_oracle_rng_skip.restype = ctypes.c_int32
        _lib = L
    return _lib


def _weights(csr_data, nnz):
    return np.ones(nnz, dtype=np.float64) if csr_data is None else np.ascontiguousarray(csr_data, np.float64)


def alias_first_order(indptr, data):
    indptr = np.ascontiguousarray(indptr, np.int64)
    nnz = int(indptr[-1])
    w = _weights(data, nnz)
    K = np.zeros(max(nnz, 1), np.int32)
    U = np.zeros(max(nnz, 1), np.float64)
    rc = lib().n2v_oracle_alias_first_order(len(indptr) - 1, indptr, w, K, U)
    assert rc == 0
    return K[:nnz], U[:nnz]


def walks(indptr, indices, data, nids, walk_len, num_walks, p=1.0, q=1.0, seed=1, mode=1, return_order=False):
    """mode 0 = one sequential TRnd stream (the single-threaded binary); mode 1 = strided streams
    (what the GPU reproduces; identical to mode 0 when no walk hits a dead end)."""
    indptr = np.ascontiguousarray(indptr, np.int64)
    indices = np.ascontiguousarray(indices, np.int32)
    nnz = int(indptr[-1])
    w = _weights(data, nnz)
    nids = np.ascontiguousarray(nids, np.int32)
    N = len(nids)
    out = np.zeros((num_walks * N, walk_len), np.int32)
    order = np.zeros((num_walks, N), np.int32)
    rc = lib().n2v_oracle_walks(len(indptr) - 1, indptr, indices if nnz else np.zeros(1, np.int32), w if nnz else np.ones(1),
                                nids, N, walk_len, num_walks, float(p), float(q), int(seed), int(mode), out,
                                order.ctypes.data_as(ctypes.c_void_p))
    assert rc == 0
    return (out, order) if return_order else out


def learn(walk_matrix, n_ids, d, win, iters, seed, return_neg=False, walk_streams=False):
    """word2vec phase on a walk matrix (node ids).  Returns X (n_ids x d fp64, row = node id, rows of
    ids that never occur are 0, exactly what loadEmbedding builds) and the token->node table.
    walk_streams=False: the binary's single TRnd stream; True: every walk of every epoch starts at its
    own stream offset, as the GPU's Hogwild mode does (see n2v_oracle_learn)."""
    wm = np.array(walk_matrix, dtype=np.int32, order='C', copy=True)
    V = ctypes.c_int64(0)
    tok = np.zeros(n_ids, np.int32)
    sp = np.zeros((n_ids, d), np.float64)
    sn = np.zeros((n_ids, d), np.float64) if return_neg else None
    rc = lib().n2v_oracle_learn(wm, wm.shape[0], wm.shape[1], n_ids, d, win, iters, int(seed), int(bool(walk_streams)),
                                ctypes.byref(V), tok, sp, None if sn is None else sn.ctypes.data_as(ctypes.c_void_p))
    assert rc == 0
    V = V.value
    X = np.zeros((n_ids, d), np.float64)
    X[tok[:V]] = sp[:V]
    if return_neg:
        Xn = np.zeros((n_ids, d), np.float64)
        Xn[tok[:V]] = sn[:V]
        return X, tok[:V].copy(), Xn
    return X, tok[:V].copy()


def node2vec(indptr, indices, data, nids, d, walk_len, num_walks, con_size, max_iter, p=1.0, q=1.0, seed=1, mode=0):
    """Whole program: same seed for the walk TRnd and the word2vec TRnd (the binary seeds both from
    time(NULL) within the same second)."""
    wm = walks(indptr, indices, data, nids, walk_len, num_walks, p, q, seed, mode)
    n_ids = max(len(indptr) - 1, int(wm.max()) + 1)
    X, tok = learn(wm, n_ids, d, con_size, max_iter, seed)
    return X, tok, wm


def rng_skip(seed, k):
    return lib().n2v_oracle_rng_skip(int(seed), int(k))
