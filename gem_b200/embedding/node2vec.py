"""node2vec on an H100 -- drop-in for reference gem/embedding/node2vec.py:8-57.

The reference writes `tempGraph.graph`, runs the prebuilt SNAP executable gem/c_exe/node2vec with
`-d -l -r -k -e -p -q -v -dr -w` (node2vec.py:35-46) and parses `tempGraph.emb`
(graph_util.loadEmbedding).  Here the same pipeline -- alias tables, shuffled biased walks,
skip-gram negative-sampling SGD -- runs in libgemb200.so on the GPU; no files, no subprocess.
Same class name (lower case), hyper-parameters (d, max_iter, walk_len, num_walks, con_size, ret_p,
inout_p), method name, signature, errors and row convention (row index = integer node id,
graph_util.py:168; V rows where V-1 is the largest id, phantom row 0 if walks were padded: SURVEY F10).

ret_p / inout_p = 1 use one alias table per node; any other positive values build the reference's second-order
tables (one per directed edge (t -> v), sum_(t->v) outdeg(v) entries) on the device -- walks stay bit-exact against the
CPU restatement of the binary; a graph whose tables do not fit in HBM fails with the size in the message.

Extra optional hyper-parameters: seed (the binary uses time(NULL); default 1), device,
sequential (parity mode: one warp follows the single-threaded binary's RNG stream), dtype.
There is no CPU path: without a GPU learn_embedding raises RuntimeError.
"""
import numpy as np

from gem_b200 import _native
from gem_b200 import dist as _gd
from gem_b200 import graph as _graph
from gem_b200.embedding.static_graph_embedding import StaticGraphEmbedding


class node2vec(StaticGraphEmbedding):
    _recon_split = False      # get_edge_weight form, for the GPU reconstruction (gemb_recon_create)

    hyper_params = {
        'method_name': 'node2vec_rw'
    }

    def __init__(self, *args, **kwargs):
        """ Initialize the node2vec class

        Args:
            d: dimension of the embedding
            max_iter: max iterations
            walk_len: length of random walk
            num_walks: number of random walks
            con_size: context size
            ret_p: return weight
            inout_p: inout weight
        """
        super(node2vec, self).__init__(*args, **kwargs)
        self.stats = None

    def learn_embedding(self, graph=None, is_weighted=False, no_python=False, **ignored):
        self._check_graph(graph)
        if isinstance(graph, tuple):          # (HostCSR, nids): large inputs without networkx
            csr, nids = graph
        else:
            csr, nids = _graph.n2v_inputs_from_networkx(graph)
        dist_mod, rank, world, device = _gd.spmd(getattr(self, '_device', None))
        with _native.Context(device) as ctx:
            if world > 1:
                # SPMD (INTEGRATION.md C): every rank holds the whole graph, walks its share of the walk index space and
                # trains on it; the embedding deltas are all-reduced once per epoch, so every rank returns the same X
                _gd.init_comm_from_torch(ctx, dist_mod, rank, world)
            with _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, None) as g:
                X, st = g.node2vec(nids, int(self._d), int(self._walk_len), int(self._num_walks),
                                   int(self._con_size), int(self._max_iter), float(self._ret_p),
                                   float(self._inout_p), seed=int(getattr(self, '_seed', 1)),
                                   sequential=bool(getattr(self, '_sequential', False)),
                                   n_rows=csr.n, weights64=csr.data)
        self.stats = st
        return self._result(X, csr.n)

    def get_edge_weight(self, i, j):
        return np.dot(self._X[i, :], self._X[j, :])
