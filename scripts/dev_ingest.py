"""Developer probe: throughput of the native wire-format readers / writers against the reference-style Python loops."""
import json, os, sys, time, tempfile, shutil
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from gem_b200 import synth
from gem_b200.utils import graph_util as gu

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
out = {'host_cores': os.cpu_count(), 'n': n}
csr = synth.sbm(n=n, block=1000, seed=42)
out['edges'] = csr.nnz
td = tempfile.mkdtemp(dir='/dev/shm' if os.path.isdir('/dev/shm') else None)
try:
    f = os.path.join(td, 'g.txt')
    t = time.perf_counter(); gu.saveEdgeListCSR(csr, f, n2v=True); out['write_s'] = time.perf_counter() - t
    out['file_MB'] = os.path.getsize(f) / 1e6
    gu.readEdgeList(f)
    t = time.perf_counter(); s, d, w = gu.readEdgeList(f); out['parse_s'] = time.perf_counter() - t
    t = time.perf_counter(); back = gu.loadEdgeListCSR(f); out['parse_plus_csr_s'] = time.perf_counter() - t
    assert np.array_equal(back.indices, csr.indices)
    m = min(csr.nnz, 400_000)
    with open(f) as fh:
        lines = [next(fh) for _ in range(m)]
    g = os.path.join(td, 's.txt'); open(g, 'w').write(''.join(lines))
    t = time.perf_counter(); G = gu.loadGraphFromEdgeListTxt(g); out['ref_loop_read_edges_per_s'] = m / (time.perf_counter() - t)
    t = time.perf_counter(); gu.saveGraphToEdgeListTxtn2v(G, g); out['ref_loop_write_edges_per_s'] = G.number_of_edges() / (time.perf_counter() - t)
    rows = min(n, 200_000)
    X = np.random.default_rng(0).standard_normal((rows, 128))
    e = os.path.join(td, 'x.emb')
    t = time.perf_counter(); gu.saveEmbedding(X, e); out['emb_write_s'] = time.perf_counter() - t
    t = time.perf_counter(); Y = gu.loadEmbedding(e); out['emb_read_s'] = time.perf_counter() - t
    out['emb_rows'] = rows; out['emb_MB'] = os.path.getsize(e) / 1e6
finally:
    shutil.rmtree(td)
out['write_M_edges_per_s'] = csr.nnz / out['write_s'] / 1e6
out['parse_M_edges_per_s'] = csr.nnz / out['parse_s'] / 1e6
out['parse_MB_per_s'] = out['file_MB'] / out['parse_s']
print(json.dumps(out))
