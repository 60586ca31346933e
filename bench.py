#!/usr/bin/env python
"""bench.py -- nodes/sec embedded at d=128 (HOPE, node2vec) on H100 vs the reference's CPU path.

    python bench.py --gpus N --steps K --warmup W [--workload hope|node2vec|recon] [--impl reference] [--dump-outputs DIR]

Default (N=1): BASELINE.json configs[1] -- HOPE d=128, beta=0.01 on the synthetic SBM with
1,000,000 nodes / ~20M directed edges (SURVEY 8(d) config 2), one H100.  A "step" is one complete
learn_embedding-equivalent pass (norm estimate, Katz/SpMM subspace iteration, Rayleigh-Ritz, X) over
the graph.
  value : n * K / (sum of the K device times), CSR already resident in HBM, X left on the device;
          device time = CUDA events inside libgemb200 around the whole solve, max over ranks.
  e2e   : the same metric through the reference-facing plugin call HOPE.learn_embedding(graph=CSR)
          with HOST buffers: pinned CSR -> H2D, solve, D2H of the n x d embedding, every step.
  N > 1 : launched by torchrun, one rank per GPU; weak scaling: n = N * 1,000,000 (rows per GPU fixed),
          CSR row-sharded; only the rows a shard references travel, stored into the peers' halo slots over NVLink by the
          kernel that produces them (gem_b200/csrc/halo.cu); b x b all-reduce per Gram on NCCL.
  The default line also carries a "node2vec" sub-record: BASELINE.json configs[2] on the same graph (one epoch, its own
  "steps": 1 -- an epoch takes seconds).
--workload node2vec: BASELINE.json configs[2] (d=128, p=q=1, 10 walks x 80, context 10, 1 epoch).
--workload recon: the step after learn_embedding in every reference test (tests/fit_model.py:10, SURVEY 8(f) rank 1):
  evaluateStaticGraphReconstruction of a HOPE embedding (d=128) of an SBM with --recon-n nodes (default 32768):
  A_hat = X1 X2^T on the device, rank of every true edge (MAP), precision@1000.  Metric: node PAIRS scored and ranked
  per second (n^2 / step time; the work is quadratic, so nodes/s would depend on n).
--impl reference: the reference's CPU implementation of the same path on the host cores
  (HOPE: oracle/hope_oracle.hope_sparse = scipy svds over the matrix-free Katz operator, the only
  form of hope.py:28-36 that fits in memory beyond ~50k nodes, at the FULL 1M-node configuration with the operator on
  all host cores; node2vec: the reference's own SNAP binary from oracle/_ref when present, else
  oracle/n2v_oracle.c, on a bounded sample).
--steps K sets the number of timed steps of the workload's line: the device-time loop and the end-to-end calls.
--dump-outputs DIR: after the timed steps, write what the timed path returned in its last step as DIR/<name>.npy
  (float32 / float64; an n x d embedding is written as a fixed, seeded sample of DUMP_ROWS rows plus their row ids).
  The inputs depend only on the arguments (seeded generators), and the HOPE and reconstruction paths add across CTAs in a
  fixed order (no floating-point atomics), so a run reproduces the outputs bit for bit and two builds can be compared output
  for output.  The default line dumps HOPE's outputs only: node2vec's Hogwild SGNS (like the reference's OpenMP training)
  applies its updates in the order the warps run, so its embedding differs between runs; `--workload node2vec` still
  writes it.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

os.environ.setdefault('OMP_WAIT_POLICY', 'PASSIVE')   # the CPU arms mix an OpenMP operator with BLAS threads

REPO = os.path.dirname(os.path.abspath(__file__))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

# The timed solver setting (explicit in the line's config.solver; parity-tested at this exact setting against the fp64
# oracle by tests/test_gpu_hope.py::test_bench_solver_setting_against_fp64_oracle): Chebyshev filter degree <= 16,
# dynamic-range guard 2^14, oversample 8 (block 72), stop when the residual of every wanted Ritz pair, mapped to the
# Katz operator, is <= 4e-3 sigma_max (stop_rule 1) -- round 1 stopped on a 1e-3 singular-value change and DELIVERED
# 4.0e-3; this setting delivers 3.0e-3 in 4 rounds instead of 8 (scripts/exp_solver.py sweeps the settings).
HOPE_SOLVER = dict(tol=4e-3, stop_rule=1, cheb_degree=16, cheb_range_log2=14, max_iters=30, min_iters=2, oversample=8, seed=1234)
CPU_ARPACK_TOL = 1e-3      # tol handed to scipy svds in the CPU arm (the reference's own tol=0 does not terminate at 1M nodes)


def read_peaks():
    p = os.path.join(REPO, 'MEASURED_PEAKS.json')
    if os.path.exists(p):
        try:
            return json.load(open(p)), 'measured (MEASURED_PEAKS.json)'
        except Exception:
            pass
    return {'hbm_gbs': 3350.0, 'bf16_tflops': 989.0}, 'H100 SXM data sheet (700 W board power)'


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region, with the card's name and power limit."""
    Q = ('index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,'
         'clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,'
         'clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap,name,power.limit')

    def __init__(self, device):
        self.device = device
        self.lines = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(['nvidia-smi', '-i', str(self.device), '--query-gpu=' + self.Q,
                                          '--format=csv,noheader,nounits', '-lms', '50'],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._pump, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if not self.proc:
            return {'sm_mhz': None, 'sm_max_mhz': None, 'reasons': ['nvidia-smi unavailable']}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons, gpu, plim = [], [], set(), None, None
        names = ['hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap']
        for ln in self.lines:
            f = [x.strip() for x in ln.split(',')]
            if len(f) < 11:
                continue
            gpu, plim = f[9], f[10]
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
            except ValueError:
                continue
            for name, val in zip(names, f[5:9]):
                if val.lower().startswith('active'):
                    reasons.add(name)
        return {'gpu': gpu, 'power_limit_w': plim, 'sm_mhz': float(np.median(sm)) if sm else None,
                'sm_max_mhz': float(max(mx)) if mx else None, 'samples': len(sm), 'reasons': sorted(reasons)}


DUMP_ROWS = 32768      # rows of an n x d output that --dump-outputs keeps (16 MB at d = 128)


def row_sample(X, row0=0):
    """A fixed, seeded sample of the rows of X (all rows when there are at most DUMP_ROWS): (global row ids as float64,
    the rows)."""
    n = X.shape[0]
    rows = np.arange(n) if n <= DUMP_ROWS else np.sort(np.random.default_rng(0).choice(n, DUMP_ROWS, replace=False))
    return (rows + row0).astype(np.float64), np.ascontiguousarray(X[rows])


def dump_outputs(path, arrays):
    """--dump-outputs: <path>/<name>.npy for every array (float32 / float64)."""
    os.makedirs(path, exist_ok=True)
    for name, a in arrays.items():
        a = np.asarray(a)
        assert a.dtype in (np.float32, np.float64), (name, a.dtype)
        np.save(os.path.join(path, name + '.npy'), a)


# ----------------------------------------------------------------------------------- distributed glue
def dist_setup(n_gpus):
    rank = int(os.environ.get('RANK', '0'))
    world = int(os.environ.get('WORLD_SIZE', '1'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if world == 1:
        return None, 0, 1, 0
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    assert world == n_gpus, 'WORLD_SIZE %d != --gpus %d' % (world, n_gpus)
    return dist, rank, world, local


def dist_barrier(dist, local):
    if dist is None:
        return
    import torch
    dist.barrier(device_ids=[local])
    torch.cuda.synchronize()


def dist_max(dist, x, local):
    if dist is None:
        return x
    import torch
    t = torch.tensor([x], dtype=torch.float64, device='cuda:%d' % local)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def dist_sum(dist, x, local):
    if dist is None:
        return x
    import torch
    t = torch.tensor([x], dtype=torch.float64, device='cuda:%d' % local)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t.item())


# ----------------------------------------------------------------------------------- CPU baselines
def cpu_hope_sample(n_sample, d, beta, tol, seed=42, A=None):
    """The reference path on the host: scipy svds (hope.py:33, ARPACK) over the Katz operator (hope.py:29-31) applied
    matrix-free in fp64, the operator's row loop on all host cores (oracle/katz_omp.c), ARPACK's own BLAS calls on
    whatever threads the BLAS takes.  Returns (nodes/s, seconds, info)."""
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import hope_oracle as ho
    from gem_b200 import synth
    if A is None:
        A = synth.sbm(n=n_sample, block=min(1000, n_sample), seed=seed).to_scipy()
    threads, calib = pick_katz_threads(ho, A, beta)
    t = time.perf_counter()
    X, s, info = ho.hope_sparse(A, d, beta, katz_tol=1e-7, tol=tol, threads=threads)
    dt = time.perf_counter() - t
    info['threads'] = int(ho.katz_omp_lib().katz_omp_threads())
    info['thread_calibration_ms'] = calib
    return A.shape[0] / dt, dt, info


def cpu_hope_rmat_sample(scale, d, beta_over_rho):
    """CPU arm of the R-MAT workload on a bounded sample: the host generator's R-MAT at `scale` (same family, seed 42),
    beta = beta_over_rho / rho(A) (rho from scipy eigsh), scipy svds(tol=1e-3) over the matrix-free Katz operator."""
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import hope_oracle as ho
    import scipy.sparse.linalg as sla
    from gem_b200 import synth
    A = synth.rmat(scale=scale, seed=42).to_scipy().astype(np.float64)
    rho = float(abs(sla.eigsh(A, k=1, which='LA', return_eigenvectors=False)[0]))
    beta = beta_over_rho / rho
    threads, calib = pick_katz_threads(ho, A, beta)
    t = time.perf_counter()
    X, s_, info = ho.hope_sparse(A, d, beta, katz_tol=1e-7, tol=CPU_ARPACK_TOL, threads=threads)
    dt = time.perf_counter() - t
    return {'value': A.shape[0] / dt, 'unit': 'nodes/s', 'cores': threads, 'kind': 'port', 'host_cores': os.cpu_count(), 'seconds': dt,
            'sample': 'R-MAT scale %d (host generator, seed 42), d=%d, beta=%g/rho=%.6g: scipy svds(tol=%g, ARPACK) over the matrix-free '
                      'fp64 Katz operator on %d OpenMP threads, J=%d, %d SpMVs' % (scale, d, beta_over_rho, beta, CPU_ARPACK_TOL, threads,
                                                                                  info['katz_terms'], info['spmv'])}


def pick_katz_threads(ho, A, beta):
    """Thread count of the OpenMP Katz operator for the CPU arm: the fastest of {1, 2, 4, ... , usable cores} on THIS
    matrix, each timed over a few operator applications interleaved with a BLAS product on an n x 32 block (ARPACK's own
    work runs on the BLAS's threads between the operator calls; with both pools at 128 threads the operator of a 100k-node
    sample ran 20x SLOWER than on one thread on the 128-core GPU box -- 349 s against 18 s -- so 'all cores' is not
    'all the host threads it can use' for small samples)."""
    try:
        usable = len(os.sched_getaffinity(0))
    except AttributeError:
        usable = os.cpu_count() or 1
    cands = sorted({t for t in (1, 2, 4, 8, 16, 32, 64, 128, 256) if t < usable} | {usable})
    L = ho.katz_omp_lib()
    n = A.shape[0]
    op = ho.KatzOMP(A, beta, 4)
    x = np.random.default_rng(0).standard_normal(n)
    Q = np.random.default_rng(1).standard_normal((n, 32))
    best, out = None, {}
    for t in cands:
        L.katz_omp_set_threads(t)
        op(x)
        t0 = time.perf_counter()
        for _ in range(3):
            y = op(x)
            x = y / np.linalg.norm(y)
            Q.T @ x
        ms = (time.perf_counter() - t0) * 1e3 / 3
        out[str(t)] = round(ms, 3)
        if best is None or ms < best[1]:
            best = (t, ms)
        if ms > 4 * best[1]:
            break                        # more threads only get slower from here
    return best[0], out


# The UNMODIFIED reference class (gem.embedding.hope.HOPE: dense inverse + scipy svds) cannot travel to the GPU box
# (/root/reference does not exist there) and cannot hold more than ~16k nodes anywhere (n x n fp64).  These are its wall
# times on the same SBM family at d = 128, beta = 0.01, measured in the build container (8 cores) with the harness-side
# networkx shim (DESIGN.md section 6); printed beside the reference arm for orientation, never used in a ratio.
REFERENCE_CLASS_TIMINGS = {'where': 'build container, 8 host cores, gem.embedding.hope.HOPE unmodified',
                           'n=1024': {'seconds': 1.9, 'nodes_per_s': 551}, 'n=2048': {'seconds': 1.7, 'nodes_per_s': 1184},
                           'n=4096': {'seconds': 11.4, 'nodes_per_s': 360}, 'n=8192': {'seconds': 53.6, 'nodes_per_s': 153}}


def cpu_n2v_sample(n_sample, d, walk_len, num_walks, con_size, threads, csr=None):
    """node2vec on the host: the reference's SNAP binary (oracle/_ref/node2vec, all threads) when it is
    present, else our single-threaded C restatement.  Returns (nodes/s, seconds, kind, cores)."""
    import tempfile
    from gem_b200 import synth
    if csr is None:
        csr = synth.sbm(n=n_sample, block=min(1000, n_sample), seed=42)
    exe = os.path.join(REPO, 'oracle/_ref/node2vec')
    if os.path.exists(exe):
        with tempfile.TemporaryDirectory() as td:
            rows = np.repeat(np.arange(csr.n), np.diff(csr.indptr))
            with open(os.path.join(td, 'g.graph'), 'w') as f:
                f.write(''.join('%d %d 1.000000\n' % (a, b) for a, b in zip(rows.tolist(), csr.indices.tolist())))
            env = dict(os.environ, OMP_NUM_THREADS=str(threads))
            args = [exe, '-i:g.graph', '-o:g.emb', '-d:%d' % d, '-l:%d' % walk_len, '-r:%d' % num_walks,
                    '-k:%d' % con_size, '-e:1', '-p:1.000000', '-q:1.000000', '-dr', '-w']
            t = time.perf_counter()
            subprocess.check_call(args, cwd=td, env=env, stdout=subprocess.DEVNULL)
            dt = time.perf_counter() - t
        return n_sample / dt, dt, 'reference', threads
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import n2v_oracle_py as no
    nids = np.arange(csr.n, dtype=np.int32)
    t = time.perf_counter()
    no.node2vec(csr.indptr, csr.indices, None, nids, d, walk_len, num_walks, con_size, 1, seed=1, mode=1)
    dt = time.perf_counter() - t
    return n_sample / dt, dt, 'port', 1


def cpu_recon_sample(n_sample, d, max_k=1000):
    """The reference's evaluation on the host, vectorised (oracle/eval_oracle.py: one GEMM instead of n^2 np.dot
    calls, stable argsorts instead of Python sorts -- far faster than gem.evaluation's loops, same results).
    Returns (pairs/s, seconds)."""
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import eval_oracle as eo
    from gem_b200 import synth
    csr = synth.sbm(n=n_sample, block=min(1024, n_sample), seed=42)
    X = np.random.default_rng(0).standard_normal((n_sample, d)) * 0.3
    t = time.perf_counter()
    A = eo.reconstruct(X, True, exact=False)
    eo.evaluate(A, eo.EdgeSet(csr.n, csr.indptr, csr.indices), is_undirected=True, max_k=max_k)
    dt = time.perf_counter() - t
    return float(n_sample) * n_sample / dt, dt


# ----------------------------------------------------------------------------------- reference arm
def run_reference(args):
    rank = int(os.environ.get('RANK', '0'))
    if rank != 0:
        return
    cores = os.cpu_count() or 1
    if args.workload == 'recon':
        n_s = args.cpu_sample or 8192
        secs = []
        for _ in range(args.warmup):
            cpu_recon_sample(2048, args.d)
        for _ in range(args.steps):
            v, dt = cpu_recon_sample(n_s, args.d)
            secs.append(dt)
        value = float(n_s) * n_s * len(secs) / sum(secs)
        line = {'impl': 'reference', 'metric': 'node pairs evaluated/sec (reconstruction + MAP + precision@1000)', 'value': value,
                'unit': 'pairs/s', 'n_gpus': args.gpus, 'steps': args.steps, 'warmup': args.warmup,
                'ms_per_step': 1e3 * sum(secs) / len(secs), 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
                'dtype': 'f64', 'data': 'synthetic',
                'config': {'workload': 'reconstruction evaluation d=%d, SBM (CPU arm runs a bounded sample)' % args.d},
                'cpu_baseline': {'value': value, 'unit': 'pairs/s', 'cores': 1, 'kind': 'port', 'host_cores': cores,
                                 'sample': 'SBM n=%d, random X (d=%d): oracle/eval_oracle.py (vectorised restatement of '
                                           'gem.evaluation; BLAS GEMM may use several threads)' % (n_s, args.d)},
                'e2e': {'value': value, 'unit': 'pairs/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}}
        print(json.dumps(line), flush=True)
        return
    # bounded CPU work: about 150 s of timed samples in total whatever --steps is (a 50k-node HOPE sample takes ~40 s,
    # a 4000-node node2vec sample ~65 s on the 128-core box; both scale about linearly in the sample size)
    def bounded(base_nodes, base_seconds, floor):
        if args.cpu_sample:
            return args.cpu_sample
        return max(floor, int(base_nodes * min(1.0, 150.0 / (max(args.steps, 1) * base_seconds))))

    if args.workload == 'hope':
        # the SAME configuration as our arm: n = args.n (1M) nodes, same generator and seed.  One solve takes minutes, so
        # the K requested steps are run only while a ~9 minute budget lasts (at least one); --cpu-sample N shrinks the graph.
        from gem_b200 import synth
        sys.path.insert(0, os.path.join(REPO, 'oracle'))
        import hope_oracle as ho
        n_s = args.cpu_sample or args.n
        A = synth.sbm(n=n_s, block=min(1000, n_s), seed=42).to_scipy()
        secs, info = [], None
        budget_s = float(os.environ.get('GEMB_REF_BUDGET_S', '420'))      # a second solve starts only if it would end inside this
        # projected time of ONE solve from the calibrated operator: ~1500 operator applications of J = 11 sweeps (ARPACK
        # eigsh on S^T S, k = 64, tol 1e-3, on this spectrum), scaled by what the box measured; if that does not fit the
        # budget the graph is shrunk proportionally (stated in the line) instead of running past the driver's patience
        if not args.cpu_sample:
            _, calib = pick_katz_threads(ho, A, args.beta)
            # calibration on the box (r02q): 1481 operator applications, 148 s at n = 479 k with 32 threads
            proj = 1500 * min(calib.values()) * (11.0 / 4.0) / 1e3 * 0.6
            if proj > budget_s:
                n_s = max(50_000, int(n_s * budget_s / proj) // 1000 * 1000)
                A = synth.sbm(n=n_s, block=1000, seed=42).to_scipy()
        t_begin = time.perf_counter()
        for i in range(args.steps):
            v, dt, info = cpu_hope_sample(n_s, args.d, args.beta, CPU_ARPACK_TOL, A=A)
            secs.append(dt)
            if time.perf_counter() - t_begin + dt > budget_s:
                break
        value = n_s * len(secs) / sum(secs)
        kind, used = 'port', info['threads']
        sample = ('the full workload: SBM n=%d (seed 42), d=%d, beta=%g; scipy svds(tol=%g, ARPACK) over the matrix-free '
                  'fp64 Katz operator (J=%d Horner terms, %d SpMVs per solve) with the operator on %d OpenMP threads; '
                  '%d of the %d requested steps timed (each a complete solve), no warm-up' % (
                      n_s, args.d, args.beta, CPU_ARPACK_TOL, info['katz_terms'], info['spmv'], used, len(secs), args.steps))
        cfg = {'workload': hope_workload_name(args.d, args.beta, n_s, 1), 'timed_solves': len(secs),
               'reference_class_itself': REFERENCE_CLASS_TIMINGS}
    else:
        n_s = bounded(4000, 65.0, 500)
        n_s = n_s // 1000 * 1000 if n_s >= 1000 else n_s // 100 * 100      # synth.sbm wants whole blocks
        for _ in range(args.warmup):
            cpu_n2v_sample(min(1000, n_s), args.d, args.walk_len, args.num_walks, args.con_size, cores)
        secs = []
        for _ in range(args.steps):
            v, dt, kind, used = cpu_n2v_sample(n_s, args.d, args.walk_len, args.num_walks, args.con_size, cores)
            secs.append(dt)
        value = n_s * len(secs) / sum(secs)
        sample = 'SBM n=%d (same density, seed 42), d=%d, r=%d, l=%d, k=%d, 1 epoch' % (
            n_s, args.d, args.num_walks, args.walk_len, args.con_size)
        cfg = {'workload': 'node2vec d=%d p=q=1 r=%d l=%d k=%d, SBM 1M nodes / 20M edges (CPU arm runs a bounded sample)' % (
            args.d, args.num_walks, args.walk_len, args.con_size)}
    line = {'impl': 'reference', 'metric': 'nodes/sec embedded at d=128', 'value': value, 'unit': 'nodes/s',
            'n_gpus': args.gpus, 'steps': args.steps, 'warmup': args.warmup_requested,
            'warmup_done': 0 if args.workload == 'hope' else args.warmup, 'steps_done': len(secs),
            'ms_per_step': 1e3 * sum(secs) / len(secs), 'higher_is_better': True, 'scaling': 'weak',
            'vs_baseline': None, 'dtype': 'f64', 'data': 'synthetic', 'config': cfg,
            'cpu_baseline': {'value': value, 'unit': 'nodes/s', 'cores': used, 'kind': kind, 'sample': sample,
                             'host_cores': cores},
            'e2e': {'value': value, 'unit': 'nodes/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}}
    print(json.dumps(line), flush=True)



# ----------------------------------------------------------------------------------- graphs
def rmat_rows(n, rank, world):
    per = (n + world - 1) // world
    r0 = min(n, rank * per)
    return r0, min(n, r0 + per) - r0


def rmat_name(args):
    return ('R-MAT scale %d (Graph500 a,b,c,d = .57,.19,.19,.05, edge factor 8, vertices permuted, symmetrised, loops and '
            'duplicates removed; generated on the device by gemb_synth_rmat, counter-based RNG seed 42)' % args.scale)

# ----------------------------------------------------------------------------------- our arm
def hope_workload_name(d, beta, n, world):
    return ('HOPE d=%d beta=%g on SBM n=%d (%d per GPU), ~20 directed edges per node, 1000-node blocks, '
            'deg 16 in / 4 out, seed 42' % (d, beta, n, n // world))


def fp64_accuracy_of_solution(csr, X, sigma, beta, n_sample=8, katz_terms=14):
    """Accuracy of the solution the timed solver setting produces, measured against the fp64 Katz operator on the host
    (plain scipy.sparse, no oracle code): for n_sample of the k triplets (always the largest one)
        resid   = max(||S v - sigma u||, ||S^T u - sigma v||) / sigma_max
        sigma   = |u^T S v - sigma| / sigma          (Rayleigh quotient of the pair vs the value the solver reports)
    and the angle between the solver's top right vector and the dominant eigenvector of A from 60 fp64 power steps
    (S = f(A) shares A's eigenvectors; the top one is isolated on the SBM, so this angle is well defined)."""
    import scipy.sparse as sp
    n, d = X.shape
    k = d // 2
    A = sp.csr_matrix((np.ones(csr.nnz), csr.indices, np.asarray(csr.indptr, dtype=np.int64)), shape=(n, n))
    sig = np.asarray(sigma, dtype=np.float64)
    cols = sorted(set([k - 1] + list(np.linspace(0, k - 1, n_sample).astype(int))))
    rs = np.sqrt(np.maximum(sig[cols], 1e-300))
    U = X[:, cols].astype(np.float64) / rs
    V = X[:, [k + c for c in cols]].astype(np.float64) / rs

    def katz(M, B):
        W = B
        for _ in range(katz_terms - 1):
            W = B + beta * (M @ W)
        return beta * (M @ W)
    SV, STU = katz(A, V), katz(A.T.tocsr(), U)
    smax = float(sig.max())
    r1 = np.linalg.norm(SV - U * sig[cols], axis=0) / smax
    r2 = np.linalg.norm(STU - V * sig[cols], axis=0) / smax
    rq = np.abs(np.sum(U * SV, axis=0) - sig[cols]) / sig[cols]
    x = np.ones(n) / np.sqrt(n)
    for _ in range(60):
        x = A @ x
        x /= np.linalg.norm(x)
    vt = V[:, cols.index(k - 1)]
    cosang = min(1.0, abs(float(vt @ x)) / float(np.linalg.norm(vt)))
    return {'triplets_checked': len(cols), 'resid_max_rel_sigma_max_fp64': float(max(r1.max(), r2.max())),
            'sigma_rel_err_vs_rayleigh_fp64': float(rq.max()), 'top1_angle_deg_vs_fp64_power_iteration': float(np.degrees(np.arccos(cosang))),
            'orthonormality_max_abs': float(max(np.abs(U.T @ U - np.eye(len(cols))).max(), np.abs(V.T @ V - np.eye(len(cols))).max()))}


def pinned_csr(csr):
    """Copy of the CSR in pinned host memory with int32 offsets (what gemb_graph_upload reads)."""
    from gem_b200 import _native
    from gem_b200.graph import HostCSR
    ip = _native.pinned_empty(csr.n + 1, np.int32)
    ip[:] = csr.indptr
    ix = _native.pinned_empty(max(csr.nnz, 1), np.int32)
    ix[:csr.nnz] = csr.indices
    return HostCSR(csr.n, ip, ix[:csr.nnz], None, symmetric=True)


def run_hope(args, dist, rank, world, local):
    from gem_b200 import _native, synth
    from gem_b200.embedding.hope import HOPE
    peaks, peak_src = read_peaks()
    rmat = args.graph == 'rmat'
    ctx = _native.Context(local)
    if world > 1:
        uid = [_native.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        ctx.comm_init(rank, world, uid[0])
    t0 = time.perf_counter()
    if rmat:
        # BASELINE.json configs[3]: the graph is FIXED (scale 24 = 16.7M nodes on 8 GPUs): strong scaling in N.
        # Every rank generates the graph on its own GPU (identical by construction) and keeps its row shard.
        from gem_b200.graph import HostCSR
        n = 1 << args.scale
        r0, rows = rmat_rows(n, rank, world)
        ip, ix, nnz_total = _native.synth_rmat(ctx, args.scale, seed=42, row0=r0, n_rows=rows)
        csr = HostCSR(n, ip, ix, None, symmetric=True) if world == 1 else None
        n_all, nnz_all = n, nnz_total
    else:
        n = args.n * world                                   # weak scaling: rows per GPU fixed
        csr = synth.sbm(n=n, block=1000, seed=42)            # host, not timed
        r0, ip, ix, _ = csr.row_shard(rank, world)
        n_all, nnz_all = csr.n, csr.nnz
    gen_s = time.perf_counter() - t0
    g = _native.DeviceGraph(ctx, n_all, ip, ix, None, row0=r0)
    n_own_rows = len(ip) - 1
    solver = dict(HOPE_SOLVER)
    beta_arg = args.beta
    if rmat:
        # skewed spectrum: the auto rule hands the solve to the thick-restart block Lanczos solver (algorithm 3), whose
        # stopping test is the Ritz residual mapped to the Katz operator, relative to sigma_max
        solver = dict(tol=1e-3, max_iters=60, oversample=16, seed=1234)
        beta_arg = -args.beta_over_rho                       # beta = 0.5 / rho_hat(A), rho_hat by power iteration in the call
    if args.tol is not None:
        solver['tol'] = args.tol
    if args.max_iters is not None:
        solver['max_iters'] = args.max_iters

    # clocks / throttle reasons are sampled from the first warm-up solve on (the same kernels under the same load): the timed
    # region of the default run lasts well under a second, too short for nvidia-smi's polling loop alone
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    for _ in range(args.warmup):
        g.hope(args.d, beta_arg, want_output=False, **solver)
    dist_barrier(dist, local)
    launches0 = _native.lib().gemb_launch_count()
    dev_ms, stats = 0.0, None
    t0 = time.perf_counter()
    for s in range(args.steps):
        # the last step hands X and sigma back to the host when they are dumped (total_ms ends before that copy)
        want = bool(args.dump_outputs) and s == args.steps - 1
        X_last, sig_last, st = g.hope(args.d, beta_arg, want_output=want, **solver)
        dev_ms += st['total_ms']
        stats = st if stats is None else {k: (stats[k] + st[k] if k in ('spmm_ms', 'dense_ms', 'comm_ms', 'spmm_count', 'pushes', 'push_bytes') else st[k])
                                          for k in st}
    dist_barrier(dist, local)
    wall_s = time.perf_counter() - t0
    launches = _native.lib().gemb_launch_count() - launches0
    clocks = sampler.stop() if rank == 0 else None
    dev_ms = dist_max(dist, dev_ms, local)
    wall_s = dist_max(dist, wall_s, local)
    value = n_all * args.steps / (dev_ms * 1e-3)
    if args.dump_outputs and rank == 0:
        rows, Xs = row_sample(X_last, r0)
        dump_outputs(args.dump_outputs, {'hope_X_rows': rows, 'hope_X': Xs, 'hope_sigma': sig_last})

    # accuracy of the timed solution, outside the timed region: one more identical solve that also applies the fp32
    # Katz operator to the result, || S^T u_j - sigma_j v_j || / sigma_max over the k triplets (collective on N > 1)
    resid_max = None
    try:
        _, _, st_r = g.hope(args.d, beta_arg, want_output=False, compute_residual=1, **solver)
        resid_max = float(st_r['resid_max'])
    except Exception as exc:                                   # diagnostics only: never fail the bench line
        resid_max = 'unavailable: %s' % exc

    # roofline of the dominant kernel (CSR SpMM): algorithmic bytes per launch / mean launch time
    spmm_ms_per = stats['spmm_ms'] / max(stats['spmm_count'], 1)
    achieved = stats['spmm_bytes'] / (spmm_ms_per * 1e-3) / 1e9 if spmm_ms_per > 0 else 0.0
    roofline = {'kernel': 'spmm (CSR x n-by-%d fp32 block)' % stats['block'], 'bound': 'hbm', 'achieved': achieved,
                'peak': peaks['hbm_gbs'], 'unit': 'GB/s', 'frac': achieved / peaks['hbm_gbs'], 'traffic': None,
                'peak_source': peak_src, 'bytes_per_launch': stats['spmm_bytes'], 'ms_per_launch': spmm_ms_per,
                'launches_per_step': stats['spmm_count'] / args.steps,
                'share_of_step': stats['spmm_ms'] / max(dev_ms, 1e-9)}

    # e2e through the plugin class with host buffers.  N > 1: the SPMD contract of the plugin (INTEGRATION.md C) -- every
    # rank calls learn_embedding under the initialised process group with the graph in pinned host memory, uploads ITS
    # row shard, and reads back ITS rows of X; the step time is the max over ranks of the host clock around the call.
    e2e = None
    accuracy = None
    if not args.no_e2e and csr is not None:
        g.free()
        g = None
        hc = pinned_csr(csr)
        n_own = len(csr.row_shard(rank, world)[1]) - 1
        out = _native.pinned_empty((n_own, args.d), np.float32)
        HOPE.hyper_params.clear(); HOPE.hyper_params.update({'method_name': 'hope_gsvd'})
        extra = dict(beta_over_rho=args.beta_over_rho) if rmat else {}
        model = HOPE(d=args.d, beta=args.beta, device=local, svd_error_probes=False, strict=False, **extra, **solver)
        model.learn_embedding(graph=hc, out=out)                      # warm-up
        # K plugin calls, each timed on the host clock around the whole call (H2D of the CSR, solve, D2H of X).
        # The GPU boxes show bursts of host-side stalls (a 9 ms D2H wait returning after 600 ms, with the device
        # idle) that have nothing to do with this process, so the reported step time is the MEDIAN call; the
        # mean, min and max are given beside it.
        ksteps = args.steps
        step_ms = []
        for _ in range(ksteps):
            dist_barrier(dist, local)
            t0 = time.perf_counter()
            X = model.learn_embedding(graph=hc, is_weighted=True, no_python=True, out=out)
            _ = float(X[0, 0])
            step_ms.append(dist_max(dist, (time.perf_counter() - t0) * 1e3, local))
        e2e_s = float(np.median(step_ms)) * 1e-3
        e2e = {'value': csr.n / e2e_s, 'unit': 'nodes/s', 'ms_per_step': e2e_s * 1e3, 'stat': 'median of %d calls' % ksteps,
               'mean_ms_per_step': float(np.mean(step_ms)), 'min_ms_per_step': float(np.min(step_ms)),
               'max_ms_per_step': float(np.max(step_ms)), 'value_from_mean': csr.n / (float(np.mean(step_ms)) * 1e-3),
               'h2d_bytes_per_step': int(4 * (n_own + 1) + 4 * int(csr.indptr[min(csr.n, (rank + 1) * ((csr.n + world - 1) // world))]
                                                                  - csr.indptr[rank * ((csr.n + world - 1) // world)])),
               'd2h_bytes_per_step': int(out.nbytes + 4 * (args.d // 2)), 'steps': ksteps,
               'per_call_setup_included': 'halo plan + IPC mapping of the work blocks (context and NCCL communicator are created by the first call and kept)' if world > 1 else 'ctx',
               'call': 'gem_b200.embedding.hope.HOPE(d, beta).learn_embedding(graph=<CSR in pinned host memory>)'
                       + (' on every rank (SPMD, rows of X per rank)' if world > 1 else '')}
        if world == 1 and not args.no_accuracy:
            accuracy = fp64_accuracy_of_solution(csr, np.asarray(X), model._sigma, float(model._beta), katz_terms=40 if rmat else 14)

    cpu = None
    if rank == 0 and not args.no_cpu:
        if rmat:
            cpu = cpu_hope_rmat_sample(args.cpu_rmat_scale, args.d, args.beta_over_rho)
        else:
            n_s = args.cpu_sample or 100000
            v, dt, info = cpu_hope_sample(n_s, args.d, args.beta, CPU_ARPACK_TOL)
            cpu = {'value': v, 'unit': 'nodes/s', 'cores': info['threads'], 'kind': 'port', 'host_cores': os.cpu_count(),
                   'seconds': dt,
                   'sample': 'SBM n=%d (same density, seed 42), d=%d, beta=%g: scipy svds(tol=%g, ARPACK) over the matrix-free fp64 '
                             'Katz operator (oracle/hope_oracle.hope_sparse, operator on %d OpenMP threads), J=%d, %d SpMVs; the '
                             'full 1M-node solve is what `--impl reference` times' % (
                                 n_s, args.d, args.beta, CPU_ARPACK_TOL, info['threads'], info['katz_terms'], info['spmv'])}
    if g is not None:
        g.free()
    line = None
    if rank == 0:
        mg = {0: 'single GPU', 1: 'row-sharded CSR x%d, ncclAllGather of the block per SpMM' % world,
              2: 'row-sharded CSR x%d; needed rows only, stored into the peers\' halo slots over NVLink (CUDA IPC) by the '
                 'producing kernel; b x b Gram all-reduce on NCCL' % world}
        mg[3] = mg[2] + '; halo copies travel as fp16'
        mg = mg[stats.get('mg_mode', 0)]
        line = {'metric': 'nodes/sec embedded at d=128', 'value': value, 'unit': 'nodes/s', 'n_gpus': world,
                'steps': args.steps, 'warmup': args.warmup, 'ms_per_step': dev_ms / args.steps,
                'higher_is_better': True, 'scaling': 'strong' if rmat else 'weak', 'vs_baseline': None, 'dtype': 'f32',
                'data': 'synthetic',
                'config': {'workload': ('HOPE d=%d beta=%g/rho_hat(A) = %.6g on %s: n=%d' % (args.d, args.beta_over_rho, stats.get('beta_used', 0.0), rmat_name(args), n_all))
                                       if rmat else hope_workload_name(args.d, args.beta, n, world), 'nnz': nnz_all,
                           'rho_hat': (args.beta_over_rho / stats['beta_used']) if rmat and stats.get('beta_used') else None,
                           'solver': dict(solver, block=stats['block'], katz_terms=stats['katz_terms'],
                                          iters=stats['iters'], converged=stats['converged'],
                                          ritz_change=stats['ritz_change'], resid_max_rel_sigma_max=resid_max,
                                          accuracy_vs_fp64=accuracy,
                                          algorithm={1: 'subspace iteration on S^T S (Katz sweeps)',
                                                     2: 'Chebyshev-filtered subspace iteration on A (S = f(A), A symmetric)',
                                                     3: 'thick-restart block Lanczos on A (S = f(A), A symmetric)'}
                                          .get(stats['algorithm'], stats['algorithm'])),
                           'parallelism': mg,
                           'exchange': None if world == 1 else {'halo_rows_rank0': stats.get('halo_rows'), 'push_rows_rank0': stats.get('push_rows'),
                                                                'blocks_exchanged_per_step': stats.get('pushes', 0) / args.steps,
                                                                'nvlink_bytes_out_per_step_rank0': stats.get('push_bytes', 0.0) / args.steps,
                                                                'wire': 'fp16 (x 2^12) for the filter / basis blocks, fp32 for the raw warm-up blocks' if stats.get('mg_mode') == 3 else 'fp32'},
                           'l2_policy': 'inputs larger than L2 (CSR %.0f MB + 5 blocks of %.0f MB vs 50 MB L2)' % (
                               (nnz_all * 4 + n_all * 4) / 1e6 / world, n_all * stats['block'] * 4 / 1e6 / world)},
                'wall_ms_per_step': wall_s * 1e3 / args.steps, 'graph_gen_s': gen_s,
                'phases_ms_per_step': {'spmm': stats['spmm_ms'] / args.steps, 'dense': stats['dense_ms'] / args.steps,
                                       'comm': stats['comm_ms'] / args.steps},
                'gpu_launches': int(launches), 'clocks': clocks, 'roofline': roofline, 'e2e': e2e, 'cpu_baseline': cpu}
    ctx.close()
    return line


def run_node2vec(args, dist, rank, world, local):
    from gem_b200 import _native, synth
    from gem_b200.embedding.node2vec import node2vec
    peaks, peak_src = read_peaks()
    rmat = args.graph == 'rmat'
    ctx = _native.Context(local)
    if world > 1:
        uid = [_native.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        ctx.comm_init(rank, world, uid[0])
    if rmat:
        # BASELINE.json configs[4]: the whole graph replicated on every GPU (generated there), walk starts sharded.
        # Half of an R-MAT's vertices have no edge at all: like the reference (whose edge-list file never mentions them)
        # only vertices with edges are in the node table, get walks and count as embedded.
        from gem_b200.graph import HostCSR
        n = 1 << args.scale
        ip, ix, _tot = _native.synth_rmat(ctx, args.scale, seed=42)
        csr = HostCSR(n, ip, ix, None, symmetric=True)
        nids = np.flatnonzero(np.diff(ip) > 0).astype(np.int32)
    else:
        n = args.n * world
        csr = synth.sbm(n=n, block=1000, seed=42)
        nids = np.arange(csr.n, dtype=np.int32)
    n_emb = int(nids.shape[0])
    g = _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, None)
    hp = (args.d, args.walk_len, args.num_walks, args.con_size, 1)
    # warm-up: full-size steps are ~10 s each; warm the kernels on short walks of the same graph
    for _ in range(args.warmup):
        g.node2vec(nids, args.d, 8, 1, 4, 1, seed=1, want_output=False)
    dist_barrier(dist, local)
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    launches0 = _native.lib().gemb_launch_count()
    dev_ms, agg = 0.0, None
    for s in range(args.steps):
        want = bool(args.dump_outputs) and s == args.steps - 1
        X_last, st = g.node2vec(nids, *hp, seed=1 + s, want_output=want)
        dev_ms += st['total_ms'] - (st['d2h_ms'] if want else 0.0)       # total_ms includes the copy of X to the host
        agg = st if agg is None else {k: agg[k] + st[k] for k in st}
    dist_barrier(dist, local)
    launches = _native.lib().gemb_launch_count() - launches0
    clocks = sampler.stop() if rank == 0 else None
    dev_ms = dist_max(dist, dev_ms, local)
    pairs = dist_sum(dist, float(agg['pairs']), local)
    value = n_emb * args.steps / (dev_ms * 1e-3)
    if args.dump_outputs and rank == 0:
        rows, Xs = row_sample(X_last)
        dump_outputs(args.dump_outputs, {'node2vec_X_rows': rows, 'node2vec_X': Xs})
    sg_bytes = pairs * 14 * 4 * args.d
    achieved = sg_bytes / world / (agg['sgns_ms'] * 1e-3) / 1e9 if agg['sgns_ms'] > 0 else 0.0
    roofline = {'kernel': 'sgns (warp per walk, fp32 tables)', 'bound': 'hbm', 'achieved': achieved,
                'peak': peaks['hbm_gbs'], 'unit': 'GB/s', 'frac': achieved / peaks['hbm_gbs'],
                'traffic': None,
                'peak_source': peak_src, 'bytes_per_launch': sg_bytes / world / args.steps,
                'ms_per_launch': agg['sgns_ms'] / args.steps, 'share_of_step': agg['sgns_ms'] / max(dev_ms, 1e-9),
                'note': 'algorithmic bytes = 7168 B per (centre, context) pair (SURVEY 8(d)); rows of the walk and the '
                        'centre row are reused from L1/L2/registers, so achieved may exceed the DRAM peak'}
    e2e = None
    if world == 1 and not args.no_e2e:
        node2vec.hyper_params.clear(); node2vec.hyper_params.update({'method_name': 'node2vec_rw'})
        model = node2vec(d=args.d, max_iter=1, walk_len=args.walk_len, num_walks=args.num_walks,
                         con_size=args.con_size, ret_p=1, inout_p=1, device=local)
        step_ms = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            X = model.learn_embedding(graph=(csr, nids))
            _ = float(X[0, 0])
            step_ms.append((time.perf_counter() - t0) * 1e3)
        e2e_s = float(np.median(step_ms)) * 1e-3
        e2e = {'value': n_emb / e2e_s, 'unit': 'nodes/s', 'ms_per_step': e2e_s * 1e3, 'stat': 'median of %d calls' % len(step_ms),
               'h2d_bytes_per_step': int(4 * (csr.n + 1) + 4 * csr.nnz + 4 * n_emb * args.num_walks),
               'd2h_bytes_per_step': int(4 * csr.n * args.d), 'steps': len(step_ms),
               'call': 'gem_b200.embedding.node2vec.node2vec(...).learn_embedding(graph=(CSR, node table))'}
    cpu = None
    if rank == 0 and not args.no_cpu:
        n_s = args.n2v_cpu_sample or 2000
        scsr = None
        if rmat:
            scsr = synth.rmat(scale=11, seed=42)
            n_s = int((np.diff(scsr.indptr) > 0).sum())
        v, dt, kind, used = cpu_n2v_sample(n_s, args.d, args.walk_len, args.num_walks, args.con_size, os.cpu_count() or 1, csr=scsr)
        cpu = {'value': v, 'unit': 'nodes/s', 'cores': used, 'kind': kind, 'host_cores': os.cpu_count(), 'seconds': dt,
               'sample': '%s, d=%d r=%d l=%d k=%d e=1 p=q=1 (%s)' % (
                   ('R-MAT scale 11 (host generator, seed 42; %d vertices with edges -- the reference binary builds one alias '
                    'table per directed edge, sum deg^2 entries: it cannot hold scale 24)' % n_s) if rmat
                   else 'SBM n=%d (same density, seed 42)' % n_s, args.d, args.num_walks, args.walk_len, args.con_size,
                   'gem/c_exe/node2vec, OMP threads = cores' if kind == 'reference' else 'oracle/n2v_oracle.c, 1 thread')}
    g.free()
    line = None
    if rank == 0:
        line = {'metric': 'nodes/sec embedded at d=128', 'value': value, 'unit': 'nodes/s', 'n_gpus': world,
                'steps': args.steps, 'warmup': args.warmup, 'ms_per_step': dev_ms / args.steps,
                'higher_is_better': True, 'scaling': 'strong' if rmat else 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
                'config': {'workload': 'node2vec d=%d p=q=1, %d walks x %d, context %d, 1 epoch, 5 negatives, on %s n=%d, nnz=%d; %d vertices have edges (node table, walks, value)'
                                       % (args.d, args.num_walks, args.walk_len, args.con_size, rmat_name(args) if rmat else 'SBM', n, csr.nnz, n_emb),
                           'parallelism': 'walk-sharded x%d, embedding-delta all-reduce per epoch' % world if world > 1 else 'single GPU',
                           'l2_policy': 'inputs larger than L2 (two %d MB embedding tables + %d MB walks vs 50 MB L2)' % (
                               csr.n * args.d * 4 // 10**6, n_emb * args.num_walks * args.walk_len * 4 // 10**6 // world)},
                'phases_ms_per_step': {k: agg[k] / args.steps for k in ('alias_ms', 'shuffle_ms', 'walk_ms', 'vocab_ms', 'sgns_ms', 'comm_ms')},
                'gpu_launches': int(launches), 'clocks': clocks, 'roofline': roofline, 'e2e': e2e, 'cpu_baseline': cpu}
    ctx.close()
    return line if rank == 0 else None


def run_recon(args, dist, rank, world, local):
    """SURVEY 8(f) rank 1.  Each rank evaluates its own replica (the path has no exchange step: 'replicas only')."""
    import ctypes
    from gem_b200 import _native, synth
    from gem_b200.embedding.hope import HOPE
    from gem_b200.evaluation import metrics
    from gem_b200.evaluation.evaluate_graph_reconstruction import evaluateStaticGraphReconstruction
    peaks, peak_src = read_peaks()
    n = args.recon_n
    csr = synth.sbm(n=n, block=1024 if n % 1024 == 0 else 1000, seed=42)
    ctx = _native.Context(local)
    g = _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, None)
    X, _, _ = g.hope(args.d, args.beta, tol=1e-4, max_iters=40, seed=1234)       # the embedding to evaluate (not timed)
    g.free()
    ip32, ix32 = csr.indptr.astype(np.int32), csr.indices.astype(np.int32)
    lib = _native.lib()
    K = 1000

    def step():
        rec = _native.Reconstruction(ctx, X, True)
        t_sel = time.perf_counter()
        m = ctypes.c_int64(0)
        _native.check(lib.gemb_recon_top(rec._h, 1, K, 0, None, None, None, ctypes.byref(m)))   # the counting passes
        t_sel = time.perf_counter() - t_sel
        ti, tj, tw = rec.top(True, K)
        ranks, npr = rec.ranks(ip32, ix32, True)
        rec.free()
        return t_sel, ranks, (ti, tj, tw)

    for _ in range(args.warmup):
        step()
    dist_barrier(dist, local)
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    l0 = lib.gemb_launch_count()
    t0 = time.perf_counter()
    sel_s = 0.0
    for s in range(args.steps):
        ts, ranks, top = step()
        sel_s += ts
    dist_barrier(dist, local)
    wall = time.perf_counter() - t0
    launches = lib.gemb_launch_count() - l0
    clocks = sampler.stop() if rank == 0 else None
    wall = dist_max(dist, wall, local)
    value = world * float(n) * n * args.steps / wall
    if args.dump_outputs and rank == 0:
        # gemb_recon_top returns the candidates unordered (compaction order); the caller orders them by weight descending,
        # then i, then j (include/gemb200.h) -- so does the dump
        o = np.lexsort((top[1], top[0], -top[2]))
        dump_outputs(args.dump_outputs, {'recon_edge_ranks': ranks.astype(np.float64), 'recon_top_i': top[0][o].astype(np.float64),
                                         'recon_top_j': top[1][o].astype(np.float64), 'recon_top_w': top[2][o]})
    n_pad = (n + 63) // 64 * 64
    passes = 32                                            # 1 total count + 31 bisection steps per selection
    bytes_per_launch = 4.0 * n * n_pad
    sel_ms = 1e3 * sel_s / (args.steps * passes)
    achieved = bytes_per_launch / (sel_ms * 1e-3) / 1e9
    roofline = {'kernel': 'recon_select_kernel<false> (count entries >= T over the n x n reconstruction)', 'bound': 'hbm',
                'achieved': achieved, 'peak': peaks['hbm_gbs'], 'unit': 'GB/s', 'frac': achieved / peaks['hbm_gbs'],
                'traffic': None, 'peak_source': peak_src, 'bytes_per_launch': bytes_per_launch, 'ms_per_launch': sel_ms,
                'launches_per_step': passes, 'share_of_step': sel_s / max(wall, 1e-9),
                'note': 'timed on the host clock around the blocking C call that runs the 32 counting passes (each pass = '
                        'one launch + an 8-byte D2H + stream sync), not with per-kernel events'}
    e2e = None
    if world == 1 and not args.no_e2e:
        HOPE.hyper_params.clear(); HOPE.hyper_params.update({'method_name': 'hope_gsvd'})
        model = HOPE(d=args.d, beta=args.beta, device=local)
        evaluateStaticGraphReconstruction(csr, model, X, None, max_k=K)
        step_ms = []
        for _ in range(args.steps):
            t1 = time.perf_counter()
            MAP, prec, _, _ = evaluateStaticGraphReconstruction(csr, model, X, None, max_k=K)
            step_ms.append((time.perf_counter() - t1) * 1e3)
        med = float(np.median(step_ms))
        e2e = {'value': float(n) * n / (med * 1e-3), 'unit': 'pairs/s', 'ms_per_step': med, 'stat': 'median of %d calls' % len(step_ms),
               'mean_ms_per_step': float(np.mean(step_ms)), 'h2d_bytes_per_step': int(X.nbytes + ip32.nbytes + ix32.nbytes),
               'd2h_bytes_per_step': int(4 * csr.nnz + 4 * n + 12 * K), 'MAP': MAP, 'precision_at_1000': prec[-1] if prec else None,
               'call': 'gem_b200.evaluation.evaluate_graph_reconstruction.evaluateStaticGraphReconstruction(csr, model, X, None, max_k=1000)'}
    cpu = None
    if rank == 0 and not args.no_cpu:
        n_s = args.cpu_sample or 8192
        v, dt = cpu_recon_sample(n_s, args.d)
        cpu = {'value': v, 'unit': 'pairs/s', 'cores': 1, 'kind': 'port', 'host_cores': os.cpu_count(), 'seconds': dt,
               'sample': 'SBM n=%d, random X (d=%d): oracle/eval_oracle.py, the vectorised restatement of gem.evaluation '
                         '(BLAS GEMM may use several threads)' % (n_s, args.d)}
    if rank == 0:
        line = {'metric': 'node pairs evaluated/sec (reconstruction + MAP + precision@1000)', 'value': value, 'unit': 'pairs/s',
                'n_gpus': world, 'steps': args.steps, 'warmup': args.warmup, 'ms_per_step': 1e3 * wall / args.steps,
                'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
                'config': {'workload': 'reconstruction evaluation of a HOPE d=%d embedding, SBM n=%d nnz=%d, undirected, max_k=%d'
                                       % (args.d, n, csr.nnz, K),
                           'parallelism': 'single GPU' if world == 1 else 'replicas only (%d independent evaluations)' % world,
                           'l2_policy': 'inputs larger than L2 (reconstruction %.1f GB vs 50 MB L2)' % (bytes_per_launch / 1e9)},
                'gpu_launches': int(launches), 'clocks': clocks, 'roofline': roofline, 'e2e': e2e, 'cpu_baseline': cpu}
        print(json.dumps(line), flush=True)
    ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=None)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
    ap.add_argument('--workload', default='hope', choices=['hope', 'node2vec', 'recon'])
    ap.add_argument('--n', type=int, default=1_000_000, help='nodes per GPU')
    ap.add_argument('--graph', default='sbm', choices=['sbm', 'rmat'], help='rmat: BASELINE.json configs[3]/[4] (fixed graph, --scale)')
    ap.add_argument('--scale', type=int, default=24, help='R-MAT scale (2^scale nodes, 8 * 2^scale undirected pairs)')
    ap.add_argument('--beta-over-rho', type=float, default=0.5, help='R-MAT HOPE: beta = this / rho_hat(A)')
    ap.add_argument('--cpu-rmat-scale', type=int, default=14, help='R-MAT scale of the CPU baseline sample')
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--beta', type=float, default=0.01)
    ap.add_argument('--tol', type=float, default=None)
    ap.add_argument('--max-iters', type=int, default=None)
    ap.add_argument('--walk-len', type=int, default=80)
    ap.add_argument('--num-walks', type=int, default=10)
    ap.add_argument('--con-size', type=int, default=10)
    ap.add_argument('--recon-n', type=int, default=32768, help='nodes of the reconstruction workload')
    ap.add_argument('--cpu-sample', type=int, default=None, help='nodes in the CPU baseline sample')
    ap.add_argument('--n2v-cpu-sample', type=int, default=None, help='nodes in the node2vec CPU baseline sample')
    ap.add_argument('--no-node2vec', action='store_true', help='HOPE line without the node2vec sub-record')
    ap.add_argument('--no-accuracy', action='store_true', help='skip the fp64 host check of the timed solution')
    ap.add_argument('--no-e2e', action='store_true')
    ap.add_argument('--no-cpu', action='store_true')
    ap.add_argument('--dump-outputs', default=None, metavar='DIR',
                    help='after the timed steps, write the outputs of the last timed step as DIR/<name>.npy')
    args = ap.parse_args()
    if args.steps is None:
        args.steps = {'hope': 20, 'recon': 5}.get(args.workload, 1)
    if args.steps < 1:
        ap.error('--steps must be >= 1')
    if args.impl == 'reference':
        args.warmup_requested = args.warmup
        args.warmup = min(args.warmup, 1)      # each CPU step is a bounded 10-30 s sample (HOPE: a full solve, no warm-up)
        run_reference(args)
        return
    dist, rank, world, local = dist_setup(args.gpus)
    try:
        if args.workload == 'hope':
            line = run_hope(args, dist, rank, world, local)
            if not args.no_node2vec and args.graph != 'rmat':
                # BASELINE.json configs[2] rides in the same line: one epoch (= one step, several seconds), whatever --steps
                # says for the HOPE record; the sub-record states its own "steps"
                steps, warm, dump = args.steps, args.warmup, args.dump_outputs
                args.steps, args.warmup, args.dump_outputs = 1, min(args.warmup, 3), None
                sub = run_node2vec(args, dist, rank, world, local)
                args.steps, args.warmup, args.dump_outputs = steps, warm, dump
                if line is not None:
                    line['node2vec'] = sub
                    line['gpu_launches'] += sub['gpu_launches']
            if line is not None:
                print(json.dumps(line), flush=True)
        elif args.workload == 'recon':
            run_recon(args, dist, rank, world, local)
        else:
            line = run_node2vec(args, dist, rank, world, local)
            if line is not None:
                print(json.dumps(line), flush=True)
    finally:
        if dist is not None:
            dist.destroy_process_group()


if __name__ == '__main__':
    main()
