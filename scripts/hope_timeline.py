"""scripts/hope_timeline.py -- where one Chebyshev HOPE solve of the bench setting spends its time on the GPU.

    python scripts/hope_timeline.py --out DIR [--solves 10] [--lib PATH/libgemb200.so]
    python scripts/hope_timeline.py --out DIR --compare OLD/libgemb200.so [--rounds 3]

One process: the bench graph (SBM, 1M nodes), 3 warm-up solves with bench.HOPE_SOLVER, then
  1. `--solves` timed solves: total_ms / spmm_ms / dense_ms per solve and their min / median / max;
  2. 3 more solves under torch.profiler (CUDA activities), reduced to a per-kernel table -- launches per solve, total and
     mean microseconds, achieved GB/s of the streaming kernels from their compulsory bytes -- and the idle time of the
     stream per solve, split into gaps next to a device-to-host copy (a host round trip) and all others;
  3. the card: name, power limit, max SM clock (nvidia-smi query).
Everything is printed and saved as DIR/timeline.json; the raw trace is DIR/hope.pt.trace.json.

--lib loads another build of the library instead of the tree's (ctypes path override, nothing in the package changes).
--compare alternates that build and the tree's build, `--rounds` child processes each running part 1, and prints the
medians, the spreads and the difference.  There is no CPU fallback: without a CUDA device the script fails."""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

D, BETA, N, WARMUP, PROFILED = 128, 0.01, 1_000_000, 3, 3


def spread(xs):
    return {'min': min(xs), 'median': statistics.median(xs), 'max': max(xs)}


def card():
    out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                                   '-i', '0'], text=True).strip().splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(',')]
    return {'name': name, 'power_limit': power, 'max_sm_clock': clock}


def short_name(name):
    """'void gemb::gram_tc_kernel<true, true, 80>(gemb::GramTcParams)' -> 'gram_tc_kernel<true, true, 80>'."""
    name = re.sub(r'^void\s+', '', name)
    depth, cut = 0, len(name)
    for i, ch in enumerate(name):      # cut at the argument list: the first '(' outside the template brackets
        if ch == '<':
            depth += 1
        elif ch == '>':
            depth -= 1
        elif ch == '(' and depth == 0:
            cut = i
            break
    return name[:cut].replace('gemb::', '').replace('(anonymous namespace)::', '')


def pad_width(w):
    return next((p for p in (32, 64, 80, 96, 128) if p >= w), 128)


def streamed_bytes(name, n, b, d):
    """Compulsory HBM bytes of one launch of a streaming kernel at the bench shapes (None: not a streaming kernel)."""
    blk = 4.0 * n * b
    m = re.match(r'gram_tc_kernel<(true|false), (true|false), (\d+)>', name)
    if m:
        return blk * (2 if m.group(1) == 'true' else 1)          # V^T AV reads two blocks, a block's own Gram one
    m = re.match(r'apply_tc_kernel<\d+, (\d+)>', name)
    if m:
        out_cols = {pad_width(b): b, pad_width(d // 2): d // 2, pad_width(d): d}.get(int(m.group(1)))
        return None if out_cols is None else blk + 4.0 * n * out_cols
    if name.startswith('axpby_kernel'):
        return 3 * blk
    return None


def reduce_trace(path, n, b, d, solves):
    with open(path) as f:
        events = [e for e in json.load(f)['traceEvents']
                  if e.get('ph') == 'X' and e.get('cat') in ('kernel', 'gpu_memcpy', 'gpu_memset')]
    events.sort(key=lambda e: e['ts'])
    rows = {}
    for e in events:
        name = short_name(e['name'])
        r = rows.setdefault(name, {'launches': 0, 'us': 0.0})
        r['launches'] += 1
        r['us'] += e['dur']
    table = []
    for name, r in sorted(rows.items(), key=lambda kv: -kv[1]['us']):
        row = {'kernel': name, 'launches_per_solve': r['launches'] / solves, 'us_per_solve': r['us'] / solves,
               'mean_us': r['us'] / r['launches']}
        nbytes = streamed_bytes(name, n, b, d)
        if nbytes:
            row['gb_per_s'] = nbytes / (row['mean_us'] * 1e-6) / 1e9
        table.append(row)
    # The timed part of a solve starts at the row-sum bound of the adjacency (the zero-fills of the work blocks come
    # before it) and ends before the zero-fills of the next call: gaps are counted inside these segments only.
    first = [i for i, e in enumerate(events) if 'csr_rowsum_kernel' in e['name']]
    assert len(first) == solves, 'expected one csr_rowsum_kernel per solve, saw %d' % len(first)
    gap_d2h = gap_other = span = busy = 0.0
    for s, lo in enumerate(first):
        hi = first[s + 1] if s + 1 < solves else len(events)
        while s + 1 < solves and events[hi - 1]['name'].startswith('Memset'):
            hi -= 1
        span += events[hi - 1]['ts'] + events[hi - 1]['dur'] - events[lo]['ts']
        busy += sum(e['dur'] for e in events[lo:hi])
        end = events[lo]['ts']
        for prev, cur in zip(events[lo:hi], events[lo + 1:hi]):
            end = max(end, prev['ts'] + prev['dur'])      # kernels of the side stream overlap those of the main one
            gap = cur['ts'] - end
            if gap <= 0:
                continue
            if 'DtoH' in prev['name'] or 'DtoH' in cur['name']:
                gap_d2h += gap
            else:
                gap_other += gap
    return {'kernels': table, 'busy_us_per_solve': busy / solves,
            'span_us_per_solve': span / solves,
            'idle_us_per_solve': {'next_to_d2h_copy': gap_d2h / solves, 'other': gap_other / solves}}


def run_solves(args):
    import bench
    from gem_b200 import _native, synth
    if args.lib:
        _native.LIB_PATH = os.path.abspath(args.lib)
    if _native.lib().gemb_device_count() < 1:
        raise RuntimeError('hope_timeline needs a CUDA device (there is no CPU fallback)')
    csr = synth.sbm(n=N, block=1000, seed=42)
    ctx = _native.Context(0)
    r0, ip, ix, _ = csr.row_shard(0, 1)
    g = _native.DeviceGraph(ctx, csr.n, ip, ix, None, row0=r0)
    solve = lambda: g.hope(D, BETA, want_output=False, **bench.HOPE_SOLVER)[2]
    for _ in range(WARMUP):
        solve()
    stats = [solve() for _ in range(args.solves)]
    res = {'lib': _native.LIB_PATH, 'card': card(), 'n': N, 'd': D, 'block': stats[0]['block'],
           'iters': stats[0]['iters'], 'spmm_count': stats[0]['spmm_count'],
           'solves': [{k: st[k] for k in ('total_ms', 'spmm_ms', 'dense_ms')} for st in stats]}
    for k in ('total_ms', 'spmm_ms', 'dense_ms'):
        res[k] = spread([st[k] for st in stats])
    if not args.timed_only:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        trace = os.path.join(args.out, 'hope.pt.trace.json')
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(PROFILED):
                solve()
            torch.cuda.synchronize()
        prof.export_chrome_trace(trace)
        res['profile'] = reduce_trace(trace, N, stats[0]['block'], D, PROFILED)
    g.free()
    ctx.close()
    return res


def print_result(res):
    print('card: %(name)s, power limit %(power_limit)s, max SM clock %(max_sm_clock)s' % res['card'])
    print('library: %s   block %d, %d rounds, %d SpMM sweeps per solve' % (res['lib'], res['block'], res['iters'], res['spmm_count']))
    for i, s in enumerate(res['solves']):
        print('solve %2d  total %.3f ms  spmm %.3f ms  dense %.3f ms' % (i, s['total_ms'], s['spmm_ms'], s['dense_ms']))
    for k in ('total_ms', 'spmm_ms', 'dense_ms'):
        print('%-9s min %.3f  median %.3f  max %.3f' % (k, res[k]['min'], res[k]['median'], res[k]['max']))
    p = res.get('profile')
    if not p:
        return
    print('%-58s %9s %12s %10s %8s' % ('kernel / copy (profiled, per solve)', 'launches', 'total us', 'mean us', 'GB/s'))
    for r in p['kernels']:
        print('%-58s %9.1f %12.1f %10.1f %8s' % (r['kernel'][:58], r['launches_per_solve'], r['us_per_solve'], r['mean_us'],
                                                '%.0f' % r['gb_per_s'] if 'gb_per_s' in r else ''))
    print('per solve: span %.1f us, busy %.1f us, idle next to a D2H copy %.1f us, other idle %.1f us'
          % (p['span_us_per_solve'], p['busy_us_per_solve'], p['idle_us_per_solve']['next_to_d2h_copy'],
             p['idle_us_per_solve']['other']))


def compare(args):
    libs = {'old': os.path.abspath(args.compare), 'new': None}
    runs = {'old': [], 'new': []}
    for _ in range(args.rounds):
        for tag, lib in libs.items():
            cmd = [sys.executable, os.path.abspath(__file__), '--out', args.out, '--solves', str(args.solves), '--timed-only', '--json']
            out = subprocess.check_output(cmd + (['--lib', lib] if lib else []), text=True)
            runs[tag].append(json.loads(out.strip().splitlines()[-1]))
    res = {'card': runs['new'][0]['card'], 'runs': runs}
    print('card: %(name)s, power limit %(power_limit)s, max SM clock %(max_sm_clock)s' % res['card'])
    for k in ('total_ms', 'spmm_ms', 'dense_ms'):
        res[k] = {tag: spread([s[k] for r in runs[tag] for s in r['solves']]) for tag in runs}
        for tag in runs:
            print('%-9s %s  min %.3f  median %.3f  max %.3f  (%d solves in %d processes; process medians %s)'
                  % (k, tag, res[k][tag]['min'], res[k][tag]['median'], res[k][tag]['max'],
                     sum(len(r['solves']) for r in runs[tag]), len(runs[tag]),
                     ' '.join('%.3f' % r[k]['median'] for r in runs[tag])))
        print('%-9s old - new (medians): %.3f ms' % (k, res[k]['old']['median'] - res[k]['new']['median']))
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--out', required=True, help='directory for timeline.json and the profiler trace')
    ap.add_argument('--solves', type=int, default=10)
    ap.add_argument('--lib', default=None, help='another build of libgemb200.so to load instead of the tree\'s')
    ap.add_argument('--compare', default=None, metavar='OLD_LIB', help='alternate OLD_LIB and the tree\'s build')
    ap.add_argument('--rounds', type=int, default=3, help='--compare: child processes per build')
    ap.add_argument('--timed-only', action='store_true', help='part 1 only (no profiler pass)')
    ap.add_argument('--json', action='store_true', help='print the result as one JSON line only')
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    if args.compare:
        res, name = compare(args), 'compare.json'
    else:
        res, name = run_solves(args), 'timeline.json'
        if args.json:
            print(json.dumps(res))
            return
        print_result(res)
    with open(os.path.join(args.out, name), 'w') as f:
        json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
