"""Every kernel of libgemb200.so is launched through gemb::launch (common.cuh), which checks the launch and counts it in
gemb_launch_count: no source under gem_b200/csrc writes a triple-chevron launch of its own.  The only launches counted
by hand are the CUB calls, which launch their kernels internally; they are listed here per file."""
import glob
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'gem_b200', 'csrc')

# file -> number of count_launch( calls after CUB dispatches
CUB_COUNT_SITES = {'cc.cu': 1, 'halo.cu': 1, 'n2v.cu': 1, 'synth.cu': 2}


def _strip_comments(src):
    """The source with // and /* */ comments blanked out (string and character literals kept)."""
    out, i, n = [], 0, len(src)
    while i < n:
        c = src[i]
        if src.startswith('//', i):
            j = src.find('\n', i)
            i = n if j < 0 else j
        elif src.startswith('/*', i):
            j = src.find('*/', i + 2)
            i = n if j < 0 else j + 2
            out.append(' ')
        elif c in '"\'':
            j = i + 1
            while j < n and src[j] != c:
                j += 2 if src[j] == '\\' else 1
            out.append(src[i:j + 1])
            i = j + 1
        else:
            out.append(c)
            i += 1
    return ''.join(out)


def _sources():
    paths = sorted(glob.glob(os.path.join(CSRC, '*.cu')) + glob.glob(os.path.join(CSRC, '*.cuh')))
    assert paths, CSRC
    return {os.path.basename(p): _strip_comments(open(p).read()) for p in paths}


def _body(src, signature):
    """(start, end) of the braces of the function whose definition starts with `signature`; (0, 0) when there is none."""
    m = re.search(signature, src)
    if not m:
        return 0, 0
    start = src.index('{', m.end())
    depth = 0
    for j in range(start, len(src)):
        depth += {'{': 1, '}': -1}.get(src[j], 0)
        if depth == 0:
            return start, j + 1
    raise AssertionError('unbalanced braces after ' + signature)


def _cut(src, span):
    return src[:span[0]] + src[span[1]:]


def test_triple_chevron_only_in_launch():
    srcs = _sources()
    launch_src = srcs['common.cuh']
    span = _body(launch_src, r'\bint\s+launch\s*\(\s*const\s+gemb_ctx\b')
    found = {f: s.count('<<<') for f, s in srcs.items()}
    found['common.cuh'] = _cut(launch_src, span).count('<<<')
    assert {f: k for f, k in found.items() if k} == {}
    assert launch_src[span[0]:span[1]].count('<<<') == 1


def test_count_launch_only_after_cub_calls():
    srcs = _sources()
    core = srcs['core.cu']
    srcs['core.cu'] = _cut(core, _body(core, r'\bint\s+launch_status\s*\('))   # launch's out-of-line check counts there
    calls = {}
    for f, s in srcs.items():
        s = re.sub(r'\bvoid\s+count_launch\s*\(', '', s)                         # its declaration and definition
        k = len(re.findall(r'\bcount_launch\s*\(', s))
        if k:
            calls[f] = k
    assert calls == CUB_COUNT_SITES
