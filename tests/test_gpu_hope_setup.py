"""HOPE's set-up -- the beta a solve runs with, its Katz terms J and what bounds A's spectrum -- gives the same results
bit for bit on every path.

tests/golden/hope_setup.npz (make_golden_hope_setup.py) holds the output of the build that decided the set-up inline in
gemb_hope.  Each case here runs the same call and must return equal X rows, sigma, non-timing stats and launch count:
  - spectral_mode 0, beta > 0: the general solver with and without katz_terms, on a directed graph past the ||A||_2 bound
    (the series probe), with compute_residual and stop_rule 1; the Chebyshev solver on a non-negative symmetric graph
    (Ritz values bound the spectrum) and a signed one (power iteration); Lanczos, asked for and switched to;
  - spectral_mode 0, beta < 0 (|beta| / ||A||_2) on the general, Chebyshev (both bounds) and Lanczos solvers;
  - spectral_modes 1 (both bounds), 2 (the composite's power iteration) and 3-5;
  - gemb_hope_svd_error on a symmetric and a directed graph (the probe), gemb_hope_apply for every mode;
  - the refusals at the bound, after the probe, of |beta| >= 0.98 and of beta < 0 on an edge-free graph: status, message
    and launches.
The 'SVD error' sums its columns with fp64 atomics, so it is held to 1e-12 relative, its launches exactly."""
import sys

import numpy as np
import pytest

from conftest import GOLDEN, golden_path

sys.path.insert(0, GOLDEN)
import make_golden_hope_setup as mk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def gold():
    return np.load(golden_path('hope_setup.npz'))


@pytest.mark.parametrize('kind,name', mk.all_cases(), ids=['%s-%s' % c for c in mk.all_cases()])
def test_setup_path_is_bit_identical(gpu_ctx, gold, kind, name):
    got = mk.run(gpu_ctx, kind, name)
    if kind == 'refusal':
        assert mk.REFUSALS[name][-1] in str(got['message']), got['message']
    prefix = '%s/%s/' % (kind, name)
    assert sorted(got) == sorted(k[len(prefix):] for k in gold.files if k.startswith(prefix))
    for key, v in got.items():
        ref = gold[prefix + key]
        if kind == 'svd_error' and key == 'err':
            assert abs(float(v) - float(ref)) <= 1e-12 * abs(float(ref)), (key, float(v), float(ref))
        else:
            assert np.asarray(v).dtype == ref.dtype and np.array_equal(v, ref), (key, v, ref)
