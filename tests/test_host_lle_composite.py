"""The host side of LocallyLinearEmbedding's composite operator (gem_b200/embedding/lle.py): the uploaded P = D^-1 W and its
transpose are the M = I - P of the explicit form and of the fp64 oracle, and 'auto' picks the form by the documented
bound sum_v deg(v)^2 + n <= 2^31 - 1.  CPU only."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import REPO, golden_path

sys.path.insert(0, os.path.join(REPO, 'oracle'))
import lle_oracle as le


def _adj(name, d):
    z = np.load(golden_path('ref_lle_%s_d%d.npz' % (name, d)))
    e, n = z['edges'], int(z['n'])
    return sp.csr_matrix((e[:, 2], (e[:, 0].astype(int), e[:, 1].astype(int))), shape=(n, n))


@pytest.mark.parametrize('name,d', [('karate', 4), ('sbm1024', 16), ('randw120', 8)])
def test_uploaded_operator_is_the_oracles(name, d):
    from gem_b200 import graph as hg
    from gem_b200.embedding.lle import lle_composite_operator, lle_operator, choose_operator
    A = _adj(name, d)
    csr = hg.from_scipy(A)
    P, PT = lle_composite_operator(csr)
    Ps, PTs = P.to_scipy(), PT.to_scipy()
    M = le.lle_matrix(A)
    n = A.shape[0]
    assert abs((sp.identity(n) - Ps) - M).max() < 1e-15
    assert abs(PTs - Ps.T).max() == 0.0
    assert not P.symmetric and not PT.symmetric
    C, c = lle_operator(csr)
    assert abs(C.to_scipy() - (c * sp.identity(n) - M.T @ M)).max() < 1e-12 * c
    assert choose_operator(csr) == 'explicit'


def test_auto_switches_above_the_entry_bound():
    from gem_b200 import graph as hg
    from gem_b200.embedding.lle import choose_operator
    for leaves, want in ((46339, 'explicit'), (46341, 'composite')):
        n = leaves + 1                          # a star: sum deg^2 + n = leaves^2 + 2 leaves + 1
        A = sp.csr_matrix((np.ones(leaves), (np.zeros(leaves, dtype=int), np.arange(1, n))), shape=(n, n))
        csr = hg.from_scipy(A)
        assert choose_operator(csr) == want, (leaves, leaves ** 2 + 2 * leaves + 1)
        assert choose_operator(csr, 'explicit') == 'explicit'
        assert choose_operator(csr, 'composite') == 'composite'
    with pytest.raises(ValueError, match='operator must be'):
        choose_operator(csr, 'dense')
