"""Host side of get_lcc on a HostCSR without a GPU: every malformed CSR is a ValueError before any device call, and
there is no CPU fallback."""
import numpy as np
import pytest


@pytest.fixture
def no_device(monkeypatch):
    """Fail loudly if get_lcc reaches the library."""
    from gem_b200 import _native

    def boom(*a, **k):
        raise AssertionError('device call before validation')
    monkeypatch.setattr(_native, 'Context', boom)
    monkeypatch.setattr(_native, 'lib', boom)


def _csr(indptr=(0, 1, 3, 3), indices=(1, 0, 2), n=3, data=None):
    from gem_b200.graph import HostCSR
    return HostCSR(n, np.array(indptr, dtype=np.int64), np.array(indices, dtype=np.int32), data)


def _huge():
    g = _csr()
    g.n = 2 ** 31
    return g


@pytest.mark.parametrize('make', [
    lambda: _csr(indptr=(0, 2, 1, 3)),                    # indptr not monotone
    lambda: _csr(indptr=(1, 1, 3, 3)),                    # indptr[0] != 0
    lambda: _csr(indices=(1, 0, 3)),                      # column id = n
    lambda: _csr(indices=(1, -1, 2)),                     # negative column id
    lambda: _csr(indptr=(0, 1, 3, 4)),                    # indptr runs past the indices
    lambda: _csr(data=np.ones(2)),                        # fewer weights than stored edges
    _huge,                                                # n >= 2^31
], ids=['non-monotone', 'indptr0', 'col-n', 'col-neg', 'short-indices', 'short-data', 'n-2^31'])
def test_value_errors_before_any_device_call(no_device, make):
    from gem_b200.utils.graph_util import get_lcc
    with pytest.raises(ValueError):
        get_lcc(make())


def test_no_cpu_fallback(native_lib):
    if native_lib.gemb_device_count() > 0:
        pytest.skip('a GPU is present')
    from gem_b200.utils.graph_util import get_lcc
    with pytest.raises(RuntimeError):
        get_lcc(_csr())
