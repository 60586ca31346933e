"""Host side of t-SNE without a GPU: every ValueError of tsne() comes before any device call, there is no CPU
fallback, plot_embedding2D names matplotlib when it is missing, and importing the product loads neither sklearn nor
matplotlib."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import REPO


@pytest.fixture
def no_device(monkeypatch):
    """Fail loudly if tsne reaches the library."""
    from gem_b200 import _native

    def boom(*a, **k):
        raise AssertionError('device call before validation')
    monkeypatch.setattr(_native, 'Context', boom)
    monkeypatch.setattr(_native, 'lib', boom)


X = np.random.RandomState(0).randn(40, 5)


@pytest.mark.parametrize('bad', [
    dict(X=X[:, 0]),                                     # not 2-D
    dict(X=X[:1]),                                       # n < 2
    dict(X=X[:, :0]),                                    # d < 1
    dict(X=np.where(X > 1, np.nan, X)),                  # not finite
    dict(X=np.where(X > 1, np.inf, X)),
    dict(X=np.random.RandomState(1).randn(100, 1025).astype(np.float32)),   # d above the PCA eigensolver's 1024
    dict(perplexity=40.0),                               # perplexity >= n
    dict(perplexity=0.0),
    dict(perplexity=-3.0),
    dict(max_iter=249),                                  # sklearn's bound
    dict(angle=-0.1),
    dict(angle=1.01),
    dict(learning_rate=0.0),
    dict(learning_rate=-10.0),
    dict(learning_rate='fast'),
    dict(early_exaggeration=0.0),
    dict(min_grad_norm=-1.0),
], ids=['x1d', 'n1', 'd0', 'nan', 'inf', 'd1025', 'perp-n', 'perp0', 'perp-neg', 'max_iter', 'angle-neg', 'angle-big', 'lr0',
        'lr-neg', 'lr-str', 'exag0', 'min_grad_norm'])
def test_value_errors_before_any_device_call(no_device, bad):
    from gem_b200.evaluation.visualize_embedding import tsne
    args = dict(X=X)
    args.update(bad)
    with pytest.raises(ValueError):
        tsne(args.pop('X'), **args)


def test_no_cpu_fallback(native_lib):
    if native_lib.gemb_device_count() > 0:
        pytest.skip('a GPU is present')
    from gem_b200.evaluation.visualize_embedding import tsne
    with pytest.raises(RuntimeError):
        tsne(X)


def test_plot_needs_matplotlib(monkeypatch, no_device):
    from gem_b200.evaluation.visualize_embedding import plot_embedding2D
    monkeypatch.setitem(sys.modules, 'matplotlib', None)
    monkeypatch.setitem(sys.modules, 'matplotlib.pyplot', None)
    with pytest.raises(ImportError, match='matplotlib'):
        plot_embedding2D(X)


def test_product_imports_neither_sklearn_nor_matplotlib():
    code = ('import sys, gem_b200, gem_b200.evaluation.visualize_embedding, gem_b200.evaluation.evaluate_node_classification; '
            'print(sorted(m for m in sys.modules if m.split(".")[0] in ("sklearn", "matplotlib")))')
    out = subprocess.run([sys.executable, '-c', code], cwd=REPO, capture_output=True, text=True, check=True).stdout
    assert out.strip() == '[]'
