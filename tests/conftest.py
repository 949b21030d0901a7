import os
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with `-m gpu`)")


def _has_gpu():
    try:
        from distributedkernelshap_b200 import parallel
        return parallel.visible_gpus() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


# ---- shared problem builders ------------------------------------------------------------------------------
def make_problem(seed=0, n=8, N=10, widths=(1, 1, 3, 2, 1), kappa=2.0, weights=False, constant_groups=()):
    """Small grouped tabular problem with a binary logistic head.  ``constant_groups``: groups whose columns are
    constant in the background and equal in X (they must come out non-varying)."""
    from distributedkernelshap_b200.predictors import LinearSoftmaxClassifier
    rng = np.random.default_rng(seed)
    D = int(sum(widths))
    groups, start = [], 0
    for wd in widths:
        groups.append(list(range(start, start + wd)))
        start += wd
    bg = rng.standard_normal((N, D))
    X = rng.standard_normal((n, D))
    for g in constant_groups:
        bg[:, groups[g]] = 0.5
        X[:, groups[g]] = 0.5
    coef = rng.normal(0, 0.7, size=(1, D))
    intercept = rng.normal(0, 0.5, size=(1,))
    clf = LinearSoftmaxClassifier(coef, intercept, multi_class="multinomial" if kappa == 2.0 else "ovr")
    w = rng.uniform(0.2, 1.0, size=N) if weights else None
    return dict(X=X, bg=bg, groups=groups, group_names=[f"g{i}" for i in range(len(groups))], clf=clf, weights=w)


def rel_err(got, want):
    """max |got - want| / max |want| per instance (the '1e-5 relative' bar of BASELINE.json's north_star)."""
    got, want = np.asarray(got), np.asarray(want)
    scale = np.maximum(np.abs(want).max(axis=-1, keepdims=True), 1e-12)
    return float((np.abs(got - want) / scale).max())


def elementwise_excess(got, want, rtol=1e-5, atol=1e-9):
    """Element-wise criterion |got - want| <= rtol |want| + atol: returns (fraction of elements violating it, the
    largest |got - want| / (rtol |want| + atol)).  Complements ``rel_err`` (error against the instance's largest
    |phi|), which lets a small component hide behind a large one."""
    got, want = np.asarray(got), np.asarray(want)
    ratio = np.abs(got - want) / (rtol * np.abs(want) + atol)
    return float((ratio > 1.0).mean()), float(ratio.max())
