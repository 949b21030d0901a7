"""Which instances run upstream's l1 feature selection (``engine.l1_selecting_sizes``): one decision per number M of
varying groups, made on the host, and what the engine still refuses."""
import numpy as np
import pytest

from distributedkernelshap_b200.engine import l1_selecting_sizes


def _hist(G, present):
    h = np.zeros(G + 1, dtype=np.int32)
    h[list(present)] = 1
    return h


def test_auto_selects_below_20_percent_per_m():
    # nsamples 'auto' = 2M + 2048: M = 13 evaluates 2074 of 8190 coalitions (25%), M = 14 2076 of 16382 (12.7%)
    assert l1_selecting_sizes("auto", "auto", 15, _hist(15, [0, 1, 12, 13, 14, 15])) == (1, 0, [14, 15])
    assert l1_selecting_sizes("auto", "auto", 15, _hist(15, [1, 13])) == (0, 0, [])
    # the boundary itself: 6 of 30 coalitions (M = 5) is 20% and does not select, 5 of 30 does
    assert l1_selecting_sizes("auto", 6, 5, _hist(5, [5])) == (0, 0, [])
    assert l1_selecting_sizes("auto", 5, 5, _hist(5, [5])) == (1, 0, [5])
    # M = 4 at nsamples 2: 2 of 14 selects, at 3: 3 of 14 (21%) does not
    assert l1_selecting_sizes("auto", 2, 5, _hist(5, [4, 5])) == (1, 0, [4, 5])
    assert l1_selecting_sizes("auto", 3, 5, _hist(5, [4, 5])) == (1, 0, [5])


def test_explicit_modes_select_every_present_m():
    h = _hist(20, [0, 1, 2, 7, 19])
    assert l1_selecting_sizes("aic", "auto", 20, h) == (1, 0, [2, 7, 19])
    assert l1_selecting_sizes("bic", 100, 20, h) == (2, 0, [2, 7, 19])
    assert l1_selecting_sizes("num_features(5)", "auto", 20, h) == (3, 5, [2, 7, 19])
    for off in (False, 0):
        assert l1_selecting_sizes(off, "auto", 20, h) == (0, 0, [])


def test_what_still_raises():
    with pytest.raises(NotImplementedError, match="fixed Lasso strength"):
        l1_selecting_sizes(0.01, "auto", 16, _hist(16, [16]))
    with pytest.raises(NotImplementedError, match="128 groups"):
        l1_selecting_sizes("auto", 600, 140, _hist(140, [140]))
    with pytest.raises(NotImplementedError, match="partial varying set"):
        l1_selecting_sizes("auto", 700, 80, _hist(80, [79, 80]))
    # beyond 64 groups, instances whose groups all vary select; up to 64 partial sets do too
    assert l1_selecting_sizes("auto", 700, 80, _hist(80, [80])) == (1, 0, [80])
    assert l1_selecting_sizes("auto", "auto", 64, _hist(64, [62, 63])) == (1, 0, [62, 63])
    # partial sets beyond 64 groups that do not select are not this function's concern
    assert l1_selecting_sizes(False, 700, 80, _hist(80, [79, 80])) == (0, 0, [])
