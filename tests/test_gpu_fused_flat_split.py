"""The fused kernel's flat split (one slice per CTA: CTA c takes the c-th of SMs equal contiguous ranges of the (row group,
instance) pairs, its warps equal contiguous pieces of that range) gives the same bits as the one-warp-per-slice layout
(``fused_warps`` 1: whole row groups dealt round-robin), at instance counts where the CTA and warp ranges start and end
at different points of a row group, and agrees with the float64 reference.  Uniform and weighted backgrounds."""
import numpy as np
import pytest

from test_gpu_kernel_paths import _check, _device, _engine, _expect, _problem
from test_gpu_weighted_background import _wproblem

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("extra", [-1, 0, 1, 7])
def test_flat_split_matches_one_warp_per_slice(extra, weighted):
    sm, _ = _device()
    n = max(1, sm + extra)
    make = _wproblem if weighted else _problem
    prob = make(7000 + extra + 50 * weighted, G=12, N=100, n=n)
    eng = _engine(prob)
    want = {}
    for cap in (0, 1):
        eng.set_option("fused_warps", cap)
        want[cap] = np.stack(eng.shap_values(prob["X"], nsamples=2048, l1_reg=False), axis=-1)
        path = eng.last_path()
        _expect(path, shared="fused", solve="fused", bg_weights="weighted" if weighted else "uniform")
        if cap == 0:
            assert path["cta_warps"] > 1, path
        else:
            assert path["cta_warps"] == 1, path
    eng.set_option("fused_warps", 0)
    assert np.array_equal(want[0], want[1]), np.abs(want[0] - want[1]).max()
    _check(eng, prob, want[0], 2048, "fused flat split")
