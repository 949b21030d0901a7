"""The fused shared-plan kernel gives the same bits whatever its layout: one warp per row-group slice or several warps
sharing a slice (``last_path()["cta_warps"]`` above ``warps``), any warps per CTA, any turn-around batch.  Each
(instance, row group) partial is delivered exactly once and summed in 2^-40 fixed point, so the layout cannot change
phi."""
import numpy as np
import pytest

from test_gpu_kernel_paths import _check, _engine, _expect, _problem

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("N", [100, 120])
def test_fused_layouts_give_identical_bits(N):
    G, S = 12, 2048
    prob = _problem(600 + N, G=G, N=N, n=300)
    eng = _engine(prob)
    want = np.stack(eng.shap_values(prob["X"], nsamples=S, l1_reg=False), axis=-1)
    base = eng.last_path()
    _expect(base, shared="fused", solve="fused")
    assert base["cta_warps"] > base["warps"], base          # few row groups: several warps share each slice
    _check(eng, prob, want, S, "fused layouts")
    for opt, val in (("fused_warps", 4), ("fused_warps", 12), ("fused_warps", 16), ("fused_batch", 16)):
        eng.set_option(opt, val)
        got = np.stack(eng.shap_values(prob["X"], nsamples=S, l1_reg=False), axis=-1)
        path = eng.last_path()
        _expect(path, shared="fused")
        if opt == "fused_warps":
            assert path["cta_warps"] <= val, path
        assert np.array_equal(got, want), (opt, val, path, np.abs(got - want).max())
        eng.set_option(opt, 0)
