"""Host side of per-instance plans of 65..128 groups (two-word rows): what the device sampler must reproduce, the limits
the engine checks before it uploads a plan's sampling tables, and the per-call row bound of the mode.  No GPU needed."""
import numpy as np
import pytest

from sampler_twin import PhiloxPlanStream


@pytest.mark.parametrize("M,nsamples", [(65, 300), (80, 1000), (127, 2000), (128, 4096)])
def test_twin_plans_are_well_formed(M, nsamples):
    from oracle.shap_kernel_oracle import build_plan as oracle_plan
    from distributedkernelshap_b200.plan import build_plan, pack_dense_plan, resolve_nsamples, sampling_info, size_weights
    S, _ = resolve_nsamples(M, nsamples)
    shared = build_plan(M, nsamples, rng=np.random.RandomState(0))
    nfixed, n_full, n_paired, cdf, weight_left = sampling_info(shared)
    for row in (0, 1, 12345):
        Z, w, _ = oracle_plan(M, S, rng=PhiloxPlanStream(99, row))
        assert Z.shape == (S, M) and np.isclose(w.sum(), 1.0, rtol=0, atol=1e-12)
        zb = pack_dense_plan(Z)
        assert zb.shape == (S, 2) and zb.dtype == np.uint64
        # the enumerated prefix is the shared plan's (deterministic per M)
        np.testing.assert_array_equal(zb[:nfixed], shared.zbits[:nfixed])
        np.testing.assert_allclose(w[:nfixed], shared.weights[:nfixed], rtol=1e-15, atol=0)
        # sampled part: a mask of a paired size is followed by its complement (when a row is left)
        r, sizes = nfixed, Z.sum(axis=1)
        while r < S:
            assert 1 <= sizes[r] <= M - 1
            if min(sizes[r], M - sizes[r]) <= n_paired and sizes[r] != M - sizes[r] and sizes[r] <= M // 2:
                if r + 1 < S:
                    np.testing.assert_array_equal(Z[r + 1], 1 - Z[r])
                r += 2
            else:
                r += 1
        # no mask appears twice
        assert len({bytes(row_) for row_ in zb.view(np.uint8).reshape(S, 16)}) == S
        np.testing.assert_allclose(w[nfixed:].sum(), weight_left, rtol=1e-12)


def test_sampling_tables_at_128_groups_fit_the_device_sampler():
    from distributedkernelshap_b200.engine import MAX_SAMPLED_SIZES, device_sampling_supported
    from distributedkernelshap_b200.plan import build_plan, sampling_info
    plan = build_plan(128, 4096, rng=np.random.RandomState(1))
    nfixed, n_full, n_paired, cdf, weight_left = sampling_info(plan)
    assert (nfixed, n_full, len(cdf)) == (256, 1, 63)            # size 1 enumerated, sizes 2..64 sampled
    assert cdf[-1] == 1.0 and np.all(np.diff(cdf) > 0)
    assert device_sampling_supported(128, len(cdf)) and MAX_SAMPLED_SIZES == 64
    assert not device_sampling_supported(129, 63)                # no per-instance plans beyond 128 groups
    for M in range(2, 129):                                      # every M up to 128 has at most 63 sampled sizes
        assert len(sampling_info(build_plan(M, "auto", rng=np.random.RandomState(M)))[3]) <= 63


def test_per_call_row_bound_of_two_word_per_instance_plans():
    from distributedkernelshap_b200 import _cabi
    from distributedkernelshap_b200.engine import (MAX_ROWS_PER_CALL, MAX_ROWS_PER_CALL_WIDE_PER_INSTANCE,
                                                   per_instance_workspace_bytes, rows_per_call)
    rows = rows_per_call(_cabi.ACT_BINARY_LOGISTIC, 2, "per_instance", 128)
    assert rows == MAX_ROWS_PER_CALL_WIDE_PER_INSTANCE
    per_row = per_instance_workspace_bytes(128, 4096)
    assert per_row == 4096 * 24 + 8 * 127 * 127                  # 64 KB words + 32 KB weights + 126 KB inverse
    assert rows * per_row <= 1 << 30                             # under 1 GiB per call at configs[4]
    assert rows_per_call(_cabi.ACT_IDENTITY, 1, "per_instance", 65) == MAX_ROWS_PER_CALL_WIDE_PER_INSTANCE
    # unchanged elsewhere
    assert rows_per_call(_cabi.ACT_BINARY_LOGISTIC, 2, "per_instance", 64) == MAX_ROWS_PER_CALL
    assert rows_per_call(_cabi.ACT_BINARY_LOGISTIC, 2, "shared", 128) == MAX_ROWS_PER_CALL
    assert rows_per_call(_cabi.ACT_SOFTMAX, 4, "shared", 10) == MAX_ROWS_PER_CALL // 2


def test_two_word_plan_entry_point_is_declared():
    import os
    import re
    from distributedkernelshap_b200 import _cabi
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dks.h")).read()
    assert re.search(r"int dks_get_instance_plans_w\(", hdr)
    assert "dks_get_instance_plans_w" in _cabi.SIGNATURES
    assert re.search(r"#define DKS_GENERAL_SIMT_WIDE 4", hdr)
