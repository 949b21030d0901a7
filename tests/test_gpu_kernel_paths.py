"""Every kernel the dispatch can pick, at the shape edges where its code changes, against the float64 reference of
tests/linear_reference.py -- and every case asserts, through ``GpuKernelExplainer.last_path()``, that it ran the path it
was written for.  Thresholds that depend on the device (SM count, shared memory per CTA) are derived from
``torch.cuda.get_device_properties`` and the warps the engine reports, never hard-coded.

Criteria per case (as in test_gpu_baseline_shapes.py): ``rel_err < 1e-5`` per instance and class 1, element-wise
``|got - want| <= 1e-5 |want| + 5e-7``, additivity of class 1 to 1e-8, and class 0 = -class 1.  Class 0 is checked
through that antisymmetry rather than against the reference: upstream computes it as ``log(ey0 / (1 - ey0))`` with ey0
close to 1, which loses digits the engine does not (2e-4 relative at the saturated scores below)."""
import numpy as np
import pytest

from conftest import elementwise_excess, rel_err
from linear_reference import LinearReference

pytestmark = pytest.mark.gpu

TOL = 1e-5
ATOL_ELEM = 5e-7
WORST = {}          # largest rel_err per group of cases (printed with -s)


def _device():
    import torch
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, p.shared_memory_per_block_optin


def _problem(seed, G, N, n, weights=False, intercept=0.0, coef_sd=None, kappa=2.0, const=None):
    """One column per group.  ``const``: {group: rows of X} -- that group is constant in the background and equal to it
    in those rows, which therefore have a partial varying set."""
    from distributedkernelshap_b200.predictors import LinearSoftmaxClassifier
    rng = np.random.default_rng(seed)
    bg = rng.standard_normal((N, G))
    X = rng.standard_normal((n, G))
    for g, rows in (const or {}).items():
        bg[:, g] = 0.25
        X[rows, g] = 0.25
    coef = rng.normal(0, coef_sd if coef_sd is not None else 1.2 / np.sqrt(G), size=(1, G))
    clf = LinearSoftmaxClassifier(coef, np.array([intercept]), multi_class="multinomial" if kappa == 2.0 else "ovr")
    w = rng.uniform(0.2, 1.0, size=N) if weights else None
    return dict(X=X, bg=bg, groups=[[k] for k in range(G)], clf=clf, weights=w, kappa=kappa)


def _engine(prob, kernel="auto", link="logit"):
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    G = len(prob["groups"])
    args = (prob["groups"],) + ((prob["weights"],) if prob["weights"] is not None else ())
    dd = DenseData(prob["bg"], [f"g{k}" for k in range(G)], *args)
    return GpuKernelExplainer(prob["clf"].predict_proba, dd, link=link, kernel=kernel, seed=7)


def _reference(prob, link="logit"):
    clf = prob["clf"]
    return LinearReference(clf.coef_, clf.intercept_, prob["bg"], prob["groups"], prob["weights"], kappa=prob["kappa"],
                           link=link)


def _run(prob, nsamples, kernel="auto", link="logit"):
    eng = _engine(prob, kernel, link)
    got = eng.shap_values(prob["X"], nsamples=nsamples, l1_reg=False)
    return eng, np.stack(got, axis=-1), eng.last_path()


def _check(eng, prob, got, nsamples, group, link="logit", compare=True):
    """Reference fed the engine's own shared plans (one per M), then the criteria of the module docstring."""
    ref = _reference(prob, link)
    np.testing.assert_allclose(eng.expected_value[1], ref.expected_value[1], rtol=1e-12, atol=1e-14)
    assert np.all(np.isfinite(got))
    np.testing.assert_allclose(got[..., 0], -got[..., 1], rtol=0, atol=1e-12)
    deltas = []
    plans = []
    for x in prob["X"]:
        v = ref.varying(x)
        plan = eng.shared_plan(len(v), nsamples) if len(v) >= 2 else None
        plans.append(None if plan is None else (plan.dense(), plan.weights))
        fx = ref._outputs(np.array([ref.intercept + x @ ref.coef]))[0]
        deltas.append(ref.link(fx[1]) - ref.link(ref.fnull[1]))
    np.testing.assert_allclose(got[..., 1].sum(axis=1), np.array(deltas), rtol=1e-8, atol=1e-8)
    if not compare:
        return
    want = ref.shap_values(prob["X"], plans)
    err = rel_err(got[..., 1], want[..., 1])
    frac, mx = elementwise_excess(got[..., 1], want[..., 1], rtol=TOL, atol=ATOL_ELEM)
    WORST[group] = max(WORST.get(group, 0.0), err)
    print(f"[{group}] rel_err {err:.2e} element-wise worst ratio {mx:.3f} (group worst {WORST[group]:.2e})")
    assert err < TOL, (group, err)
    assert frac == 0.0, (group, frac, mx)


def _expect(path, **want):
    for k, v in want.items():
        assert path[k] == v, (k, path[k], v, path)


def _pmat_fits(G, S_pad, smem):
    """Does the float32 projection table of wls_pmat_kernel fit shared memory (the engine's test, dks.cu)?"""
    kpad = (G - 1 + 3) // 4 * 4
    return G - 1 <= 24 and kpad * S_pad * 4 + 8192 <= smem


def _spad(S):
    return (S + 31) // 32 * 32


# ---- fused shared-plan kernel --------------------------------------------------------------------------------------
# N: every (nq_t, rem_t) tail of the run-time chunk (N % 16 in 1, 2, 3, 5, 15, 0 and 1 past a chunk), the NCT = 64 / 100 /
# 128 specialisations and their run-time neighbours 63 / 65, 99 / 101, 127.
FUSED_N = [1, 2, 3, 5, 15, 16, 17, 20, 47, 63, 64, 65, 99, 100, 101, 127, 128]


@pytest.mark.parametrize("N", FUSED_N)
def test_fused_background_sizes(N):
    prob = _problem(100 + N, G=13, N=N, n=6)
    eng, got, path = _run(prob, 400)
    _expect(path, shared="fused", solve="fused", chunks=1)
    _check(eng, prob, got, 400, "fused N")


# G = 2 (one nibble table, S = 2), 14 (four tables, kpad 16), 16 (the widest fused plan); kpad 12 -> 16 between 13 and 14
@pytest.mark.parametrize("G", [2, 14, 16])
@pytest.mark.parametrize("N", [17, 100, 128])
def test_fused_group_counts(G, N):
    prob = _problem(200 + G * 7 + N, G=G, N=N, n=5)
    eng, got, path = _run(prob, 300)
    _expect(path, shared="fused", solve="fused")
    _check(eng, prob, got, 300, "fused G")


def test_fused_instance_counts_around_the_batch():
    """n in {1, B - 1, B, B + 1, 2B + 3}: partial and full turn-around batches, B as the engine chose it."""
    probe = _engine(_problem(300, G=13, N=64, n=1))
    probe.shap_values(_problem(300, G=13, N=64, n=1)["X"], nsamples=200, l1_reg=False)
    B = probe.last_path()["fused_B"]
    assert B in (8, 16, 32)
    for n in (1, B - 1, B, B + 1, 2 * B + 3):
        prob = _problem(300 + n, G=13, N=64, n=n)
        eng, got, path = _run(prob, 200)
        _expect(path, shared="fused", fused_B=B)
        _check(eng, prob, got, 200, "fused n")


# S below one row group of 32, exactly one, and one more.  The group counts keep the plans full rank: a sampled plan of
# S <= 2 (M - 1) rows is mostly complement pairs (z, 1 - z), which give the same row of E up to sign -- the 13-group plans
# of 20 and 32 rows are singular (rank 10 and 11 of 12), and neither upstream nor the engine has an answer for them.
@pytest.mark.parametrize("G,S", [(4, 14), (5, 20), (6, 32), (6, 33), (13, 33)])
def test_fused_fewer_coalitions_than_a_row_group(G, S):
    prob = _problem(400 + S, G=G, N=37, n=7)
    eng, got, path = _run(prob, S)
    _expect(path, shared="fused")
    _check(eng, prob, got, S, "fused S")


def test_fused_one_replica_per_row_group_then_the_unfused_fallback():
    """S_pad / 32 == sm_count * warps: nparts = 1, every warp streams every instance (n = B + 3: a partial last batch).
    One row group more and the fused kernel no longer has a warp per row group: the unfused kernel takes over."""
    sm, smem = _device()
    probe_prob = _problem(500, G=16, N=128, n=1)
    probe = _engine(probe_prob)
    probe.shap_values(probe_prob["X"], nsamples=100, l1_reg=False)
    p0 = probe.last_path()
    _expect(p0, shared="fused")
    S = 32 * sm * p0["warps"]
    assert S <= 2 ** 16 - 2, "the nparts = 1 boundary needs more coalitions than 16 groups have"
    prob = _problem(501, G=16, N=128, n=p0["fused_B"] + 3)
    eng, got, path = _run(prob, S)
    _expect(path, shared="fused", warps=p0["warps"], grid=sm)
    _check(eng, prob, got, S, "fused nparts=1")
    eng, got, path = _run(prob, S + 1)
    n_rg = _spad(S + 1) // 32
    _expect(path, shared="smem", solve="pmat" if _pmat_fits(16, _spad(S + 1), smem) else "wls_shared")
    assert path["grid"] == max(sm, -(-n_rg // path["warps"]))
    _check(eng, prob, got, S + 1, "fused->unfused")


# ---- unfused shared-plan kernel and its solves ----------------------------------------------------------------------
@pytest.mark.parametrize("N", range(16, 32))
def test_unfused_every_ntail(N):
    """G = 20 takes the unfused kernel; N = 16..31 instantiates NTAIL = N % 16 = 0..15."""
    prob = _problem(600 + N, G=20, N=N, n=4)
    eng, got, path = _run(prob, 200)
    _expect(path, shared="smem", chunks=1, solve="pmat", pmat_kpad=20)
    _check(eng, prob, got, 200, "unfused NTAIL")


@pytest.mark.parametrize("N", [128, 129, 144, 256, 257])
def test_unfused_background_chunks(N):
    prob = _problem(700 + N, G=20, N=N, n=4, weights=False)
    eng, got, path = _run(prob, 200)
    _expect(path, shared="smem", chunks=-(-N // 128))
    _check(eng, prob, got, 200, "unfused chunks")


# KPAD = 4 * ceil((G - 1) / 4): G = 5, 9, 13 at N = 129 (past the fused kernel's 128 rows), G = 17, 21, 25 at N = 64
@pytest.mark.parametrize("G,N,kpad", [(5, 129, 4), (9, 129, 8), (13, 129, 12), (17, 64, 16), (21, 64, 20), (25, 64, 24)])
def test_projection_solve_every_kpad(G, N, kpad):
    prob = _problem(800 + G, G=G, N=N, n=5)
    eng, got, path = _run(prob, 300)
    _expect(path, shared="smem", solve="pmat", pmat_kpad=kpad)
    _check(eng, prob, got, 300, "pmat")


@pytest.mark.parametrize("G,nsamples", [(26, 300), (20, 3000)])
def test_wls_shared_solve(G, nsamples):
    """G = 26: 25 coefficients, more than the projection solve holds in registers; G = 20 at S = 3000: P does not fit
    shared memory (checked against the device's limit)."""
    _, smem = _device()
    if G == 20:
        assert not _pmat_fits(G, _spad(nsamples), smem)
    prob = _problem(900 + G, G=G, N=40, n=5)
    eng, got, path = _run(prob, nsamples)
    _expect(path, shared="smem", solve="wls_shared")
    _check(eng, prob, got, nsamples, "wls_shared")


@pytest.mark.parametrize("G", [65, 128])
@pytest.mark.parametrize("N", [17, 130])
def test_two_word_rows(G, N):
    prob = _problem(1000 + G + N, G=G, N=N, n=3)
    eng, got, path = _run(prob, 600)
    _expect(path, shared="smem", solve="wls_shared", chunks=-(-N // 128), general="flagged")
    _check(eng, prob, got, 600, "two-word rows")


# ---- large plans: more row groups than a grid of sm_count CTAs has warps ---------------------------------------------
def test_full_enumeration_16_groups_128_background_rows():
    """Exact Shapley values of 16 groups: S = 65534, 2048 row groups.  The fused kernel does not have a warp per row
    group; the unfused kernel must size its grid so that it does, and the general kernel (which cannot hold S = 65534)
    must not fail a call that left it nothing to do."""
    sm, _ = _device()
    prob = _problem(1100, G=16, N=128, n=3)
    eng, got, path = _run(prob, 65534)
    n_rg = 65536 // 32
    _expect(path, shared="smem", solve="wls_shared", general="flagged")
    assert path["grid"] == max(sm, -(-n_rg // path["warps"])) and path["grid"] * path["warps"] >= n_rg
    assert eng.shared_plan(16, 65534).S == 65534
    _check(eng, prob, got, 65534, "large plans")


def test_two_word_rows_65536_coalitions():
    sm, _ = _device()
    prob = _problem(1200, G=70, N=128, n=3)
    eng, got, path = _run(prob, 65536)
    n_rg = 65536 // 32
    _expect(path, shared="smem", solve="wls_shared", general="flagged")
    assert path["grid"] * path["warps"] >= n_rg
    _check(eng, prob, got, 65536, "large plans")


def test_large_plan_with_a_partial_varying_set_is_reported_not_computed():
    """One instance of the S = 65534 batch has 15 varying groups: no general kernel holds its plan, so the call reports
    status 3 (unsupported) instead of computing it some other way."""
    from distributedkernelshap_b200._cabi import DksError
    prob = _problem(1300, G=16, N=128, n=3, const={4: [1]})
    eng = _engine(prob)
    with pytest.raises((DksError, NotImplementedError)) as ei:
        eng.shap_values(prob["X"], nsamples=65534, l1_reg=False)
    if isinstance(ei.value, DksError):
        assert ei.value.code == 3
    _expect(eng.last_path(), shared="smem", general="flagged")


# ---- tensor-core kernel ---------------------------------------------------------------------------------------------
# N crosses consume_quad / consume_pair and full / partial 32-column blocks
@pytest.mark.parametrize("N", [1, 31, 32, 33, 64, 65, 96, 97, 128])
@pytest.mark.parametrize("weights", [False, True])
def test_tc_background_sizes(N, weights):
    prob = _problem(1400 + N + weights, G=9, N=N, n=6, weights=weights)
    eng, got, path = _run(prob, 300, kernel="tcgen05")
    _expect(path, shared="none", general="tc")
    _check(eng, prob, got, 300, "tc N")


@pytest.mark.parametrize("G", [2, 15])
def test_tc_group_counts(G):
    prob = _problem(1500 + G, G=G, N=50, n=6, weights=True)
    eng, got, path = _run(prob, 300, kernel="tcgen05")
    _expect(path, shared="none", general="tc")
    _check(eng, prob, got, 300, "tc G")


# tiles of 128 coalitions around multiples of the 4 consumer warpgroups (S = 14: the full plan of 4 groups, one partial tile)
@pytest.mark.parametrize("S", [14, 128, 129, 640, 1024, 1025])
def test_tc_coalition_counts(S):
    prob = _problem(1600 + S, G=4 if S == 14 else 11, N=40, n=5)
    eng, got, path = _run(prob, S, kernel="tcgen05")
    _expect(path, shared="none", general="tc")
    _check(eng, prob, got, S, "tc S")


def test_tc_plans_of_different_sizes_in_one_batch():
    """Instances with 10, 9 and 8 varying groups: each evaluates the shared plan of its own M."""
    prob = _problem(1700, G=10, N=45, n=9, const={2: [3, 4, 5, 6, 7, 8], 7: [6, 7, 8]})
    eng, got, path = _run(prob, 250, kernel="tcgen05")
    _expect(path, general="tc")
    assert sorted(set(eng.varying(prob["X"])[0])) == [8, 9, 10]
    _check(eng, prob, got, 250, "tc mixed M")


def test_tc_instance_counts_around_the_sm_count():
    sm, _ = _device()
    for n in (1, sm - 1, sm, sm + 1, 2 * sm + 1):
        prob = _problem(1800 + n, G=6, N=20, n=n)
        eng, got, path = _run(prob, 62, kernel="tcgen05")
        _expect(path, general="tc")
        _check(eng, prob, got, 62, "tc n")


@pytest.mark.parametrize("N", [16, 33, 97, 128])
def test_tc_score_tile_columns_past_the_background_are_zero(N):
    prob = _problem(1900 + N, G=7, N=N, n=4)
    eng = _engine(prob, kernel="tcgen05")
    T = eng.debug_scores(prob["X"], 2, nsamples=100)
    _expect(eng.last_path(), general="tc")
    plan = eng.shared_plan(7, 100)
    ref = _reference(prob)
    Z = plan.dense().astype(np.float64)
    XW = prob["X"][2] * ref.coef
    want = -2.0 * np.log2(np.e) * (ref.base[None, :] + Z @ (XW[None, :] - ref.BW).T)
    assert T.shape[1] == (N + 15) // 16 * 16 and T.shape[0] >= plan.S
    np.testing.assert_allclose(T[:plan.S, :N], want, rtol=0, atol=2e-5)
    assert np.all(T[:, N:] == 0)


def test_auto_fused_and_tc_in_one_call():
    """Half the instances vary in every group (fused kernel), half in all but one (the tensor-core kernel on the side
    stream), in the same call."""
    prob = _problem(2000, G=12, N=50, n=10, const={5: [5, 6, 7, 8, 9]})
    eng, got, path = _run(prob, 500)
    _expect(path, shared="fused", general="tc")
    assert sorted(set(eng.varying(prob["X"])[0])) == [11, 12]
    _check(eng, prob, got, 500, "auto fused + tc")


def test_last_path_of_a_graph_replay_is_the_captured_call():
    """dks_last_path is recorded while a call is enqueued: replays of the captured graph report the captured call."""
    import torch
    prob = _problem(2050, G=12, N=30, n=20)
    eng = _engine(prob)
    want = eng.shap_values(prob["X"], nsamples=300, l1_reg=False)[1]
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(prob["X"]).cuda()
        phi = torch.zeros((2, 20, 12), dtype=torch.float64, device="cuda")
        for _ in range(3):
            eng.explain_device(X_dev.data_ptr(), 20, phi.data_ptr(), nsamples=300)
        eng.check_status()
        assert eng.graph_launches() >= 1
        _expect(eng.last_path(), shared="fused", solve="fused")
        np.testing.assert_allclose(phi[1].cpu().numpy(), want, rtol=0, atol=1e-12)
    eng.set_stream(0)


# ---- near-saturated scores -------------------------------------------------------------------------------------------
# kappa * score of the background rows in about [-36, -20] for most coalitions: p1 ~ 1e-16 .. 2e-9, A up to 2^52, the pair
# product q = A^2 Dm Dm near 2^104.  Upstream's float64 class 1 is exact there.
SATURATED = [("auto", 64, "fused"), ("auto", 129, "smem"), ("tcgen05", 64, "tc"), ("simt", 64, "simt")]


@pytest.mark.parametrize("kernel,N,which", SATURATED)
def test_near_saturated_scores(kernel, N, which):
    prob = _problem(2100 + N, G=8, N=N, n=8, intercept=-14.0, coef_sd=0.45)
    t = 2.0 * (prob["clf"].intercept_[0] + prob["bg"] @ prob["clf"].coef_[0])
    assert np.mean((t > -36) & (t < -20)) > 0.9
    eng, got, path = _run(prob, 200, kernel=kernel)
    if which in ("fused", "smem"):
        _expect(path, shared=which)
    else:
        _expect(path, shared="none", general=which)
    _check(eng, prob, got, 200, "saturated")


@pytest.mark.parametrize("kernel,N,which", SATURATED)
def test_past_the_clamp_stays_finite(kernel, N, which):
    """kappa * score <= -45 takes the clamped scalar path (A > 1e18, DESIGN.md 5.2): finite values, antisymmetry and
    additivity only."""
    prob = _problem(2200 + N, G=8, N=N, n=6, intercept=-30.0, coef_sd=0.45)
    eng, got, path = _run(prob, 200, kernel=kernel)
    if which in ("fused", "smem"):
        _expect(path, shared=which)
    else:
        _expect(path, shared="none", general=which)
    _check(eng, prob, got, 200, "past the clamp", compare=False)
