"""Parity of the CUDA path (through the C ABI) with the CPU oracle on identical inputs.  Tolerance: 1e-5 relative
to the largest |phi| of the instance (BASELINE.json north_star: "within 1e-5 relative"); additivity to 1e-8."""
import numpy as np
import pytest

from conftest import make_problem, rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-5


def _oracle(prob, link="logit", predict="predict_proba"):
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    args = (prob["groups"],) + ((prob["weights"],) if prob["weights"] is not None else ())
    dd = DenseData(prob["bg"], prob["group_names"], *args)
    return KernelExplainerOracle(getattr(prob["clf"], predict), dd, link=link, record_plans=True)


def _engine(prob, link="logit", predict="predict_proba", **kw):
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    args = (prob["groups"],) + ((prob["weights"],) if prob["weights"] is not None else ())
    dd = DenseData(prob["bg"], prob["group_names"], *args)
    return GpuKernelExplainer(getattr(prob["clf"], predict), dd, link=link, **kw)


KERNELS = ["simt", "tcgen05", "auto"]      # tcgen05 = the tensor-core (wgmma) kernel; auto = shared-plan fast path where it applies + it for the rest


def _compare(got, want, tol=TOL):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.shape == w.shape
        assert rel_err(g, w) < tol, rel_err(g, w)


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("link", ["logit", "identity"])
@pytest.mark.parametrize("kappa", [2.0, 1.0])
def test_full_enumeration_matches_oracle(link, kappa, kernel):
    """S >= 2^M - 2: the plan is RNG-free (SURVEY §4 item 4); GPU and oracle build it independently."""
    prob = make_problem(seed=1, n=16, N=12, widths=(1, 1, 3, 2, 1, 2), kappa=kappa)
    orc, eng = _oracle(prob, link), _engine(prob, link, kernel=kernel)
    want = orc.shap_values(prob["X"], nsamples=10000, l1_reg=False)
    got = eng.shap_values(prob["X"], nsamples=10000, l1_reg=False)
    _compare(got, want)
    np.testing.assert_allclose(eng.expected_value, orc.expected_value, rtol=1e-12)


@pytest.mark.parametrize("kernel", KERNELS)
def test_expected_value_and_additivity(kernel):
    prob = make_problem(seed=2, n=32, N=20, widths=(1, 1, 1, 4, 3, 1, 1, 2), weights=True)
    eng = _engine(prob, "logit", kernel=kernel)
    sv = eng.shap_values(prob["X"], nsamples=150, l1_reg=False)
    fx = prob["clf"].predict_proba(prob["X"])
    for c in range(2):
        total = np.log(fx[:, c] / (1 - fx[:, c])) - eng.expected_value[c]
        np.testing.assert_allclose(sv[c].sum(axis=1), total, rtol=1e-8, atol=1e-8)
    # two-class antisymmetry (SURVEY §4 item 3)
    np.testing.assert_allclose(sv[0], -sv[1], rtol=0, atol=1e-12)


@pytest.mark.parametrize("kernel", KERNELS)
def test_external_per_instance_plans_match_oracle(kernel):
    """Sampled plans: the oracle draws one plan per instance from the advancing MT19937 stream (what shap does);
    the very same plans are fed to the GPU."""
    prob = make_problem(seed=3, n=24, N=16, widths=(1, 1, 1, 1, 3, 2, 1, 2, 1, 4, 1, 1))
    orc, eng = _oracle(prob), _engine(prob, kernel=kernel)
    np.random.seed(0)
    want = orc.shap_values(prob["X"], nsamples=500, l1_reg=False)
    plans = [(Z, w) for (_, Z, w) in orc.plans]
    got = eng.shap_values(prob["X"], nsamples=500, l1_reg=False, plans=plans)
    _compare(got, want)


@pytest.mark.parametrize("kernel", KERNELS)
def test_shared_plan_matches_oracle_fed_the_same_plan(kernel):
    from distributedkernelshap_b200.plan import build_plan
    prob = make_problem(seed=4, n=20, N=25, widths=(1,) * 4 + (3, 2, 2, 1, 5, 1), weights=True)
    orc = _oracle(prob)
    np.random.seed(11)
    eng = _engine(prob, kernel=kernel)
    got = eng.shap_values(prob["X"], nsamples=300, l1_reg=False)
    np.random.seed(11)  # the engine drew its M=10 plan from this state
    plan = build_plan(10, 300)
    want = [np.zeros_like(g) for g in got]
    for i in range(prob["X"].shape[0]):
        phi = orc.explain(prob["X"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=300, l1_reg=False)
        for c in range(2):
            want[c][i] = phi[:, c]
    _compare(got, want)


@pytest.mark.parametrize("kernel", KERNELS)
def test_non_varying_groups_and_degenerate_M(kernel):
    prob = make_problem(seed=5, n=10, N=8, widths=(1, 2, 1, 3, 1), constant_groups=(1, 3))
    X = prob["X"]
    prob["bg"][:] = prob["bg"][0]                            # constant background: a group varies iff x differs from it
    X[1] = prob["bg"][0]                                     # M = 0
    X[2] = prob["bg"][0]; X[2, 0] += 1.0                     # M = 1
    orc, eng = _oracle(prob), _engine(prob, kernel=kernel)
    want = orc.shap_values(X, nsamples=100, l1_reg=False)
    got = eng.shap_values(X, nsamples=100, l1_reg=False)
    _compare(got, want)
    assert np.all(got[1][:, 1] == 0) and np.all(got[1][:, 3] == 0)   # non-varying groups get exactly 0
    assert np.all(got[1][1] == 0)
    M, mask = eng.varying(X)
    assert M[1] == 0 and M[2] == 1
    want_M = [len(orc.varying_groups(X[i:i + 1])) for i in range(X.shape[0])]
    assert list(M) == want_M


def test_varying_groups_isclose_rule():
    """np.isclose(x, bg, rtol=1e-5, atol=1e-8): differences below the tolerance do not make a group vary."""
    prob = make_problem(seed=6, n=6, N=5, widths=(1, 1, 2))
    prob["bg"][:, 0] = 3.0
    prob["X"][:, 0] = [3.0, 3.0 + 2e-5, 3.0 + 4e-5, 3.0 - 2e-5, 3.0 + 3.1e-5, 3.0 - 3.1e-5]
    orc, eng = _oracle(prob), _engine(prob)
    M, mask = eng.varying(prob["X"])
    for i in range(6):
        vi = orc.varying_groups(prob["X"][i:i + 1])
        assert sorted(np.nonzero([(int(mask[i]) >> g) & 1 for g in range(3)])[0]) == sorted(vi), i


def test_varying_groups_with_nan_columns():
    """np.isclose(..., equal_nan=True): a NaN in x matches a NaN in the background (SURVEY §8a row A4).  Columns holding
    NaNs take the full background scan on the device instead of the min / max shortcut."""
    prob = make_problem(seed=16, n=6, N=7, widths=(1, 2, 1, 1))
    bg, X = prob["bg"], prob["X"]
    bg[:, 0] = np.nan                       # group 0: background all NaN
    X[0, 0] = np.nan                        # equal to every background value: group 0 does not vary
    X[1, 0] = 1.0                           # a number against NaNs: varies
    bg[:, 3] = 2.0
    bg[2, 3] = np.nan                       # group 2 (column 3): one NaN among constants
    X[:, 3] = 2.0                           # differs from the NaN row only: varies
    X[3, 3] = np.nan                        # NaN against mostly numbers: varies
    bg[:, 4] = 5.0
    X[:, 4] = 5.0                           # group 3 never varies
    orc, eng = _oracle(prob), _engine(prob)
    M, mask = eng.varying(X)
    for i in range(X.shape[0]):
        want = sorted(int(v) for v in orc.varying_groups(X[i:i + 1]))
        got = [g for g in range(4) if (int(mask[i]) >> g) & 1]
        assert got == want, (i, got, want)
        assert M[i] == len(want)
    assert not (int(mask[0]) & 1) and (int(mask[1]) & 1) and all((int(m) >> 2) & 1 for m in mask) and not any((int(m) >> 3) & 1 for m in mask)


def test_identity_head_closed_form():
    """Affine model + identity link: phi_g = sum_{k in g} w_k (x_k - E_bg[bg_k]) exactly (SURVEY §4 item 2)."""
    prob = make_problem(seed=7, n=12, N=9, widths=(1, 2, 1, 3, 1, 1, 2), weights=True)
    eng = _engine(prob, link="identity", predict="decision_function")
    orc = _oracle(prob, link="identity", predict="decision_function")
    got = eng.shap_values(prob["X"], nsamples=64, l1_reg=False)
    assert isinstance(got, np.ndarray) and got.shape == (12, 7) and not eng.vector_out
    wb = prob["weights"] / prob["weights"].sum()
    coef = prob["clf"].coef_[0]
    for g, cols in enumerate(prob["groups"]):
        closed = ((prob["X"][:, cols] - (wb[:, None] * prob["bg"][:, cols]).sum(0)) * coef[cols]).sum(1)
        np.testing.assert_allclose(got[:, g], closed, rtol=1e-9, atol=1e-10)
    np.random.seed(0)
    want = orc.shap_values(prob["X"], nsamples=64, l1_reg=False)
    assert rel_err(got, want) < 1e-8


@pytest.mark.parametrize("kernel", KERNELS)
def test_adult_shape_shared_plan_parity_and_sharding_invariance(kernel):
    """BASELINE config[1] shape (D=49, 12 groups, bg=100, nsamples=2048) on a subset of instances."""
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.plan import build_plan
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    d = adult_like(n_explain=64)
    prob = dict(X=d["X_explain"], bg=d["background"], groups=d["groups"], group_names=d["group_names"],
                clf=d["predictor"], weights=None)
    np.random.seed(0)
    eng = _engine(prob, kernel=kernel)
    got = eng.shap_values(prob["X"], nsamples=2048, l1_reg=False)
    M, _ = eng.varying(prob["X"])
    np.random.seed(0)
    plans = {}
    for m in sorted(set(int(v) for v in M if v >= 2)):   # the engine builds missing plans in increasing M
        plans[m] = build_plan(m, 2048)
    orc = KernelExplainerOracle(d["predictor"].predict_proba, DenseData(prob["bg"], prob["group_names"], prob["groups"]),
                                link="logit")
    for i in range(0, 64, 4):
        p = plans[int(M[i])]
        phi = orc.explain(prob["X"][i:i + 1], plan=(p.dense(), p.weights), nsamples=2048, l1_reg=False)
        assert rel_err(got[1][i], phi[:, 1]) < TOL
    # explaining in two halves gives the same rows (replaces order_result, distributed.py:156-179)
    a = eng.shap_values(prob["X"][:30], nsamples=2048, l1_reg=False)
    b = eng.shap_values(prob["X"][30:], nsamples=2048, l1_reg=False)
    np.testing.assert_array_equal(np.concatenate([a[1], b[1]]), got[1])


def test_l1_reg_settings_the_engine_does_not_cover_are_refused_not_ignored():
    """The l1 selection itself runs on the device (tests/test_gpu_l1.py); what it does not cover raises."""
    prob = make_problem(seed=8, n=4, N=6, widths=(1,) * 16)
    eng = _engine(prob)
    with pytest.raises(NotImplementedError):
        eng.shap_values(prob["X"], nsamples=200, l1_reg=0.01)           # fixed Lasso strength
    per = _engine(prob, plan_mode="per_instance", seed=1)
    with pytest.raises(NotImplementedError):
        per.shap_values(prob["X"], nsamples=200)                          # 'auto' would select: shared plans only
    per.shap_values(prob["X"], nsamples=200, l1_reg=False)
    eng.shap_values(prob["X"], nsamples=200, l1_reg=False)


def test_model_mismatch_is_refused():
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.predictors import LinearModelSpec
    prob = make_problem(seed=9)
    with pytest.raises(TypeError):
        GpuKernelExplainer(lambda X: X.sum(1), prob["bg"])

    class Liar:
        coef_ = prob["clf"].coef_
        intercept_ = prob["clf"].intercept_

        def predict_proba(self, X):
            return prob["clf"].predict_proba(X) ** 2
    with pytest.raises(ValueError):
        GpuKernelExplainer(Liar().predict_proba, prob["bg"])
    assert LinearModelSpec(prob["clf"].coef_, prob["clf"].intercept_, "binary_logistic", 2.0).n_outputs == 2


def test_kernelshap_api_end_to_end():
    """The reference's own call sequence (benchmarks/ray_pool.py:34-37, :73)."""
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    d = adult_like(n_explain=40)
    data = d["data"]
    explainer = KernelShap(d["predictor"].predict_proba, link="logit", feature_names=d["group_names"], seed=0)
    explainer.fit(data["background"]["X"]["preprocessed"], group_names=d["group_names"], groups=d["groups"])
    explanation = explainer.explain(d["X_explain"], silent=True, nsamples=2048, l1_reg=False)
    sv = explanation.shap_values
    assert len(sv) == 2 and sv[0].shape == (40, 12)
    raw = explanation.raw["raw_prediction"]
    np.testing.assert_allclose(sv[1].sum(1) + explanation.expected_value[1], raw[:, 1], rtol=1e-7, atol=1e-7)
    # raw_prediction comes from stage 1 of the explain call on the device: same numbers as link(predictor(X))
    p = d["predictor"].predict_proba(d["X_explain"])
    np.testing.assert_allclose(raw, np.log(p / (1 - p)), rtol=1e-12, atol=1e-12)
    assert np.array_equal(explanation.raw["prediction"], p.argmax(1))
    # distributed_opts: mini-batches of 10 rows through DistributedExplainer give the same values
    dist = KernelShap(d["predictor"].predict_proba, link="logit", feature_names=d["group_names"], seed=0,
                      distributed_opts={"n_cpus": 1, "batch_size": 10, "actor_cpu_fraction": 1.0})
    dist.fit(data["background"]["X"]["preprocessed"], group_names=d["group_names"], groups=d["groups"])
    sv2 = dist.explain(d["X_explain"], silent=True, nsamples=2048, l1_reg=False).shap_values
    np.testing.assert_allclose(sv2[1], sv[1], rtol=0, atol=1e-12)
    js = explanation.to_json()
    assert '"shap_values"' in js


def test_tcgen05_accumulator_tile_matches_numpy():
    """The tensor-core contraction on its own: T[s][j] = scale * masked score, against float64 NumPy."""
    from distributedkernelshap_b200.plan import build_plan
    prob = make_problem(seed=12, n=5, N=37, widths=(1, 1, 3, 2, 1, 2, 1, 1, 4), weights=True)
    np.random.seed(2)
    eng = _engine(prob, kernel="tcgen05")
    inst = 3
    T = eng.debug_scores(prob["X"], inst, nsamples=300)
    np.random.seed(2)
    plan = build_plan(9, 300)
    Z = plan.dense().astype(np.float64)
    coef, b = prob["clf"].coef_[0], prob["clf"].intercept_[0]
    x = prob["X"][inst]
    XW = np.array([(x[g] * coef[g]).sum() for g in prob["groups"]])
    BW = np.stack([(prob["bg"][:, g] * coef[g]).sum(1) for g in prob["groups"]], axis=1)      # [N, G]
    score = b + BW.sum(1)
    scale = -2.0 * np.log2(np.e)
    want = scale * (score[None, :] + Z @ (XW[None, :] - BW).T)                               # [S, N]
    assert T.shape[1] == 48 and T.shape[0] >= 300
    np.testing.assert_allclose(T[:300, :37], want, rtol=0, atol=2e-5)
    assert np.all(T[:300, 37:] == 0)


def test_tcgen05_and_simt_kernels_agree_and_many_instances_per_cta():
    """More instances than SMs (persistent CTAs walk several instances, odd tile counts: S = 2072 -> 17 tiles)."""
    from distributedkernelshap_b200.datasets import adult_like
    d = adult_like(n_explain=700)
    prob = dict(X=d["X_explain"], bg=d["background"], groups=d["groups"], group_names=d["group_names"],
                clf=d["predictor"], weights=None)
    res = {}
    for kernel in KERNELS:
        np.random.seed(0)
        eng = _engine(prob, kernel=kernel)
        res[kernel] = eng.shap_values(prob["X"], l1_reg=False)          # nsamples='auto' = 2072
    assert rel_err(res["tcgen05"][1], res["simt"][1]) < 2e-6
    assert rel_err(res["auto"][1], res["simt"][1]) < 2e-6


def test_golden_fixtures_on_gpu():
    import glob
    import os
    from distributedkernelshap_b200.predictors import LinearSoftmaxClassifier
    for path in sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz"))):
        g = np.load(path, allow_pickle=True)
        groups = [list(map(int, x)) for x in g["groups"]]
        clf = LinearSoftmaxClassifier(g["coef"], g["intercept"], multi_class=str(g["multi_class"]))
        prob = dict(X=g["X"], bg=g["bg"], groups=groups, group_names=[f"g{i}" for i in range(len(groups))], clf=clf,
                    weights=g["weights"])
        for kernel in (KERNELS if len(groups) <= 15 else ["simt", "auto"]):
            eng = _engine(prob, link=str(g["link"]), kernel=kernel)
            plans = None if g["full"] else [(g["Z"][i], g["w"][i]) for i in range(g["X"].shape[0])]
            got = eng.shap_values(g["X"], nsamples=int(g["nsamples"]), l1_reg=False, plans=plans)
            for c in range(2):
                assert rel_err(got[c], g["phi"][:, :, c]) < TOL, (path, kernel)
            if g["full"]:
                assert rel_err(got[1], g["phi_exact"][:, :, 1]) < TOL
            np.testing.assert_allclose(eng.expected_value, g["expected_value"], rtol=1e-12)


@pytest.mark.parametrize("seed", range(10))
def test_randomized_shapes_all_kernels(seed):
    """Random group structures / background sizes / sample budgets / weights through every kernel that supports them."""
    rng = np.random.default_rng(1000 + seed)
    G = int(rng.choice([2, 3, 5, 8, 12, 15, 16, 23, 40]))
    widths = tuple(int(w) for w in rng.integers(1, 4, size=G))
    N = int(rng.choice([1, 7, 16, 31, 32, 64, 100, 127, 128, 150]))
    n = int(rng.integers(3, 40))
    weights = bool(rng.integers(0, 2))
    nsamples = int(rng.choice([50, 128, 257, 500, 1000]))
    const = tuple(int(g) for g in rng.choice(G, size=int(rng.integers(0, max(1, G // 3))), replace=False)) if G > 3 else ()
    prob = make_problem(seed=2000 + seed, n=n, N=N, widths=widths, kappa=float(rng.choice([1.0, 2.0])), weights=weights,
                        constant_groups=const)
    link = str(rng.choice(["logit", "identity"]))
    orc = _oracle(prob, link)
    np.random.seed(seed)
    want = orc.shap_values(prob["X"], nsamples=nsamples, l1_reg=False)
    plans = [(Z, w) if Z is not None else None for (_, Z, w) in orc.plans]
    kernels = ["simt", "auto"] + (["tcgen05"] if G <= 15 and N <= 128 else [])
    for kernel in kernels:
        eng = _engine(prob, link, kernel=kernel)
        got = eng.shap_values(prob["X"], nsamples=nsamples, l1_reg=False, plans=plans)      # oracle's per-instance plans
        _compare(got, want)
        np.random.seed(77)
        shared = eng.shap_values(prob["X"], nsamples=nsamples, l1_reg=False)                # engine's shared plans
        fx = prob["clf"].predict_proba(prob["X"])
        lf = orc.link.f
        np.testing.assert_allclose(shared[1].sum(1), lf(fx[:, 1]) - eng.expected_value[1], rtol=1e-7, atol=1e-8)
    # shared plans: every kernel draws the same plan from the same stream state => same values
    res = []
    for kernel in kernels:
        np.random.seed(77)
        res.append(_engine(prob, link, kernel=kernel).shap_values(prob["X"], nsamples=nsamples, l1_reg=False)[1])
    for r in res[1:]:
        assert rel_err(r, res[0]) < 5e-6


def test_config2_shape_64_features_bg512():
    """BASELINE configs[2] shape at reduced n: 64 ungrouped features, 512 background rows, nsamples 4096."""
    from distributedkernelshap_b200.datasets import dense_tabular
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from oracle.shap_kernel_oracle import KernelExplainerOracle
    d = dense_tabular(n=6, n_features=64, n_background=512, seed=0)
    orc = KernelExplainerOracle(d["predictor"].predict_proba, d["background"], link="logit", record_plans=True)
    np.random.seed(0)
    want = orc.shap_values(d["X_explain"], nsamples=4096, l1_reg=False)
    eng = GpuKernelExplainer(d["predictor"].predict_proba, d["background"], link="logit")
    got = eng.shap_values(d["X_explain"], nsamples=4096, l1_reg=False, plans=[(Z, w) for (_, Z, w) in orc.plans])
    _compare(got, want)
    with pytest.raises(NotImplementedError):          # l1 selection runs on the engine's shared plans, not on these
        eng.shap_values(d["X_explain"], nsamples=4096, plans=[(Z, w) for (_, Z, w) in orc.plans])


def test_config2_shape_shared_plan():
    """configs[2] shape with the engine's own shared plan (M = 64: the plan's 63 x 63 normal matrix is factored on the
    device at upload) against the oracle fed that plan."""
    from distributedkernelshap_b200.datasets import dense_tabular
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.plan import build_plan
    from oracle.shap_kernel_oracle import KernelExplainerOracle
    d = dense_tabular(n=4, n_features=64, n_background=512, seed=1)
    orc = KernelExplainerOracle(d["predictor"].predict_proba, d["background"], link="logit")
    np.random.seed(5)
    eng = GpuKernelExplainer(d["predictor"].predict_proba, d["background"], link="logit")
    got = eng.shap_values(d["X_explain"], nsamples=4096, l1_reg=False)
    np.random.seed(5)
    plan = build_plan(64, 4096)
    for i in range(4):
        phi = orc.explain(d["X_explain"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=4096, l1_reg=False)
        for c in range(2):
            assert rel_err(got[c][i], phi[:, c]) < TOL


def test_config3_grouped_shape_1024_onehot_columns():
    """BASELINE configs[3] in its grouped reading (64 one-hot variables x 16 levels = 1024 columns, one group per
    variable) at a reduced background / budget the oracle can hold in memory: shared plan and per-instance plans."""
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import wide_onehot
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.plan import build_plan
    from oracle.shap_kernel_oracle import DenseData as ODenseData, KernelExplainerOracle
    d = wide_onehot(n=3, n_blocks=64, block_width=16, n_background=24, seed=2)
    orc = KernelExplainerOracle(d["predictor"].predict_proba, ODenseData(d["background"], d["group_names"], d["groups"]),
                                link="logit", record_plans=True)
    np.random.seed(1)
    want = orc.shap_values(d["X_explain"], nsamples=1500, l1_reg=False)
    np.random.seed(8)
    eng = GpuKernelExplainer(d["predictor"].predict_proba, DenseData(d["background"], d["group_names"], d["groups"]),
                             link="logit")
    got = eng.shap_values(d["X_explain"], nsamples=1500, l1_reg=False, plans=[(Z, w) for (_, Z, w) in orc.plans])
    _compare(got, want)
    shared = eng.shap_values(d["X_explain"], nsamples=1500, l1_reg=False)          # engine's own M = 64 plan
    np.random.seed(8)
    plan = build_plan(64, 1500)
    Ms, _ = eng.varying(d["X_explain"])
    for i in range(3):
        if Ms[i] != 64:
            continue
        phi = orc.explain(d["X_explain"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=1500, l1_reg=False)
        for c in range(2):
            assert rel_err(shared[c][i], phi[:, c]) < TOL


@pytest.mark.parametrize("N", [129, 300])
def test_shared_fast_path_with_backgrounds_larger_than_one_chunk(N):
    """The shared-plan fast path keeps 128 columns of Dm in registers; larger backgrounds go through in chunks whose
    (sum p1, sum p0) are accumulated."""
    from distributedkernelshap_b200.plan import build_plan
    prob = make_problem(seed=31, n=9, N=N, widths=(1, 2, 1, 1, 3, 1, 1, 2, 1))
    orc = _oracle(prob)
    np.random.seed(3)
    eng = _engine(prob, kernel="shared")
    got = eng.shap_values(prob["X"], nsamples=200, l1_reg=False)
    np.random.seed(3)
    plan = build_plan(9, 200)
    for i in range(prob["X"].shape[0]):
        phi = orc.explain(prob["X"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=200, l1_reg=False)
        for c in range(2):
            assert rel_err(got[c][i], phi[:, c]) < TOL


def test_large_input_is_chunked(monkeypatch):
    """Inputs above MAX_ROWS_PER_CALL are explained in row chunks with identical results."""
    from distributedkernelshap_b200 import engine as engine_mod
    prob = make_problem(seed=13, n=700, N=20, widths=(1, 1, 2, 1, 3, 1))
    np.random.seed(3)
    eng = _engine(prob)
    whole = eng.shap_values(prob["X"], nsamples=62, l1_reg=False)
    monkeypatch.setattr(engine_mod, "MAX_ROWS_PER_CALL", 256)
    chunked = eng.shap_values(prob["X"], nsamples=62, l1_reg=False)
    np.testing.assert_array_equal(chunked[1], whole[1])
    assert chunked[0].shape == (700, 6)


@pytest.mark.parametrize("link", ["logit", "identity"])
def test_multiclass_softmax_head(link):
    """C = 4 multinomial logistic regression (general softmax head, CUDA-core kernel) against the oracle."""
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.predictors import LinearSoftmaxClassifier
    from oracle.shap_kernel_oracle import DenseData as ODenseData, KernelExplainerOracle
    rng = np.random.default_rng(5)
    widths = (1, 2, 1, 3, 1, 1, 2)
    groups, start = [], 0
    for wd in widths:
        groups.append(list(range(start, start + wd))); start += wd
    D, N, n, C = start, 23, 14, 4
    bg, X = rng.standard_normal((N, D)), rng.standard_normal((n, D))
    clf = LinearSoftmaxClassifier(rng.normal(0, 0.8, (C, D)), rng.normal(0, 0.5, C))
    names = [f"g{i}" for i in range(len(groups))]
    wts = rng.uniform(0.3, 1.0, N)
    orc = KernelExplainerOracle(clf.predict_proba, ODenseData(bg, names, groups, wts), link=link, record_plans=True)
    eng = GpuKernelExplainer(clf.predict_proba, DenseData(bg, names, groups, wts), link=link)
    assert eng.vector_out and eng.D == C
    np.testing.assert_allclose(eng.expected_value, orc.expected_value, rtol=1e-12)
    want = orc.shap_values(X, nsamples=10 ** 6, l1_reg=False)              # full enumeration (M = 7)
    got = eng.shap_values(X, nsamples=10 ** 6, l1_reg=False)
    assert len(got) == C
    _compare(got, want)
    np.random.seed(4)
    want = orc.shap_values(X, nsamples=60, l1_reg=False)                   # sampled, per-instance plans
    got = eng.shap_values(X, nsamples=60, l1_reg=False, plans=[(Z, w) for (_, Z, w) in orc.plans[n:]])
    _compare(got, want)
    fx = clf.predict_proba(X)
    for c in range(C):
        np.testing.assert_allclose(got[c].sum(1), orc.link.f(fx[:, c]) - eng.expected_value[c], rtol=1e-7, atol=1e-8)


def test_two_word_coalition_rows_up_to_128_groups():
    """65..128 groups (BASELINE configs[4] has 128 ungrouped features): coalition rows take two 64-bit words; supported
    on the shared-plan path.  GPU against the oracle fed the engine's plan, at a size the oracle holds in memory."""
    from distributedkernelshap_b200.datasets import dense_tabular
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.plan import build_plan
    from oracle.shap_kernel_oracle import KernelExplainerOracle
    for G, N, ns, seed in [(128, 40, 1500, 0), (70, 33, 600, 1)]:
        d = dense_tabular(n=3, n_features=G, n_background=N, seed=seed)
        orc = KernelExplainerOracle(d["predictor"].predict_proba, d["background"], link="logit")
        np.random.seed(11)
        eng = GpuKernelExplainer(d["predictor"].predict_proba, d["background"], link="logit")
        got = eng.shap_values(d["X_explain"], nsamples=ns, l1_reg=False)
        np.random.seed(11)
        plan = build_plan(G, ns)
        assert plan.zbits.shape == (ns, 2)
        for i in range(3):
            phi = orc.explain(d["X_explain"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=ns, l1_reg=False)
            for c in range(2):
                assert rel_err(got[c][i], phi[:, c]) < TOL
        fx = d["predictor"].predict_proba(d["X_explain"])
        np.testing.assert_allclose(got[1].sum(1), np.log(fx[:, 1] / fx[:, 0]) - eng.expected_value[1], rtol=1e-8, atol=1e-8)
    # what the two-word path does not cover is refused, not approximated
    d = dense_tabular(n=2, n_features=80, n_background=8, seed=3)
    X = d["X_explain"].copy()
    X[0, 5] = d["background"][0, 5]
    d["background"][:, 5] = d["background"][0, 5]          # group 5 does not vary for instance 0: partial varying set
    eng = GpuKernelExplainer(d["predictor"].predict_proba, d["background"], link="logit")
    with pytest.raises(Exception, match="status 3|UNSUPPORTED|unsupported|more than 64"):
        eng.shap_values(X, nsamples=300, l1_reg=False)
    with pytest.raises(NotImplementedError):
        eng.shap_values(X[1:], nsamples=300, l1_reg=False, plans=[None])


def test_device_resident_calls_replay_as_one_cuda_graph():
    """explain_device on a user stream: the second identical call captures the launch sequence, later ones replay it.
    The graph reads the buffers at launch time, so new data under the same pointers gives new results."""
    import torch
    prob = make_problem(seed=51, n=40, N=14, widths=(1, 2, 1, 1, 3, 1, 1, 2))
    eng = _engine(prob)
    want = eng.shap_values(prob["X"], nsamples=120, l1_reg=False)           # host path; plans get built here
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(prob["X"]).cuda()
        phi = torch.zeros((2, 40, 8), dtype=torch.float64, device="cuda")
        for _ in range(4):
            eng.explain_device(X_dev.data_ptr(), 40, phi.data_ptr(), nsamples=120)
        eng.check_status()
        assert eng.graph_launches() >= 2
        np.testing.assert_allclose(phi[1].cpu().numpy(), want[1], rtol=0, atol=1e-12)
        X2 = prob["X"][::-1].copy()
        X_dev.copy_(torch.from_numpy(X2))
        eng.explain_device(X_dev.data_ptr(), 40, phi.data_ptr(), nsamples=120)
        eng.check_status()
        np.testing.assert_allclose(phi[1].cpu().numpy(), want[1][::-1], rtol=0, atol=1e-12)
        before = eng.graph_launches()
        eng.explain_device(X_dev.data_ptr(), 17, phi.data_ptr(), nsamples=120)   # another shape: plain launches
        eng.check_status()
        assert eng.graph_launches() == before
        np.testing.assert_allclose(phi.cpu().numpy().reshape(-1)[17 * 8 * 0:17 * 8].reshape(17, 8), -want[1][::-1][:17],
                                   rtol=0, atol=1e-12)
    eng.set_stream(0)


@pytest.mark.parametrize("kernel", ["auto", "tcgen05", "simt"])
def test_small_probabilities_keep_their_relative_precision(kernel):
    """Scores around -10 (p1 ~ 1e-9, about as far as the reference's own float64 ``log(x / (1 - x))`` stays meaningful for
    the complementary class): 2^t reaches 2^30 and the shared-plan kernel works with A and A^2 of the normalised rows.
    p1 and p0 are accumulated separately, so the small class keeps its relative precision."""
    from distributedkernelshap_b200.predictors import LinearSoftmaxClassifier
    prob = make_problem(seed=61, n=12, N=20, widths=(1, 1, 2, 1, 1, 3, 1, 1))
    rng = np.random.default_rng(5)
    prob["clf"] = LinearSoftmaxClassifier(rng.normal(0, 0.8, size=(1, 11)), np.array([-10.0]), multi_class="multinomial")
    orc, eng = _oracle(prob), _engine(prob, kernel=kernel)
    np.random.seed(2)
    want = orc.shap_values(prob["X"], nsamples=150, l1_reg=False)
    got = eng.shap_values(prob["X"], nsamples=150, l1_reg=False, plans=[(Z, w) for (_, Z, w) in orc.plans])
    for i in range(12):                      # class 1 (the small probability): the oracle's own 1 - x is exact there
        assert rel_err(got[1][i], want[1][i]) < TOL
    shared = eng.shap_values(prob["X"], nsamples=150, l1_reg=False)       # shared plan through the fast path
    fx = prob["clf"].predict_proba(prob["X"])
    np.testing.assert_allclose(shared[1].sum(1), np.log(fx[:, 1] / fx[:, 0]) - eng.expected_value[1], rtol=1e-8, atol=1e-8)
    assert np.abs(shared[1]).max() > 0.1
