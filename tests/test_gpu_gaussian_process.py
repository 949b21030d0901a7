"""Gaussian-process regressors, KernelRidge with a kernel object and one-class SVMs on the device (the kernel-machine
route's program kernel, ``last_path()['general'] == 'kmach'``) against the oracle fed the real scikit-learn method and the
coalition plans the engine used: every leaf of the kernel algebra, composites of up to four statistics, three targets,
both one-class SVM methods, partial varying sets, weighted and grouped backgrounds, every plan source, l1 selection, an
encoded pipeline, voting and stacking members, the tile edges, the device-resident entry and its graph replay, the public
``KernelShap`` API and the refusals."""
import warnings

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.ensemble import StackingRegressor, VotingRegressor  # noqa: E402
from sklearn.gaussian_process import GaussianProcessRegressor  # noqa: E402
from sklearn.gaussian_process.kernels import (RBF, ConstantKernel, DotProduct, ExpSineSquared, Matern,  # noqa: E402
                                              RationalQuadratic, WhiteKernel)
from sklearn.kernel_ridge import KernelRidge  # noqa: E402
from sklearn.linear_model import Ridge  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import OneHotEncoder, StandardScaler  # noqa: E402
from sklearn.svm import SVR, OneClassSVM  # noqa: E402

from distributedkernelshap_b200.kernel_machines import extract_kernel_machine_spec  # noqa: E402

PLAIN_TOL = 1e-9        # float64 end to end without selection
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point


def _ls(P):
    return np.linspace(0.8, 3.0, P)


KERNELS = {
    "rbf_percol": lambda P: RBF(_ls(P)),
    "matern05": lambda P: Matern(2.0, nu=0.5),
    "matern15": lambda P: Matern(_ls(P), nu=1.5),
    "matern25": lambda P: Matern(2.5, nu=2.5),
    "matern_inf": lambda P: Matern(_ls(P), nu=np.inf),
    "rq": lambda P: RationalQuadratic(length_scale=2.0, alpha=0.7),
    "expsine": lambda P: ExpSineSquared(length_scale=3.0, periodicity=20.0),
    "dot": lambda P: DotProduct(sigma_0=0.5),
    "const_white": lambda P: ConstantKernel(2.0) * RBF(1.5) + WhiteKernel(0.1),
    "power": lambda P: (DotProduct(sigma_0=1.0) + ConstantKernel(0.3)) ** 2,
    "rbf_plus_dot": lambda P: RBF(_ls(P)) + DotProduct(sigma_0=0.5),
    # C * RBF(per column) + C * Matern + DotProduct ** 2 + WhiteKernel: three statistics
    "composite": lambda P: (ConstantKernel(1.5) * RBF(_ls(P)) + ConstantKernel(0.7) * Matern(2.0, nu=2.5)
                            + DotProduct(sigma_0=0.4) ** 2 + WhiteKernel(0.2)),
    # four statistics: two squared distances with their own length scales, one unscaled, one dot product
    "four_stats": lambda P: (ConstantKernel(1.5) * RBF(_ls(P)) * Matern(2.0, nu=1.5) + RationalQuadratic(1.5, 0.8)
                             + DotProduct(sigma_0=0.4) ** 2 + WhiteKernel(0.2)),
}
# the kernel of each statistic count (the tile holds 32 / L support vectors)
BY_L = {1: "rbf_percol", 2: "rbf_plus_dot", 3: "composite", 4: "four_stats"}


def _fit(est, X, y):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return est.fit(X, y)


def _fit_data(seed, P, n=60):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    y = np.sin(X[:, 0]) + 0.3 * X[:, 1 % P] * X[:, 2 % P] - 0.2 * X[:, -1]
    return X, y, rng


def _gp(kernel, P, seed=0, n=60, targets=1, scaled=True, normalize_y=False):
    X, y, _ = _fit_data(seed, P, n)
    Y = y if targets == 1 else np.stack([y, 0.5 * y ** 2, 1.0 - y], axis=1)
    # ExpSineSquared is not positive definite over several columns: a larger noise term keeps the fit's Cholesky finite
    alpha = 1.0 if "ExpSineSquared" in repr(kernel) else 0.1
    est = GaussianProcessRegressor(kernel, alpha=alpha, optimizer=None, normalize_y=normalize_y)
    return _fit(make_pipeline(StandardScaler(), est) if scaled else est, X, Y)


def _problem(seed, P, N, n, constant_cols=(), weights=False, zero_row=False):
    rng = np.random.default_rng(seed + 1000)
    bg = rng.normal(size=(N, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    for c in constant_cols:              # partial varying sets: x equals the constant background column on some rows
        bg[:, c] = 0.25
        X[::2, c] = 0.25
    w = rng.uniform(0.1, 1.0, N) if weights else None
    if zero_row:
        w[1] = 0.0
    return bg, X, w


def _data(bg, w=None, groups=None):
    from distributedkernelshap_b200.data import DenseData
    groups = groups or [[k] for k in range(bg.shape[1])]
    return DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w)


def _engine(fn, bg, w=None, groups=None, **kw):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    return GpuKernelExplainer(fn, _data(bg, w, groups), link="identity", seed=7, **kw)


def _oracle(fn, bg, w=None, groups=None):
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    groups = groups or [[k] for k in range(bg.shape[1])]
    return KernelExplainerOracle(fn, DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w), link="identity")


def _as_list(phi):
    return phi if isinstance(phi, list) else [phi]


def _compare(got, oracle, X, plans, tol, l1_reg=False, nsamples="auto"):
    got = _as_list(got)
    worst = 0.0
    for i in range(X.shape[0]):
        want = oracle.explain(X[i:i + 1], plan=plans(i), l1_reg=l1_reg, nsamples=nsamples)
        want = want.reshape(want.shape[0], -1)
        for c in range(want.shape[1]):
            e = rel_err(got[c][i], want[:, c])
            worst = max(worst, e)
            assert e < tol, (i, c, e)
    return worst


def _own_plans(eng, X, ns="auto"):
    M, _ = eng.varying(X)
    return lambda i: None if M[i] < 2 else (eng.shared_plan(int(M[i]), ns).dense(), eng.shared_plan(int(M[i]), ns).weights)


def _check_additivity(eng, fn, got, X):
    fx = np.asarray(fn(X), dtype=np.float64).reshape(X.shape[0], -1)
    ev = np.atleast_1d(eng.expected_value)
    for c, ph in enumerate(_as_list(got)):
        np.testing.assert_allclose(ph.sum(1), fx[:, c] - ev[c], rtol=1e-8, atol=1e-8)


def _parity(fn, P, bg, X, tol=PLAIN_TOL, **kw):
    eng = _engine(fn, bg, **kw)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(fn, bg, w=kw.get("w"), groups=kw.get("groups")), X, _own_plans(eng, X), tol)
    _check_additivity(eng, fn, got, X)
    return eng, got


@pytest.mark.parametrize("kernel", list(KERNELS))
def test_parity_every_leaf_and_composite(kernel):
    P = 7
    gp = _gp(KERNELS[kernel](P), P)
    spec = extract_kernel_machine_spec(gp.predict)
    if kernel == "four_stats":
        assert spec.program.L == 4
    bg, X, _ = _problem(11, P, N=12, n=4, constant_cols=(6,))
    eng, _ = _parity(gp.predict, P, bg, X)
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {6, 7}                    # full and partial varying sets in one call


@pytest.mark.parametrize("normalize_y", [False, True])
def test_three_targets(normalize_y):
    P = 6
    gp = _gp(KERNELS["composite"](P), P, targets=3, normalize_y=normalize_y)
    bg, X, _ = _problem(12, P, N=10, n=3, constant_cols=(5,))
    _, got = _parity(gp.predict, P, bg, X)
    assert len(got) == 3


def test_kernel_ridge_with_a_kernel_object():
    P = 6
    X, y, _ = _fit_data(3, P)
    krr = _fit(make_pipeline(StandardScaler(), KernelRidge(alpha=0.5, kernel=Matern(2.0, nu=1.5) + DotProduct(0.3))),
               X, y)
    bg, X2, _ = _problem(13, P, N=9, n=3)
    _parity(krr.predict, P, bg, X2)


@pytest.mark.parametrize("kernel", ["rbf", "poly"])
@pytest.mark.parametrize("method", ["decision_function", "score_samples"])
def test_one_class_svm(method, kernel):
    P = 6
    X, _, _ = _fit_data(4, P, 150)
    oc = _fit(make_pipeline(StandardScaler(), OneClassSVM(kernel=kernel, nu=0.3)), X, None)
    bg, X2, _ = _problem(14, P, N=10, n=3, constant_cols=(5,))
    _parity(getattr(oc, method), P, bg, X2)


def test_weighted_background_with_a_zero_weight_row():
    P = 6
    gp = _gp(KERNELS["four_stats"](P), P)
    bg, X, w = _problem(3, P, N=10, n=3, weights=True, zero_row=True)
    _parity(gp.predict, P, bg, X, w=w)


def test_grouped_columns():
    P = 8
    gp = _gp(KERNELS["composite"](P), P)
    groups = [[0, 1], [2], [3, 4, 5], [6], [7]]
    bg, X, _ = _problem(5, P, N=9, n=3)
    eng = _engine(gp.predict, bg, groups=groups)
    got = eng.shap_values(X, l1_reg=False, nsamples=20)
    assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(gp.predict, bg, groups=groups), X, _own_plans(eng, X, 20), PLAIN_TOL, nsamples=20)


def test_per_instance_device_plans():
    P = 9
    gp = _gp(KERNELS["matern25"](P), P)
    bg, X, _ = _problem(21, P, N=8, n=4, constant_cols=(8,))
    eng = _engine(gp.predict, bg, plan_mode="per_instance")
    got = eng.shap_values(X, l1_reg=False, nsamples=300)
    assert eng.last_path()["general"] == "kmach"
    zb, w = eng.instance_plans()
    M, _ = eng.varying(X)
    from distributedkernelshap_b200.plan import resolve_nsamples

    def plans(i):
        S, _ = resolve_nsamples(int(M[i]), 300)
        k = np.arange(int(M[i]))
        Z = ((zb[i, :S, None] >> k.astype(np.uint64)) & np.uint64(1)).astype(np.uint8)
        return Z, w[i, :S]
    _compare(got, _oracle(gp.predict, bg), X, plans, PLAIN_TOL, nsamples=300)


def test_caller_supplied_plans():
    P = 6
    gp = _gp(KERNELS["rq"](P), P)
    bg, X, _ = _problem(8, P, N=7, n=3)
    rng = np.random.default_rng(0)
    plans = []
    for i in range(3):
        Z = rng.integers(0, 2, size=(40, P)).astype(np.uint8)
        Z[0] = 0
        Z[1] = 1
        Z[2:2 + P] = np.eye(P, dtype=np.uint8)
        plans.append((Z, rng.uniform(0.1, 1.0, 40)))
    eng = _engine(gp.predict, bg)
    got = eng.shap_values(X, l1_reg=False, nsamples=40, plans=plans)
    assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(gp.predict, bg), X, lambda i: plans[i], PLAIN_TOL, nsamples=40)


def test_l1_selection_auto():
    P = 14                                    # 'auto' selects: a fraction of the 16382 coalitions is evaluated
    gp = _gp(KERNELS["composite"](P), P)
    bg, X, _ = _problem(31, P, N=5, n=3, constant_cols=(13,))
    eng = _engine(gp.predict, bg)
    got = eng.shap_values(X, l1_reg="auto")
    path = eng.last_path()
    assert path["general"] in ("kmach", "simt", "none") and path["general_l1"] == 1, path
    _compare(got, _oracle(gp.predict, bg), X, _own_plans(eng, X), L1_TOL, l1_reg="auto")


def test_encoded_pipeline_in_front_of_a_gp():
    rng = np.random.default_rng(6)
    n = 80
    Xr = np.c_[rng.normal(size=(n, 3)), rng.integers(0, 3, size=n).astype(np.float64)]
    y = Xr[:, 0] + np.where(Xr[:, 3] == 1, 1.0, -0.5) + 0.3 * Xr[:, 1] * Xr[:, 2]
    ct = ColumnTransformer([("num", StandardScaler(), [0, 1, 2]), ("cat", OneHotEncoder(), [3])])
    pipe = _fit(make_pipeline(ct, GaussianProcessRegressor(RBF(2.0) + DotProduct(0.3), alpha=0.1, optimizer=None)),
                Xr, y)
    bg, X = Xr[:10].copy(), Xr[60:64].copy()
    eng = _engine(pipe.predict, bg)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(pipe.predict, bg), X, _own_plans(eng, X), PLAIN_TOL)
    _check_additivity(eng, pipe.predict, got, X)


@pytest.mark.parametrize("kind", ["voting", "stacking"])
def test_gp_as_an_ensemble_member(kind):
    P = 6
    X, y, _ = _fit_data(7, P, 80)
    gp = GaussianProcessRegressor(KERNELS["composite"](P), alpha=0.1, optimizer=None)
    if kind == "voting":
        ens = _fit(VotingRegressor([("gp", gp), ("svr", SVR()), ("ridge", Ridge())], weights=[2.0, 1.0, 0.5]), X, y)
    else:
        ens = _fit(StackingRegressor([("gp", gp), ("svr", SVR())], final_estimator=Ridge(), cv=3), X, y)
    bg, X2, _ = _problem(15, P, N=8, n=3, constant_cols=(5,))
    eng = _engine(ens.predict, bg)
    got = eng.shap_values(X2, l1_reg=False)
    assert eng.last_path()["general"] == ("ensemble" if kind == "voting" else "stacking")
    _compare(got, _oracle(ens.predict, bg), X2, _own_plans(eng, X2), PLAIN_TOL)
    _check_additivity(eng, ens.predict, got, X2)


@pytest.mark.parametrize("L,n_sv", [(1, 31), (1, 33), (2, 15), (2, 16), (2, 17), (3, 9), (3, 10), (3, 11), (3, 31),
                                    (4, 7), (4, 8), (4, 9), (4, 17)])
def test_training_rows_around_the_tile(L, n_sv):
    """the tile holds 32 // L support vectors of L statistics"""
    P = 5
    gp = _gp(KERNELS[BY_L[L]](P), P, seed=n_sv, n=n_sv)
    assert extract_kernel_machine_spec(gp.predict).program.L == L
    bg, X, _ = _problem(4, P, N=6, n=3, constant_cols=(4,))
    _parity(gp.predict, P, bg, X)


def test_64_groups():
    P = 64
    gp = _gp(KERNELS["composite"](P), P, n=40)
    rng = np.random.default_rng(2)
    bg = rng.normal(size=(4, P))
    X = rng.normal(size=(2, P))
    bg[:, 0] = 0.5
    X[:, 0] = 0.5
    eng = _engine(gp.predict, bg)
    got = eng.shap_values(X, l1_reg=False, nsamples=300)
    assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(gp.predict, bg), X, _own_plans(eng, X, 300), PLAIN_TOL, nsamples=300)
    _check_additivity(eng, gp.predict, got, X)


def test_shared_memory_limit():
    """8 outputs at 13 groups: the largest coalition count the one-statistic kernels take also fits four statistics"""
    import torch
    from distributedkernelshap_b200._cabi import DksError
    P, R = 13, 8
    limit = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    S = ((limit - 4 * 64) // 8 - max(32 * (1 + R + P + 16 * 4), 63 * 63 + 64)) // R
    X, y, _ = _fit_data(9, P, 40)
    Y = np.stack([y * (k + 1) + k for k in range(R)], axis=1)
    gp = _fit(GaussianProcessRegressor(KERNELS["four_stats"](P), alpha=0.1, optimizer=None), X, Y)
    assert extract_kernel_machine_spec(gp.predict).program.L == 4
    bg, X2, _ = _problem(7, P, N=3, n=2)
    eng = _engine(gp.predict, bg)
    got = eng.shap_values(X2, l1_reg=False, nsamples=S)
    assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(gp.predict, bg), X2, _own_plans(eng, X2, S), PLAIN_TOL, nsamples=S)
    with pytest.raises(DksError, match="shared memory"):
        _engine(gp.predict, bg).shap_values(X2, l1_reg=False, nsamples=S + 1)


def test_graph_replay_is_bit_identical_to_the_host_path():
    import torch
    P = 8
    gp = _gp(KERNELS["four_stats"](P), P, targets=3)
    bg, X, _ = _problem(41, P, N=10, n=16, constant_cols=(7,))
    eng = _engine(gp.predict, bg)
    want = np.stack(eng.shap_values(X, nsamples=200, l1_reg=False))
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(X).cuda()
        phi = torch.zeros((want.shape[0], 16, P), dtype=torch.float64, device="cuda")
        for _ in range(4):
            eng.explain_device(X_dev.data_ptr(), 16, phi.data_ptr(), nsamples=200)
        eng.check_status()
        assert eng.graph_launches() >= 1
        assert eng.last_path()["general"] == "kmach"
        np.testing.assert_array_equal(phi.cpu().numpy(), want)
    eng.set_stream(0)


def test_kernel_shap_default_kwargs():
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    d = adult_like(n_explain=60, n_background=30, seed=0)
    X_fit = d["X_explain"][:50]
    y = d["predictor"].predict_proba(X_fit)[:, 1]
    gpr = _fit(make_pipeline(StandardScaler(), GaussianProcessRegressor(
        ConstantKernel() * RBF(np.ones(X_fit.shape[1])) + WhiteKernel(), normalize_y=True)), X_fit, y)
    ks = KernelShap(gpr.predict, feature_names=d["group_names"], seed=0)
    ks.fit(d["background"], group_names=d["group_names"], groups=d["groups"])
    Xe = d["X_explain"][50:55]
    exp = ks.explain(Xe, silent=True)          # default kwargs: nsamples='auto', l1_reg='auto'
    assert ks._explainer.last_path()["general"] in ("kmach", "none")
    np.testing.assert_allclose(np.asarray(exp.shap_values[0]).sum(1), gpr.predict(Xe) - exp.expected_value[0],
                               rtol=1e-8, atol=1e-8)


def test_nan_refusals():
    P = 5
    gp = _gp(KERNELS["matern15"](P), P)
    bg, X, _ = _problem(2, P, N=6, n=2)
    eng = _engine(gp.predict, bg)
    Xn = X.copy()
    Xn[1, 2] = np.nan
    with pytest.raises(ValueError, match="instance 1"):
        eng.shap_values(Xn, l1_reg=False)
    bgn = bg.copy()
    bgn[3, 0] = np.nan
    with pytest.raises(ValueError, match="background row 3"):
        _engine(gp.predict, bgn)


def test_bad_programs_are_refused():
    """dks_set_kernel_program refuses out-of-range operands, a stack that overflows and non-finite constants"""
    import ctypes as C

    from distributedkernelshap_b200 import _cabi
    from distributedkernelshap_b200._cabi import DksError
    lib = _cabi.load()
    P = 3
    bg = np.random.default_rng(0).normal(size=(4, P))
    ctx = C.c_void_p()
    _cabi.check(lib.dks_create(C.byref(ctx), 0))
    try:
        _cabi.check(lib.dks_set_background(ctx, _cabi.ptr(bg), 4, P, None))
        sv = np.ascontiguousarray(bg[:2])
        one = np.ones((1, P))
        zero = np.zeros((1, P))
        _cabi.check(lib.dks_set_kernel_machine(ctx, 1, _cabi.ptr(np.array([0, 2], np.int32)), _cabi.ptr(sv),
                                               _cabi.ptr(np.ones(2)), 1, _cabi.ptr(np.zeros(1)), _cabi.ptr(one),
                                               _cabi.ptr(zero), _cabi.ptr(np.ones(1)), 4, 0.0, 0.0, 0, None, None, None,
                                               1))
        kinds = np.zeros(1, np.int32)

        def prog(ops, args, a, L=1):
            ops, args = np.asarray(ops, np.int32), np.asarray(args, np.int32)
            a = np.asarray(a, np.float64)
            b = np.ones(len(ops))
            return lib.dks_set_kernel_program(ctx, L, _cabi.ptr(kinds), _cabi.ptr(one), _cabi.ptr(zero), len(ops),
                                              _cabi.ptr(ops), _cabi.ptr(args), _cabi.ptr(a), _cabi.ptr(b))
        assert prog([2], [0], [0.5]) == 0                                       # exp(-t / 2)
        for bad in (([2], [1], [0.5]),                                          # statistic 1 of 1
                    ([0, 0, 0, 0, 0, 8, 8, 8, 8], [0] * 9, [1.0] * 9),          # five operands at once
                    ([8], [0], [0.0]),                                          # nothing to add
                    ([2, 2], [0, 0], [0.5, 0.5]),                               # two values left
                    ([2], [0], [np.inf]),                                       # non-finite constant
                    ([13], [0], [0.0])):                                        # unknown instruction
            with pytest.raises(DksError, match="dks_set_kernel_program"):
                _cabi.check(prog(*bad))
    finally:
        lib.dks_destroy(ctx)
