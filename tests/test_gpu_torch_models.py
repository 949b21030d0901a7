"""torch.nn.Module predictors on the device (the module route, ``last_path()['general'] == 'torch'``) against the oracle fed
``module(torch.as_tensor(x, dtype, device))`` and the coalition plans the engine used: float64 and float32 modules,
binary softmax under the logit link, one-column sigmoid outputs, multi-output regression, groups, partial varying sets,
M = 0 / 1 instances, weighted backgrounds, per-instance device plans, caller-supplied plans, l1 selection, the block
split of the masked rows, NaN outputs, the public ``KernelShap`` API, the refusals that need a device, and the same
phi as the MLP and shared-plan routes for the same function."""
import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

PLAIN_TOL = 1e-9        # float64 end to end without selection
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point, as on the MLP route
# float32 module: the engine and the oracle feed the module the same float32 rows (both round float64 to nearest), but the
# module sums a batch of masked rows where the oracle sums one instance's, and float32 GEMMs may reduce in another order
# per batch shape; a few float32 ulps (~1e-7) in y become ~1e-5 of max |phi| after the solve
F32_TOL = 1e-4


def _dev():
    return torch.device("cuda", 0)


def _mlp(P, C, dtype=torch.float64, head=None, hidden=16, seed=0):
    torch.manual_seed(seed)
    layers = [torch.nn.Linear(P, hidden), torch.nn.Tanh(), torch.nn.Linear(hidden, C)]
    if head is not None:
        layers.append(head)
    return torch.nn.Sequential(*layers).to(dtype=dtype, device=_dev()).eval()


class _Squeeze(torch.nn.Module):
    def forward(self, x):
        return x[:, 0]


def _fn(module, dtype):
    def f(x):
        with torch.inference_mode():
            return module(torch.as_tensor(np.asarray(x, dtype=np.float64), dtype=dtype, device=_dev())).double().cpu().numpy()
    return f


def _problem(seed, P, N, n, constant_cols=(), weights=False, zero_row=False):
    rng = np.random.default_rng(seed)
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


def _engine(fn, bg, link, w=None, groups=None, **kw):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    return GpuKernelExplainer(fn, _data(bg, w, groups), link=link, seed=7, **kw)


def _oracle(fn, bg, link, w=None, groups=None):
    from oracle.shap_kernel_oracle import DenseData, KernelExplainerOracle
    groups = groups or [[k] for k in range(bg.shape[1])]
    return KernelExplainerOracle(fn, DenseData(bg, [f"g{i}" for i in range(len(groups))], groups, w), link=link)


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


def _own_plans(eng, M, ns="auto"):
    return lambda i: None if M[i] < 2 else (eng.shared_plan(int(M[i]), ns).dense(), eng.shared_plan(int(M[i]), ns).weights)


def _explain(eng, X, **kw):
    """phi on the module route and M of every row, read from the call's own stage 1 (a module's needs its outputs)."""
    from distributedkernelshap_b200 import _cabi
    got = eng.shap_values(X, **kw)
    assert eng.last_path()["general"] == "torch", eng.last_path()
    M = np.zeros(X.shape[0], dtype=np.int32)
    _cabi.check(eng.lib.dks_get_varying(eng._ctx, _cabi.ptr(M), None))
    return got, M


def _additivity(eng, fn, got, X, link):
    from distributedkernelshap_b200.data import convert_to_link
    fx = np.asarray(fn(X), dtype=np.float64).reshape(X.shape[0], -1)
    ev = np.atleast_1d(eng.expected_value)
    for c, ph in enumerate(_as_list(got)):
        np.testing.assert_allclose(ph.sum(1), convert_to_link(link).f(fx[:, c]) - ev[c], rtol=1e-8, atol=1e-8)


@pytest.mark.parametrize("C,head,link", [(2, "softmax", "logit"), (2, "softmax", "identity"), (3, None, "identity"),
                                         (8, None, "identity")])
def test_float64_modules(C, head, link):
    P = 7
    module = _mlp(P, C, head=torch.nn.Softmax(dim=1) if head == "softmax" else None)
    fn = _fn(module, torch.float64)
    bg, X, _ = _problem(11, P, N=12, n=4, constant_cols=(6,))
    eng = _engine(module, bg, link)
    got, M = _explain(eng, X, l1_reg=False)
    assert {int(m) for m in M} == {6, 7}                    # full and partial varying sets in one call
    _compare(got, _oracle(fn, bg, link), X, _own_plans(eng, M), PLAIN_TOL)
    _additivity(eng, fn, got, X, link)


def test_float32_module():
    P = 6
    module = _mlp(P, 2, dtype=torch.float32, head=torch.nn.Softmax(dim=1))
    fn = _fn(module, torch.float32)
    bg, X, _ = _problem(3, P, N=20, n=4)
    eng = _engine(module, bg, "logit")
    got, M = _explain(eng, X, l1_reg=False)
    worst = _compare(got, _oracle(fn, bg, "logit"), X, _own_plans(eng, M), F32_TOL)
    print(f"float32 module: max|d|/max|phi| = {worst:.2e}")


@pytest.mark.parametrize("scalar", [True, False])
def test_one_column_sigmoid(scalar):
    P = 5
    head = torch.nn.Sequential(torch.nn.Sigmoid(), _Squeeze()) if scalar else torch.nn.Sigmoid()
    module = _mlp(P, 1, head=head)
    fn = _fn(module, torch.float64)
    bg, X, _ = _problem(5, P, N=9, n=3)
    eng = _engine(module, bg, "logit")
    assert eng.vector_out == (not scalar)
    got, M = _explain(eng, X, l1_reg=False)
    assert isinstance(got, list) != scalar
    _compare(got, _oracle(fn, bg, "logit"), X, _own_plans(eng, M), PLAIN_TOL)


def test_groups_and_zero_or_one_varying_groups():
    P = 6
    module = _mlp(P, 3)
    fn = _fn(module, torch.float64)
    _, X, _ = _problem(9, P, N=1, n=5)
    bg = np.tile(X[4], (5, 1))                               # every background row the same: x decides which groups vary
    groups = [[0, 3], [1], [2, 4], [5]]
    X[1, [0, 1, 3, 5]] = bg[0, [0, 1, 3, 5]]                 # row 1: group 2 only (M = 1)
    X[2] = bg[0]                                             # row 2: nothing varies (M = 0)
    X[3, [2, 4, 5]] = bg[0, [2, 4, 5]]                       # row 3: groups 0 and 1 (M = 2)
    X[4, 0] += 1.0                                           # row 4: group 0 only, through one of its two columns
    eng = _engine(module, bg, "identity", groups=groups)
    got, M = _explain(eng, X, l1_reg=False)
    assert list(M) == [4, 1, 0, 2, 1]
    _compare(got, _oracle(fn, bg, "identity", groups=groups), X, _own_plans(eng, M), PLAIN_TOL)
    _additivity(eng, fn, got, X, "identity")
    for i in np.where(M == 0)[0]:
        assert all(np.all(g[i] == 0) for g in _as_list(got))


def test_weighted_background_with_a_zero_weight():
    P = 5
    module = _mlp(P, 2, head=torch.nn.Softmax(dim=1))
    fn = _fn(module, torch.float64)
    bg, X, w = _problem(13, P, N=11, n=3, weights=True, zero_row=True)
    eng = _engine(module, bg, "logit", w=w)
    got, M = _explain(eng, X, l1_reg=False)
    _compare(got, _oracle(fn, bg, "logit", w=w), X, _own_plans(eng, M), PLAIN_TOL)


def test_per_instance_device_plans():
    P = 9
    module = _mlp(P, 3)
    fn = _fn(module, torch.float64)
    bg, X, _ = _problem(21, P, N=8, n=5, constant_cols=(8,))
    eng = _engine(module, bg, "identity", plan_mode="per_instance")
    got, M = _explain(eng, X, l1_reg=False, nsamples=300)
    zb, w = eng.instance_plans()
    from distributedkernelshap_b200.plan import resolve_nsamples

    def plans(i):
        S, _ = resolve_nsamples(int(M[i]), 300)
        k = np.arange(int(M[i]))
        Z = ((zb[i, :S, None] >> k.astype(np.uint64)) & np.uint64(1)).astype(np.uint8)
        return Z, w[i, :S]
    _compare(got, _oracle(fn, bg, "identity"), X, plans, PLAIN_TOL, nsamples=300)


def test_caller_supplied_plans():
    P = 6
    module = _mlp(P, 2, head=torch.nn.Softmax(dim=1))
    fn = _fn(module, torch.float64)
    bg, X, _ = _problem(8, P, N=7, n=3)
    rng = np.random.default_rng(0)
    plans = []
    for i in range(3):
        Z = rng.integers(0, 2, size=(40, P)).astype(np.uint8)
        Z[0] = 0
        Z[1] = 1
        Z[2:2 + P] = np.eye(P, dtype=np.uint8)
        plans.append((Z, rng.uniform(0.1, 1.0, 40)))
    eng = _engine(module, bg, "logit")
    got, M = _explain(eng, X, l1_reg=False, nsamples=40, plans=plans)
    _compare(got, _oracle(fn, bg, "logit"), X, lambda i: plans[i], PLAIN_TOL, nsamples=40)


def test_l1_auto_selects():
    P = 14                                    # 'auto' selects: 2076 of 16382 coalitions evaluated
    module = _mlp(P, 2, head=torch.nn.Softmax(dim=1))
    fn = _fn(module, torch.float64)
    bg, X, _ = _problem(31, P, N=5, n=3, constant_cols=(13,))
    eng = _engine(module, bg, "logit")
    got, M = _explain(eng, X, l1_reg="auto")
    assert eng.last_path()["general_l1"] == 1
    _compare(got, _oracle(fn, bg, "logit"), X, _own_plans(eng, M), L1_TOL, l1_reg="auto")


class _RowWise(torch.nn.Module):
    """A row-wise function of elementwise ops only: its value on a row does not depend on the batch around it."""

    def __init__(self, P):
        super().__init__()
        self.a = torch.nn.Parameter(torch.linspace(0.3, 1.2, P, dtype=torch.float64))

    def forward(self, x):
        t = torch.tanh(x * self.a)
        return torch.stack([t[:, 0] * t[:, 1] + t[:, 2], torch.sin(x[:, 3]) - t[:, 1]], dim=1)


@pytest.mark.parametrize("rowwise", [True, False])
def test_model_batch_rows_do_not_change_phi(rowwise):
    P, N = 6, 10
    module = _RowWise(P).to(_dev()).eval() if rowwise else _mlp(P, 2)
    bg, X, _ = _problem(17, P, N=N, n=4, constant_cols=(5,))
    from distributedkernelshap_b200.plan import resolve_nsamples
    S = resolve_nsamples(P, 60)[0]
    results = []
    for rows in (None, N, (S + S // 2) * N + 3, 3 * S * N):   # default, one coalition, splits an instance, spans several
        eng = _engine(module, bg, "identity", model_batch_rows=rows)
        results.append(_as_list(_explain(eng, X, l1_reg=False, nsamples=60)[0]))
    for other in results[1:]:
        for a, b in zip(results[0], other):
            if rowwise:
                np.testing.assert_array_equal(a, b)
            else:
                np.testing.assert_allclose(a, b, rtol=0, atol=1e-12 * np.abs(a).max())


class _NanWhere(torch.nn.Module):
    """NaN where column 0 exceeds 1.5 and column 1 is below -1.5, a linear function elsewhere."""

    def __init__(self, P):
        super().__init__()
        self.lin = torch.nn.Linear(P, 1).double()

    def forward(self, x):
        y = self.lin(x)
        bad = (x[:, :1] > 1.5) & (x[:, 1:2] < -1.5)
        return torch.where(bad, torch.full_like(y, float("nan")), y)


@pytest.mark.parametrize("where", ["f(x)", "coalitions only"])
def test_nan_outputs_raise_numeric(where):
    from distributedkernelshap_b200._cabi import DKS_ERR_NUMERIC, DksError
    P = 4
    module = _NanWhere(P).to(_dev()).eval()
    bg, X, _ = _problem(2, P, N=6, n=2)
    bg[:, 0] = -1.0                                           # the background is finite: column 0 never exceeds 1.5
    X[:, 0] = [3.0, 2.0]
    if where == "f(x)":
        X[:, 1] = -3.0                                        # f(x) is NaN (stage 1 reports it)
    else:
        X[:, 1] = 0.0                                         # f(x) is finite ...
        bg[:, 1] = -3.0                                       # ... but x_0 over bg_1 is NaN: only the tail sees it
        assert np.isfinite(_fn(module, torch.float64)(X)).all() and np.isfinite(_fn(module, torch.float64)(bg)).all()
    eng = _engine(module, bg, "identity")
    with pytest.raises(DksError) as e:
        eng.shap_values(X, l1_reg=False)
    assert e.value.code == DKS_ERR_NUMERIC


def test_independent_sigmoid_outputs_under_the_logit():
    """Two independent sigmoids (outputs that do not sum to one) under the logit link: every output's elementwise logit,
    as the oracle takes it."""
    P = 6
    module = _mlp(P, 2, head=torch.nn.Sigmoid())
    fn = _fn(module, torch.float64)
    bg, X, _ = _problem(19, P, N=10, n=4, constant_cols=(5,))
    assert np.abs(fn(bg).sum(axis=1) - 1).min() > 1e-3
    eng = _engine(module, bg, "logit")
    got, M = _explain(eng, X, l1_reg=False)
    _compare(got, _oracle(fn, bg, "logit"), X, _own_plans(eng, M), PLAIN_TOL)
    _additivity(eng, fn, got, X, "logit")


def test_float32_masked_rows_round_like_torch():
    """A float32 row-wise module of elementwise ops sees, on the engine's masked rows, the values it sees on
    torch.as_tensor(masked row, float32): the oracle's y agree to the last bit, so phi agrees to float64 rounding of the
    sums (a mask that truncated instead of rounding would move y by float32 ulps, ~1e-7 relative)."""
    P = 6
    module = _RowWise(P).to(dtype=torch.float32, device=_dev()).eval()
    fn = _fn(module, torch.float32)
    rng = np.random.default_rng(4)
    bg = rng.normal(size=(9, P)) / 3.0                        # not representable in float32: every row is rounded
    X = rng.normal(size=(4, P)) / 3.0
    eng = _engine(module, bg, "identity")
    got, M = _explain(eng, X, l1_reg=False)
    _compare(got, _oracle(fn, bg, "identity"), X, _own_plans(eng, M), PLAIN_TOL)


def test_steps_refuse_a_call_begun_before_a_change():
    """After dks_external_begin, a change of options or another stage 1 makes the later steps refuse, not launch on stale
    state."""
    import ctypes as C
    from distributedkernelshap_b200 import _cabi
    from distributedkernelshap_b200.engine import _dtype_code
    P = 5
    module = _mlp(P, 2)
    bg, X, _ = _problem(6, P, N=6, n=3)
    eng = _engine(module, bg, "identity")
    eng.shap_values(X, l1_reg=False)                          # plans uploaded
    lib, ctx = eng.lib, eng._ctx
    Xd = torch.as_tensor(X, device=_dev())
    fx = module(Xd).detach().contiguous()
    out = torch.empty((10 * 6, P), dtype=torch.float64, device=_dev())

    def begin():
        _cabi.check(lib.dks_external_prepare(ctx, C.c_void_p(Xd.data_ptr()), 3, C.c_void_p(fx.data_ptr()),
                                             _dtype_code(fx)))
        total = C.c_int64(0)
        _cabi.check(lib.dks_external_begin(ctx, None, None, 0, C.byref(total)))
        assert total.value >= 6
    begin()
    assert lib.dks_external_mask(ctx, 0, 6, C.c_void_p(out.data_ptr())) == _cabi.DKS_OK
    _cabi.check(lib.dks_set_nsamples(ctx, 7))
    assert lib.dks_external_mask(ctx, 0, 6, C.c_void_p(out.data_ptr())) == _cabi.DKS_ERR_INVALID
    _cabi.check(lib.dks_set_nsamples(ctx, 0))
    assert lib.dks_external_mask(ctx, 0, 6, C.c_void_p(out.data_ptr())) == _cabi.DKS_ERR_INVALID   # dropped for good
    begin()
    _cabi.check(lib.dks_external_prepare(ctx, C.c_void_p(Xd.data_ptr()), 3, C.c_void_p(fx.data_ptr()), _dtype_code(fx)))
    assert lib.dks_external_reduce(ctx, 0, 6, C.c_void_p(out.data_ptr()), _cabi.EXTERNAL_FLOAT64) == _cabi.DKS_ERR_INVALID
    phi = np.empty((2, 3, P))
    assert lib.dks_external_finish(ctx, _cabi.ptr(phi)) == _cabi.DKS_ERR_INVALID
    eng._nsamples_req = None                                  # the engine's cache of nsamples: set it again
    eng.shap_values(X, l1_reg=False)                          # the next full call runs


def test_refusals_on_the_device():
    P = 4
    bg, X, _ = _problem(1, P, N=5, n=2)
    with pytest.raises(NotImplementedError, match="kernel"):
        _engine(_mlp(P, 2), bg, "identity", kernel="tcgen05")
    with pytest.raises(NotImplementedError, match="kernel"):
        _engine(_mlp(P, 2), bg, "identity", kernel="shared")
    with pytest.raises(ValueError, match="outputs"):
        _engine(_mlp(P, 9), bg, "identity")

    class _Wide(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.ones(1, dtype=torch.float64))

        def forward(self, x):
            return x.reshape(x.shape[0], 1, -1) * self.w
    with pytest.raises(ValueError, match="expected"):
        _engine(_Wide().to(_dev()).eval(), bg, "identity")
    bg70 = np.random.default_rng(0).normal(size=(4, 70))
    with pytest.raises(NotImplementedError, match="64 groups"):
        _engine(_mlp(70, 2), bg70, "identity")
    eng = _engine(_mlp(P, 2), bg, "identity")
    phi = torch.empty((2, 2, P), dtype=torch.float64, device=_dev())
    Xd = torch.as_tensor(X, device=_dev())
    with pytest.raises(NotImplementedError, match="explain_device"):
        eng.explain_device(Xd.data_ptr(), 2, phi.data_ptr())
    with pytest.raises(NotImplementedError, match="explain_block_to_device"):
        eng.explain_block_to_device(X)
    module = _mlp(P, 2)
    state = {k: v.clone() for k, v in module.state_dict().items()}
    eng = _engine(module, bg, "identity")
    eng.shap_values(X, l1_reg=False)
    assert not module.training
    assert all(torch.equal(state[k], v) for k, v in module.state_dict().items())


def test_kernel_shap_public_api():
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.data import convert_to_link
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    d = adult_like(n_explain=20, n_background=40, seed=0)
    P = d["background"].shape[1]
    module = _mlp(P, 2, head=torch.nn.Softmax(dim=1), hidden=32)
    ks = KernelShap(module, link="logit", feature_names=d["group_names"], seed=0, model_batch_rows=5000)
    ks.fit(d["background"], group_names=d["group_names"], groups=d["groups"])
    exp = ks.explain(d["X_explain"][:5], silent=True)
    assert ks._explainer.last_path()["general"] == "torch"
    fx = _fn(module, torch.float64)(d["X_explain"][:5])
    lfx = convert_to_link("logit").f(fx)
    np.testing.assert_allclose(exp.data["raw"]["raw_prediction"], lfx, rtol=1e-10, atol=1e-12)
    for c in range(2):
        np.testing.assert_allclose(exp.shap_values[c].sum(1), lfx[:, c] - exp.expected_value[c], rtol=1e-8, atol=1e-8)
    imp = exp.data["raw"]["importances"]
    want = np.abs(np.stack(exp.shap_values)).mean(axis=1).sum(axis=0)     # mean |phi| per output, summed
    np.testing.assert_allclose(imp["aggregated"]["ranked_effect"], np.sort(want)[::-1], rtol=1e-10)
    # raw predictions without the device's stage 1 go through the module on the device too
    bx = ks.build_explanation(d["X_explain"][:5], exp.shap_values, list(exp.expected_value))
    np.testing.assert_allclose(bx.data["raw"]["raw_prediction"], lfx, rtol=1e-10, atol=1e-12)


def test_same_phi_as_the_mlp_route():
    """A fitted MLPClassifier rewritten as a float64 nn.Sequential: the MLP route's phi."""
    import warnings
    from sklearn.exceptions import ConvergenceWarning
    from sklearn.neural_network import MLPClassifier
    P = 7
    bg, X, _ = _problem(23, P, N=12, n=4, constant_cols=(6,))
    rng = np.random.default_rng(1)
    Xf = rng.normal(size=(200, P))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        clf = MLPClassifier(hidden_layer_sizes=(10, 6), activation="tanh", max_iter=60, random_state=0).fit(
            Xf, (Xf[:, 0] + Xf[:, 1] * Xf[:, 2] > 0).astype(int))
    layers = []
    for k, (W, b) in enumerate(zip(clf.coefs_, clf.intercepts_)):
        lin = torch.nn.Linear(*W.shape).double()
        with torch.no_grad():
            lin.weight.copy_(torch.as_tensor(W.T))
            lin.bias.copy_(torch.as_tensor(b))
        layers.append(lin)
        layers.append(torch.nn.Tanh() if k < len(clf.coefs_) - 1 else torch.nn.Sigmoid())

    class _Proba(torch.nn.Module):
        def forward(self, p):
            return torch.cat([1 - p, p], dim=1)
    module = torch.nn.Sequential(*layers, _Proba()).to(_dev()).eval()
    np.testing.assert_allclose(_fn(module, torch.float64)(X), clf.predict_proba(X), rtol=1e-12, atol=1e-14)
    ref = _engine(clf.predict_proba, bg, "logit")
    want = _as_list(ref.shap_values(X, l1_reg=False))
    assert ref.last_path()["general"] == "mlp"
    eng = _engine(module, bg, "logit")
    got = _as_list(_explain(eng, X, l1_reg=False)[0])
    for c in range(2):
        assert rel_err(got[c], want[c]) < PLAIN_TOL


def test_same_phi_as_the_shared_plan_route():
    """A LogisticRegression rewritten as Linear + softmax: the shared-plan route's phi."""
    from sklearn.linear_model import LogisticRegression
    P = 8
    bg, X, _ = _problem(29, P, N=15, n=6)
    rng = np.random.default_rng(2)
    Xf = rng.normal(size=(200, P))
    clf = LogisticRegression().fit(Xf, (Xf[:, 0] - Xf[:, 3] > 0).astype(int))
    lin = torch.nn.Linear(P, 2).double()
    with torch.no_grad():
        w, b = clf.coef_[0], clf.intercept_[0]
        lin.weight.copy_(torch.as_tensor(np.stack([-w / 2, w / 2])))
        lin.bias.copy_(torch.as_tensor([-b / 2, b / 2]))
    module = torch.nn.Sequential(lin, torch.nn.Softmax(dim=1)).to(_dev()).eval()
    ref = _engine(clf.predict_proba, bg, "logit")
    want = _as_list(ref.shap_values(X, l1_reg=False))
    assert ref.last_path()["shared"] != "none"
    got = _as_list(_explain(_engine(module, bg, "logit"), X, l1_reg=False)[0])
    for c in range(2):
        assert rel_err(got[c], want[c]) < PLAIN_TOL
