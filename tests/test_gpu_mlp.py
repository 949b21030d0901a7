"""Multi-layer perceptrons on the device (the MLP route, ``last_path()['general'] == 'mlp'``) against the oracle fed the
model's own method and the coalition plans the engine used: every activation, head and link, widths around the FP64 mma
fragment shapes, depths 1 to 4, varying-set sizes around the 16-wide K step, full and partial varying sets, weighted
backgrounds, per-instance device plans, caller-supplied plans, l1 selection, the kernel's own edges, the device-resident
entry and its graph replay, the public ``KernelShap`` API and the refusals."""
import warnings

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.exceptions import ConvergenceWarning  # noqa: E402
from sklearn.neural_network import MLPClassifier, MLPRegressor  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import MinMaxScaler, StandardScaler  # noqa: E402

from distributedkernelshap_b200.mlp import MlpSpec, extract_mlp_spec  # noqa: E402

PLAIN_TOL = 1e-9        # float64 end to end without selection
L1_TOL = 1e-5           # the l1 moments go through the 2^-40 fixed point


def _fit_data(seed, P, n=150):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    s = X[:, 0] - X[:, 0].mean() + 0.5 * (X[:, 1 % P] - X[:, 1 % P].mean()) * (X[:, 2 % P] - X[:, 2 % P].mean())
    return X, s, rng


def _sk(est, X, y, scaler=StandardScaler):
    model = make_pipeline(scaler(), est) if scaler is not None else est
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return model.fit(X, y)


def _model(head, act, P, hidden=(9, 6), seed=0):
    """The scikit-learn method of a fitted MLP with the given head."""
    X, s, _ = _fit_data(seed, P)
    if head == "sigmoid":
        return _sk(MLPClassifier(hidden_layer_sizes=hidden, activation=act, max_iter=80, random_state=0), X,
                   (s > 0).astype(int)).predict_proba
    if head == "softmax":
        y = np.digitize(s, np.quantile(s, [0.3, 0.6]))
        return _sk(MLPClassifier(hidden_layer_sizes=hidden, activation=act, max_iter=80, random_state=0), X, y).predict_proba
    Y = np.stack([s, 2 * s + X[:, 1], X[:, 2] - s], axis=1)
    return _sk(MLPRegressor(hidden_layer_sizes=hidden, activation=act, max_iter=80, random_state=0), X, Y,
               MinMaxScaler).predict


def _problem(seed, P, N, n, constant_cols=(), weights=False, zero_row=False):
    _, _, rng = _fit_data(seed, P, 4)
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


def _own_plans(eng, X, ns="auto"):
    M, _ = eng.varying(X)
    return lambda i: None if M[i] < 2 else (eng.shared_plan(int(M[i]), ns).dense(), eng.shared_plan(int(M[i]), ns).weights)


def _check_additivity(eng, fn, got, X, link):
    from distributedkernelshap_b200.data import convert_to_link
    lk = convert_to_link(link)
    fx = np.asarray(fn(X), dtype=np.float64).reshape(X.shape[0], -1)
    ev = np.atleast_1d(eng.expected_value)
    for c, ph in enumerate(_as_list(got)):
        np.testing.assert_allclose(ph.sum(1), lk.f(fx[:, c]) - ev[c], rtol=1e-8, atol=1e-8)


def _hand_spec(widths, act="tanh", head="identity", seed=0, scale=1.0):
    """An MLP of random layers: widths = [D, H_1, .., R]."""
    rng = np.random.default_rng(seed)
    coefs = [rng.normal(size=(k, h)) * scale / np.sqrt(k) for k, h in zip(widths[:-1], widths[1:])]
    intercepts = [rng.normal(size=h) * 0.3 for h in widths[1:]]
    return MlpSpec(coefs, intercepts, act, head, widths[0], scalar_out=head == "identity" and widths[-1] == 1)


CASES = [(act, head, link) for act in ("identity", "logistic", "tanh", "relu") for head in ("identity", "sigmoid", "softmax")
         for link in (("identity",) if head == "identity" else ("identity", "logit"))]


@pytest.mark.parametrize("act,head,link", CASES)
def test_parity_every_activation_head_and_link(act, head, link):
    P = 7
    fn = _model(head, act, P)
    bg, X, _ = _problem(11, P, N=12, n=4, constant_cols=(6,))
    eng = _engine(fn, bg, link)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "mlp" and eng.last_path()["shared"] == "none"
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {6, 7}                    # full and partial varying sets in one call
    worst = _compare(got, _oracle(fn, bg, link), X, _own_plans(eng, X), PLAIN_TOL)
    print(f"{act} {head} {link}: max|d|/max|phi| = {worst:.2e}")
    _check_additivity(eng, fn, got, X, link)
    if head == "sigmoid":
        out = _as_list(got)
        np.testing.assert_array_equal(out[0], -out[1] + 0.0)    # class 0 is the exact negation of class 1


@pytest.mark.parametrize("width", [1, 7, 8, 9, 16, 17, 100, 256])
def test_widths_around_the_fragment_shapes(width):
    P = 6
    spec = _hand_spec([P, width, width, 3], act="logistic", head="softmax", seed=width)   # padded logistic units output 0.5
    bg, X, _ = _problem(4, P, N=6, n=3, constant_cols=(5,))
    eng = _engine(spec, bg, "logit")
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "mlp"
    _compare(got, _oracle(spec, bg, "logit"), X, _own_plans(eng, X), PLAIN_TOL)
    _check_additivity(eng, spec, got, X, "logit")


@pytest.mark.parametrize("depth", [1, 2, 3, 4])
def test_depths(depth):
    P = 8
    fn = _model("softmax", "tanh", P, hidden=(12, 7, 9, 5)[:depth], seed=depth)
    assert extract_mlp_spec(fn).n_hidden == depth
    bg, X, _ = _problem(depth, P, N=7, n=3, constant_cols=(0,))
    eng = _engine(fn, bg, "identity")
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "mlp"
    _compare(got, _oracle(fn, bg, "identity"), X, _own_plans(eng, X), PLAIN_TOL)


@pytest.mark.parametrize("M", [0, 1, 2, 15, 16, 17])
def test_varying_set_sizes_around_the_k_step(M):
    P = 20
    spec = _hand_spec([P, 24, 1], act="relu", head="sigmoid", seed=M)
    rng = np.random.default_rng(M)
    bg = rng.normal(size=(5, P))
    X = rng.normal(size=(3, P))
    bg[:, M:] = 0.5
    X[:, M:] = 0.5
    eng = _engine(spec, bg, "logit")
    ns = 600
    got = eng.shap_values(X, l1_reg=False, nsamples=ns)
    got_M, _ = eng.varying(X)
    assert {int(m) for m in got_M} == {M}
    if M >= 2:
        assert eng.last_path()["general"] == "mlp"
    _compare(got, _oracle(spec, bg, "logit"), X, _own_plans(eng, X, ns), PLAIN_TOL, nsamples=ns)
    _check_additivity(eng, spec, got, X, "logit")


@pytest.mark.parametrize("which", ["first", "last"])
def test_64_groups_with_one_not_varying(which):
    P = 64
    spec = _hand_spec([P, 33, 2], act="tanh", head="identity", seed=3)
    rng = np.random.default_rng(2)
    bg = rng.normal(size=(4, P))
    X = rng.normal(size=(2, P))
    c = 0 if which == "first" else P - 1                     # group 0 or 63 does not vary
    bg[:, c] = 0.5
    X[:, c] = 0.5
    eng = _engine(spec, bg, "identity")
    got = eng.shap_values(X, l1_reg=False, nsamples=300)
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {63} and eng.last_path()["general"] == "mlp"
    _compare(got, _oracle(spec, bg, "identity"), X, _own_plans(eng, X, 300), PLAIN_TOL, nsamples=300)


def test_weighted_background_with_a_zero_weight_row():
    P = 6
    fn = _model("sigmoid", "relu", P)
    bg, X, w = _problem(3, P, N=10, n=3, weights=True, zero_row=True)
    eng = _engine(fn, bg, "logit", w=w)
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "mlp"
    _compare(got, _oracle(fn, bg, "logit", w=w), X, _own_plans(eng, X), PLAIN_TOL)


def test_grouped_columns():
    P = 8
    fn = _model("identity", "logistic", P)
    groups = [[0, 1], [2], [3, 4, 5], [6], [7]]
    bg, X, _ = _problem(5, P, N=9, n=3)
    eng = _engine(fn, bg, "identity", groups=groups)
    got = eng.shap_values(X, l1_reg=False, nsamples=20)
    assert eng.last_path()["general"] == "mlp"
    _compare(got, _oracle(fn, bg, "identity", groups=groups), X, _own_plans(eng, X, 20), PLAIN_TOL, nsamples=20)


def test_per_instance_device_plans():
    P = 9
    fn = _model("softmax", "relu", P)
    bg, X, _ = _problem(21, P, N=8, n=5, constant_cols=(8,))
    eng = _engine(fn, bg, "identity", plan_mode="per_instance")
    got = eng.shap_values(X, l1_reg=False, nsamples=300)
    assert eng.last_path()["general"] == "mlp"
    zb, w = eng.instance_plans()
    M, _ = eng.varying(X)
    from distributedkernelshap_b200.plan import resolve_nsamples

    def plans(i):
        S, _ = resolve_nsamples(int(M[i]), 300)
        k = np.arange(int(M[i]))
        Z = ((zb[i, :S, None] >> k.astype(np.uint64)) & np.uint64(1)).astype(np.uint8)
        return Z, w[i, :S]
    _compare(got, _oracle(fn, bg, "identity"), X, plans, PLAIN_TOL, nsamples=300)


def test_caller_supplied_plans():
    P = 6
    fn = _model("sigmoid", "tanh", P)
    bg, X, _ = _problem(8, P, N=7, n=3)
    rng = np.random.default_rng(0)
    plans = []
    for i in range(3):
        Z = rng.integers(0, 2, size=(40, P)).astype(np.uint8)
        Z[0] = 0
        Z[1] = 1
        Z[2:2 + P] = np.eye(P, dtype=np.uint8)
        plans.append((Z, rng.uniform(0.1, 1.0, 40)))
    eng = _engine(fn, bg, "logit")
    got = eng.shap_values(X, l1_reg=False, nsamples=40, plans=plans)
    assert eng.last_path()["general"] == "mlp"
    _compare(got, _oracle(fn, bg, "logit"), X, lambda i: plans[i], PLAIN_TOL, nsamples=40)


@pytest.mark.parametrize("l1_reg", ["auto", "aic", "num_features(4)"])
def test_l1_selection(l1_reg):
    P = 14                                    # 'auto' selects: 2076 of 16382 coalitions evaluated
    fn = _model("sigmoid", "relu", P)
    bg, X, _ = _problem(31, P, N=5, n=3, constant_cols=(13,))
    eng = _engine(fn, bg, "logit")
    got = eng.shap_values(X, l1_reg=l1_reg)
    path = eng.last_path()
    assert path["general"] in ("mlp", "simt", "none") and path["general_l1"] == 1, path
    _compare(got, _oracle(fn, bg, "logit"), X, _own_plans(eng, X), L1_TOL, l1_reg=l1_reg)


def test_identity_mlp_matches_the_linear_route():
    """An identity-activation MLP is the linear model W_0 W_1 .. W_L: the same phi on the linear route's identity head,
    without scikit-learn."""
    from distributedkernelshap_b200.predictors import LinearModelSpec
    P = 10
    spec = _hand_spec([P, 13, 9, 2], act="identity", head="identity", seed=5)
    W = spec.coefs[0]
    b = spec.intercepts[0]
    for Wl, bl in zip(spec.coefs[1:], spec.intercepts[1:]):
        b = b @ Wl + bl
        W = W @ Wl
    lin = LinearModelSpec(W.T, b, "identity")
    bg, X, _ = _problem(6, P, N=8, n=5, constant_cols=(3,))
    eng = _engine(spec, bg, "identity")
    got = eng.shap_values(X, l1_reg=False, nsamples=200)
    assert eng.last_path()["general"] == "mlp"
    ref = _engine(lin, bg, "identity")
    want = ref.shap_values(X, l1_reg=False, nsamples=200)
    for c in range(2):
        for i in range(X.shape[0]):
            assert rel_err(got[c][i], want[c][i]) < PLAIN_TOL


def test_grid_stride_batches_are_bit_identical_to_each_instance_alone():
    P = 5
    fn = _model("softmax", "logistic", P)
    rng = np.random.default_rng(9)
    bg = rng.normal(size=(6, P))
    n = 132 * 8 * 3 + 17                      # more than three instances per CTA at the kernel's largest grid
    X = rng.normal(size=(n, P))
    X[::3, 4] = bg[0, 4]                      # mixed M between real instances
    bg[:, 4] = bg[0, 4]
    eng = _engine(fn, bg, "identity")
    got = np.stack(eng.shap_values(X, l1_reg=False, nsamples=60))
    assert eng.last_path()["general"] == "mlp"
    for i in (0, 1, 2, 500, n - 1):
        alone = np.stack(eng.shap_values(X[i:i + 1], l1_reg=False, nsamples=60))
        np.testing.assert_array_equal(got[:, i], alone[:, 0])


def test_coalition_count_not_a_multiple_of_the_tile():
    P = 7
    fn = _model("identity", "relu", P)
    bg, X, _ = _problem(13, P, N=5, n=3)
    eng = _engine(fn, bg, "identity")
    got = eng.shap_values(X, l1_reg=False, nsamples=37)     # 37 rows: two full 16-row tiles and a tail of 5
    assert eng.last_path()["general"] == "mlp"
    _compare(got, _oracle(fn, bg, "identity"), X, _own_plans(eng, X, 37), PLAIN_TOL, nsamples=37)


def _mlp_smem_bytes(S, C, G, pads, nbuf, nw):
    """explain_mlp_kernel's layout (dks_mlp.cuh, smem_bytes): sums, then Delta_j, B[j] and nw warps' buffers (or the
    solve), then the varying groups."""
    pad16 = (G + 15) // 16 * 16
    hmax = max(pads)
    loop = pad16 * pads[0] + pads[0] + nw * 16 * (nbuf * hmax + 8)
    return 8 * (((C * S + 1) // 2 * 2) + max(loop, 63 * 63 + 64)) + 4 * 64


def test_shared_memory_limit():
    import torch
    from distributedkernelshap_b200._cabi import DksError
    P, R = 13, 8
    limit = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    S = 2
    while _mlp_smem_bytes(S + 1, R, P, [256], 1, 1) <= limit:
        S += 1
    assert S + 1 < 2 ** P - 2
    spec = _hand_spec([P, 256, R], act="relu", head="identity", seed=1)
    bg, X, _ = _problem(7, P, N=3, n=2)
    eng = _engine(spec, bg, "identity")
    got = eng.shap_values(X, l1_reg=False, nsamples=S)
    assert eng.last_path()["general"] == "mlp"
    _compare(got, _oracle(spec, bg, "identity"), X, _own_plans(eng, X, S), PLAIN_TOL, nsamples=S)
    with pytest.raises(DksError, match="shared memory"):
        _engine(spec, bg, "identity").shap_values(X, l1_reg=False, nsamples=S + 1)


def test_saturated_logistic_output_under_the_logit_link():
    """f(x) and the background stay finite, but coalitions that take x's first column and not its second saturate the
    logistic output to 1.0: their logit is not finite, DKS_ERR_NUMERIC, and nothing non-finite is written."""
    import torch
    from distributedkernelshap_b200 import _cabi
    P = 4
    coefs = [np.eye(P)[:, :2].copy(), np.array([[100.0], [-100.0]])]
    spec = MlpSpec(coefs, [np.zeros(2), np.zeros(1)], "identity", "sigmoid", P)
    rng = np.random.default_rng(0)
    bg = rng.uniform(-0.05, 0.05, size=(6, P))
    X = rng.uniform(-0.05, 0.05, size=(3, P))
    X[1, :2] = 50.0                                           # z(x) = 0, z with column 0 alone = 5000
    eng = _engine(spec, bg, "logit")
    with pytest.raises(_cabi.DksError) as e:
        eng.shap_values(X, l1_reg=False)
    assert e.value.code == _cabi.DKS_ERR_NUMERIC
    X_dev = torch.from_numpy(X).cuda()
    phi = torch.zeros((2, 3, P), dtype=torch.float64, device="cuda")
    eng.explain_device(X_dev.data_ptr(), 3, phi.data_ptr())
    torch.cuda.synchronize()
    assert torch.isfinite(phi).all() and not phi[:, 1].any()


def test_all_dead_relu_network_gives_zero():
    P = 6
    rng = np.random.default_rng(4)
    coefs = [rng.normal(size=(P, 12)) * 0.01, rng.normal(size=(12, 1))]
    spec = MlpSpec(coefs, [np.full(12, -50.0), np.array([0.3])], "relu", "sigmoid", P)
    bg, X, _ = _problem(9, P, N=6, n=3)
    eng = _engine(spec, bg, "logit")
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "mlp"
    for ph in _as_list(got):
        np.testing.assert_array_equal(ph, 0.0)


def test_graph_replay_is_bit_identical_to_the_host_path():
    import torch
    P = 8
    fn = _model("identity", "tanh", P, hidden=(20, 11))
    bg, X, _ = _problem(41, P, N=10, n=16, constant_cols=(7,))
    eng = _engine(fn, bg, "identity")
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
        assert eng.last_path()["general"] == "mlp"
        np.testing.assert_array_equal(phi.cpu().numpy(), want)
    eng.set_stream(0)


def _adult():
    from distributedkernelshap_b200.datasets import adult_like
    d = adult_like(n_explain=20, n_background=40, seed=0)
    X_all = np.concatenate([d["background"], d["X_explain"]])
    y = d["predictor"].predict(X_all)
    return d, X_all, y


def _kernel_shap(fn, d, link):
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    ks = KernelShap(fn, link=link, feature_names=d["group_names"], seed=0)
    ks.fit(d["background"], group_names=d["group_names"], groups=d["groups"])
    exp = ks.explain(d["X_explain"][:5], silent=True)          # default kwargs: nsamples='auto', l1_reg='auto'
    assert ks._explainer.last_path()["general"] in ("mlp", "none")
    return exp


def test_kernel_shap_on_the_default_scaled_mlp_classifier_with_the_logit_link():
    from distributedkernelshap_b200.data import convert_to_link
    d, X_all, y = _adult()
    clf = _sk(MLPClassifier(max_iter=50, random_state=0), X_all, y)
    exp = _kernel_shap(clf.predict_proba, d, "logit")
    fx = convert_to_link("logit").f(clf.predict_proba(d["X_explain"][:5]))
    for c in range(2):
        np.testing.assert_allclose(exp.shap_values[c].sum(1), fx[:, c] - exp.expected_value[c], rtol=1e-8, atol=1e-8)


def test_kernel_shap_on_a_three_class_mlp_classifier():
    d, X_all, y = _adult()
    y3 = y + (X_all[:, 0] > np.median(X_all[:, 0])).astype(int)
    clf = _sk(MLPClassifier(hidden_layer_sizes=(16,), max_iter=50, random_state=0), X_all, y3)
    exp = _kernel_shap(clf.predict_proba, d, "identity")
    fx = clf.predict_proba(d["X_explain"][:5])
    for c in range(3):
        np.testing.assert_allclose(exp.shap_values[c].sum(1), fx[:, c] - exp.expected_value[c], rtol=1e-8, atol=1e-8)


def test_kernel_shap_on_an_mlp_regressor():
    d, X_all, y = _adult()
    reg = _sk(MLPRegressor(hidden_layer_sizes=(32,), max_iter=50, random_state=0), X_all, y + 0.1 * X_all[:, 0])
    exp = _kernel_shap(reg.predict, d, "identity")
    fx = reg.predict(d["X_explain"][:5])
    np.testing.assert_allclose(np.asarray(exp.shap_values[0]).sum(1), fx - exp.expected_value[0], rtol=1e-8, atol=1e-8)


def test_refusals():
    from distributedkernelshap_b200._cabi import DksError
    P = 5
    fn = _model("sigmoid", "relu", P)
    bg, X, _ = _problem(2, P, N=6, n=2)
    for kernel in ("tcgen05", "shared"):
        eng = _engine(fn, bg, "identity", kernel=kernel)
        with pytest.raises(DksError, match="MLP kernel"):
            eng.shap_values(X, l1_reg=False)
    X65, s65, _ = _fit_data(0, 65)
    wide = _sk(MLPRegressor(hidden_layer_sizes=(4,), max_iter=5, random_state=0), X65, s65, None)
    with pytest.raises(NotImplementedError, match="64"):
        _engine(wide.predict, X65[:4], "identity")
    eng = _engine(fn, bg, "identity")
    Xn = X.copy()
    Xn[1, 2] = np.nan
    with pytest.raises(ValueError, match="instance 1"):
        eng.shap_values(Xn, l1_reg=False)
    bgi = bg.copy()
    bgi[3, 0] = np.inf
    with pytest.raises(ValueError, match="background row 3"):
        _engine(fn, bgi, "identity")
