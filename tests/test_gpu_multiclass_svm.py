"""Multi-class SVMs on the kernel-machine route (the one-vs-one head, ``last_path()['general'] == 'kmach'``) against the
oracle fed the independent reference model (tests/multiclass_svm_reference.py) and the coalition plans the engine used:
pair values and calibrated probabilities over 3 to 8 classes, both links, every plan source, weighted backgrounds, l1
selection, the kernel's chunk and tile edges, the vote's tie rule, the uniform fallback, the shared-memory limit, bit
identity across batches and graph replay, refusals, the public API, ensembles and an encoded pipeline.

Every problem asserts that min |dec| over the masked rows the oracle evaluates exceeds 1e-9, so a vote cannot flip on a
rounding difference between the device's and the reference's order of summation."""
import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")
from sklearn.calibration import CalibratedClassifierCV  # noqa: E402
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.ensemble import RandomForestClassifier, StackingClassifier, VotingClassifier  # noqa: E402
from sklearn.linear_model import LogisticRegression  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import MinMaxScaler, OneHotEncoder, StandardScaler  # noqa: E402
from sklearn.svm import SVC, NuSVC  # noqa: E402

from distributedkernelshap_b200.kernel_machines import MulticlassSvmSpec, extract_kernel_machine_spec  # noqa: E402
from multiclass_svm_reference import outputs, pair_values  # noqa: E402

PLAIN_TOL = 1e-9
L1_TOL = 1e-5
DEC_MARGIN = 1e-9


def _fit_data(seed, P, classes, n=150):
    """Labels drawn from a softmax of a seeded random linear score (every class present)."""
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    Z = (X - X.mean(0)) / X.std(0) @ rng.normal(size=(P, classes)) * 2.0
    pr = np.exp(Z - Z.max(1, keepdims=True))
    pr /= pr.sum(1, keepdims=True)
    y = np.array([rng.choice(classes, p=p) for p in pr])
    y[:classes] = np.arange(classes)
    return X, y, rng


def _model(kind, kernel, P, classes, seed=0):
    """(spec, sklearn method): 'ovo' pair values, 'cal1' / 'cal3' calibrated probabilities (ensemble False / True)."""
    X, y, _ = _fit_data(seed, P, classes)
    kw = {"gamma": 0.05} if kernel == "sigmoid" else {}
    if kind == "ovo":
        fn = make_pipeline(StandardScaler(), SVC(kernel=kernel, decision_function_shape="ovo", **kw)).fit(X, y)
        fn = fn.decision_function
    elif kind == "cal1":
        fn = CalibratedClassifierCV(make_pipeline(StandardScaler(), SVC(kernel=kernel, **kw)), ensemble=False,
                                    cv=3).fit(X, y).predict_proba
    else:
        fn = make_pipeline(MinMaxScaler(), CalibratedClassifierCV(
            make_pipeline(StandardScaler(), NuSVC(kernel=kernel, nu=0.05, **kw)), ensemble=True, cv=3)).fit(X, y)
        fn = fn.predict_proba
    spec = extract_kernel_machine_spec(fn)
    assert isinstance(spec, MulticlassSvmSpec)
    return spec, fn


class _Ref:
    """The reference model, recording min |dec| over every row it evaluates (the masked rows of the oracle)."""

    def __init__(self, spec, skip_pairs=()):
        self.spec = spec
        self.keep = [k for k in range(spec.P) if k not in skip_pairs]
        self.min_dec = np.inf

    def __call__(self, Z):
        Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
        self.min_dec = min(self.min_dec, float(np.abs(pair_values(self.spec, Z)[:, :, self.keep]).min()))
        return outputs(self.spec, Z)


def _problem(seed, P, N, n, constant_cols=(), weights=False, zero_row=False):
    rng = np.random.default_rng(seed + 1000)
    bg = rng.normal(size=(N, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 2.0, P) + np.linspace(-1.0, 2.0, P)
    for c in constant_cols:
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
        assert want.shape[1] == len(got)
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


def _run(spec, bg, X, link, tol=PLAIN_TOL, w=None, nsamples="auto", skip_pairs=(), **kw):
    ref = _Ref(spec, skip_pairs)
    eng = _engine(spec, bg, link, w=w, **kw)
    got = eng.shap_values(X, l1_reg=False, nsamples=nsamples)
    assert eng.last_path()["general"] == "kmach"
    worst = _compare(got, _oracle(ref, bg, link, w=w), X, _own_plans(eng, X, nsamples), tol, nsamples=nsamples)
    assert ref.min_dec > DEC_MARGIN, ref.min_dec
    _check_additivity(eng, ref, got, X, link)
    return eng, got, worst


CASES = ([("ovo", kernel, k, "identity") for k in (3, 4) for kernel in ("rbf", "poly", "sigmoid")] +
         [(kind, kernel, k, link) for kind in ("cal1", "cal3") for k in (3, 5, 8) for kernel in ("rbf", "poly", "sigmoid")
          for link in ("identity", "logit")])


@pytest.mark.parametrize("kind,kernel,classes,link", CASES)
def test_parity_every_model_and_link(kind, kernel, classes, link):
    P = 7
    spec, _ = _model(kind, kernel, P, classes)
    bg, X, _ = _problem(11, P, N=10, n=4, constant_cols=(6,))
    eng, got, worst = _run(spec, bg, X, link)
    M, _ = eng.varying(X)
    assert {int(m) for m in M} == {6, 7}                    # full and partial varying sets in one call
    assert len(_as_list(got)) == spec.n_outputs
    print(f"{kind} {kernel} K={classes} {link}: max|d|/max|phi| = {worst:.2e}")


def test_weighted_background_with_a_zero_weight_row():
    P = 6
    spec, _ = _model("cal3", "rbf", P, 5)
    bg, X, w = _problem(3, P, N=10, n=3, weights=True, zero_row=True)
    _run(spec, bg, X, "logit", w=w)


def test_per_instance_device_plans():
    P = 9
    spec, _ = _model("cal1", "rbf", P, 4)
    bg, X, _ = _problem(21, P, N=6, n=4, constant_cols=(8,))
    ref = _Ref(spec)
    eng = _engine(spec, bg, "logit", plan_mode="per_instance")
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
    _compare(got, _oracle(ref, bg, "logit"), X, plans, PLAIN_TOL, nsamples=300)
    assert ref.min_dec > DEC_MARGIN


def test_caller_supplied_plans():
    P = 6
    spec, _ = _model("ovo", "poly", P, 4)
    bg, X, _ = _problem(8, P, N=7, n=3)
    rng = np.random.default_rng(0)
    plans = []
    for i in range(3):
        Z = rng.integers(0, 2, size=(40, P)).astype(np.uint8)
        Z[0] = 0
        Z[1] = 1
        Z[2:2 + P] = np.eye(P, dtype=np.uint8)
        plans.append((Z, rng.uniform(0.1, 1.0, 40)))
    ref = _Ref(spec)
    eng = _engine(spec, bg, "identity")
    got = eng.shap_values(X, l1_reg=False, nsamples=40, plans=plans)
    assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(ref, bg, "identity"), X, lambda i: plans[i], PLAIN_TOL, nsamples=40)
    assert ref.min_dec > DEC_MARGIN


@pytest.mark.parametrize("l1_reg", ["auto", "aic", "bic", "num_features(4)"])
def test_l1_selection(l1_reg):
    P = 14                                    # 'auto' selects
    spec, _ = _model("cal1", "rbf", P, 3)
    bg, X, _ = _problem(31, P, N=4, n=2, constant_cols=(13,))
    ref = _Ref(spec)
    eng = _engine(spec, bg, "logit")
    got = eng.shap_values(X, l1_reg=l1_reg)
    path = eng.last_path()
    assert path["general"] in ("kmach", "simt", "none") and path["general_l1"] == 1, path
    _compare(got, _oracle(ref, bg, "logit"), X, _own_plans(eng, X), L1_TOL, l1_reg=l1_reg)
    assert ref.min_dec > DEC_MARGIN


@pytest.mark.parametrize("nsamples", [100, 256, 257, 300, 700])
def test_coalition_chunk_edges(nsamples):
    """coalitions go in chunks of the block (256): S below, at, one past and between multiples of it"""
    P = 12
    spec, _ = _model("cal1", "rbf", P, 5)
    bg, X, _ = _problem(12, P, N=4, n=2)
    _run(spec, bg, X, "logit", nsamples=nsamples)


def _hand_spec(blocks, P, head="ovo_proba", seed=0, members=1, zero_pair=False, cal_b=None):
    """A hand-built one-member (or more) spec whose class c owns blocks[c] support vectors."""
    rng = np.random.default_rng(seed)
    nc = len(blocks)
    n_m = int(sum(blocks))
    sv_off = np.arange(members + 1) * n_m
    cls_off = np.stack([m * n_m + np.concatenate([[0], np.cumsum(blocks)]) for m in range(members)])
    dual = rng.normal(size=(n_m * members, nc - 1))
    P_ = nc * (nc - 1) // 2
    icpt = rng.normal(size=(members, P_)) * 0.3
    if zero_pair:                              # pair (0, 1): class 0's row 0 and class 1's row 0 are zero, no intercept
        for m in range(members):
            dual[cls_off[m, 0]:cls_off[m, 1], 0] = 0.0
            dual[cls_off[m, 1]:cls_off[m, 2], 0] = 0.0
        icpt[:, 0] = 0.0
    cal_a = -rng.uniform(0.5, 2.0, (members, nc))
    cb = rng.normal(size=(members, nc)) if cal_b is None else np.full((members, nc), cal_b)
    return MulticlassSvmSpec(rng.normal(size=(n_m * members, P)), sv_off, cls_off, dual, icpt,
                             rng.uniform(0.5, 2.0, (members, P)), rng.normal(size=(members, P)) * 0.1,
                             [0.3] * members, "rbf", 3, 0.5, head, P, nc, cal_a=cal_a, cal_b=cb)


@pytest.mark.parametrize("blocks", [(1, 31, 32, 33), (33, 0, 5), (32, 1, 64), (0, 31, 2)])
def test_class_blocks_around_the_tile(blocks):
    P = 6
    spec = _hand_spec(blocks, P, seed=sum(blocks))
    bg, X, _ = _problem(4, P, N=5, n=3, constant_cols=(5,))
    _run(spec, bg, X, "logit")
    spec = _hand_spec(blocks, P, head="ovo", seed=sum(blocks)) if len(blocks) <= 4 else None
    if spec is not None:
        _run(spec, bg, X, "identity")


def test_tie_goes_to_the_first_class():
    """dec of pair (0, 1) is exactly 0 on every row: its vote goes to class 0, as libsvm decides it"""
    P = 5
    spec = _hand_spec((7, 9, 6), P, seed=3, zero_pair=True)
    bg, X, _ = _problem(5, P, N=5, n=3)

    assert np.all(pair_values(spec, np.r_[bg, X])[:, :, 0] == 0.0)
    _run(spec, bg, X, "logit", skip_pairs=(0,))
    _run(spec, bg, X, "identity", skip_pairs=(0,))


def test_uniform_fallback_when_every_calibrated_class_underflows():
    P = 5
    spec = _hand_spec((8, 8, 8, 8), P, seed=4, cal_b=2000.0)   # expit(-(a f + b)) == 0 for every class
    bg, X, _ = _problem(6, P, N=4, n=2)
    np.testing.assert_array_equal(outputs(spec, X), np.full((2, 4), 0.25))
    eng, got, _ = _run(spec, bg, X, "identity")
    np.testing.assert_array_equal(np.stack(_as_list(got)), 0.0)


def _ovo_smem_bytes(C, S, R, G):
    tile = 32 * (1 + R + G + 16 * ((G + 3) // 4))          # explain_kmach_ovo_kernel's layout (dks_kmach.cuh)
    return 8 * (C * S + max(tile, 63 * 63 + 64)) + 4 * 64


def test_shared_memory_limit_at_eight_classes():
    import torch
    from distributedkernelshap_b200._cabi import DksError
    P, nc = 13, 8
    limit = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    S = ((limit - 4 * 64) // 8 - max(32 * (1 + nc - 1 + P + 16 * 4), 63 * 63 + 64)) // nc
    assert _ovo_smem_bytes(nc, S, nc - 1, P) <= limit < _ovo_smem_bytes(nc, S + 1, nc - 1, P) and S + 1 < 2 ** P - 2
    spec = _hand_spec((3, 2, 4, 1, 2, 3, 2, 3), P, seed=8)
    bg, X, _ = _problem(7, P, N=2, n=1)
    _run(spec, bg, X, "identity", nsamples=S)
    with pytest.raises(DksError, match="shared memory"):
        _engine(spec, bg, "identity").shap_values(X, l1_reg=False, nsamples=S + 1)


def test_grid_stride_batches_are_bit_identical_to_each_instance_alone():
    P = 5
    spec, _ = _model("cal3", "rbf", P, 4)
    rng = np.random.default_rng(9)
    bg = rng.normal(size=(4, P))
    n = 132 * 8 * 2 + 17
    X = rng.normal(size=(n, P))
    X[::3, 4] = bg[0, 4]
    bg[:, 4] = bg[0, 4]
    eng = _engine(spec, bg, "logit")
    got = np.stack(eng.shap_values(X, l1_reg=False, nsamples=60))
    assert eng.last_path()["general"] == "kmach"
    for i in (0, 1, 2, 500, n - 1):
        alone = np.stack(eng.shap_values(X[i:i + 1], l1_reg=False, nsamples=60))
        np.testing.assert_array_equal(got[:, i], alone[:, 0])


def test_graph_replay_is_bit_identical_to_the_host_path():
    import torch
    P = 8
    spec, _ = _model("cal1", "rbf", P, 5)
    bg, X, _ = _problem(41, P, N=6, n=16, constant_cols=(7,))
    eng = _engine(spec, bg, "logit")
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


def test_nan_refusals():
    P = 5
    spec, _ = _model("cal1", "rbf", P, 3)
    bg, X, _ = _problem(2, P, N=6, n=2)
    eng = _engine(spec, bg, "logit")
    Xn = X.copy()
    Xn[1, 2] = np.nan
    with pytest.raises(ValueError, match="instance 1"):
        eng.shap_values(Xn, l1_reg=False)
    bgn = bg.copy()
    bgn[3, 0] = np.nan
    with pytest.raises(ValueError, match="background row 3"):
        _engine(spec, bgn, "logit")


def test_kernel_shap_on_a_scaled_calibrated_svc_with_default_kwargs():
    from distributedkernelshap_b200.data import convert_to_link
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    P = 8
    X, y, _ = _fit_data(5, P, 4, n=200)
    model = make_pipeline(StandardScaler(), CalibratedClassifierCV(SVC(), ensemble=False)).fit(X, y)
    ks = KernelShap(model.predict_proba, link="logit", seed=0)
    ks.fit(X[:20])
    exp = ks.explain(X[150:154], silent=True)
    assert ks._explainer.last_path()["general"] == "kmach"
    fx = convert_to_link("logit").f(model.predict_proba(X[150:154]))
    for c in range(4):
        np.testing.assert_allclose(exp.shap_values[c].sum(1), fx[:, c] - exp.expected_value[c], rtol=1e-8, atol=1e-8)


@pytest.mark.parametrize("kind", ["voting", "stacking"])
def test_calibrated_multiclass_svc_as_an_ensemble_member(kind):
    P = 6
    X, y, _ = _fit_data(7, P, 3, n=150)
    cal = CalibratedClassifierCV(make_pipeline(StandardScaler(), SVC()), ensemble=False, cv=3)
    members = [("svc", cal), ("rf", RandomForestClassifier(5, max_depth=3, random_state=0)),
               ("lr", LogisticRegression(max_iter=500))]
    if kind == "voting":
        ens = VotingClassifier(members, voting="soft", weights=[2.0, 1.0, 0.5]).fit(X, y)
    else:
        ens = StackingClassifier(members[:2], final_estimator=LogisticRegression(max_iter=500), cv=3).fit(X, y)
    bg, X2, _ = _problem(15, P, N=6, n=3, constant_cols=(5,))
    eng = _engine(ens.predict_proba, bg, "identity")
    got = eng.shap_values(X2, l1_reg=False)
    assert eng.last_path()["general"] == ("ensemble" if kind == "voting" else "stacking")
    _compare(got, _oracle(ens.predict_proba, bg, "identity"), X2, _own_plans(eng, X2), PLAIN_TOL)
    _check_additivity(eng, ens.predict_proba, got, X2, "identity")


def test_encoded_pipeline_in_front_of_the_calibrator():
    rng = np.random.default_rng(6)
    n = 150
    Xr = np.c_[rng.normal(size=(n, 3)), rng.integers(0, 3, size=n).astype(np.float64)]
    s = Xr[:, 0] + np.where(Xr[:, 3] == 1, 1.0, -0.5) + 0.3 * Xr[:, 1]
    y = np.digitize(s, np.quantile(s, [0.33, 0.66]))
    ct = ColumnTransformer([("num", StandardScaler(), [0, 1, 2]), ("cat", OneHotEncoder(), [3])])
    pipe = make_pipeline(ct, CalibratedClassifierCV(SVC(), ensemble=False, cv=3)).fit(Xr, y)
    bg, X = Xr[:8].copy(), Xr[100:103].copy()
    eng = _engine(pipe.predict_proba, bg, "logit")
    got = eng.shap_values(X, l1_reg=False)
    assert eng.last_path()["general"] == "kmach"
    _compare(got, _oracle(pipe.predict_proba, bg, "logit"), X, _own_plans(eng, X), PLAIN_TOL)
    _check_additivity(eng, pipe.predict_proba, got, X, "logit")
