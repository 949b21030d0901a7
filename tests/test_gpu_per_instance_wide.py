"""Per-instance coalition plans of 65..128 groups drawn on the device (two-word rows, plan_mode='per_instance').

The device plans must equal, bit for bit, what upstream's sequential loop builds from the same Philox stream
(tests/sampler_twin.py + oracle.build_plan); phi must match the oracle / the float64 linear reference fed those plans;
results must not depend on how the rows are split into calls; and what the two-word path does not cover is refused."""
import numpy as np
import pytest

from conftest import elementwise_excess, make_problem, rel_err
from linear_reference import LinearReference
from sampler_twin import PhiloxPlanStream
from test_gpu_parity import _engine, _oracle

pytestmark = pytest.mark.gpu

TOL = 1e-5
ATOL_ELEM = 5e-7


def _expected_plan(M, nsamples, seed, row):
    from oracle.shap_kernel_oracle import build_plan
    from distributedkernelshap_b200.plan import pack_dense_plan, resolve_nsamples
    S, _ = resolve_nsamples(M, nsamples)
    Z, w, _ = build_plan(M, S, rng=PhiloxPlanStream(seed, row))
    return pack_dense_plan(Z), w, Z


def _dense(zb, M):
    """[S, 2] words -> [S, M] 0/1."""
    k = np.arange(M)
    return ((zb[:, k // 64] >> (k % 64).astype(np.uint64)) & np.uint64(1)).astype(np.uint8)


def _scaled_problem(M, n, N, seed, weights=False):
    """make_problem with coefficients scaled for M columns (the logit link must not saturate)."""
    prob = make_problem(seed=seed, n=n, N=N, widths=(1,) * M, weights=weights)
    prob["clf"].coef_ *= 2.0 / np.sqrt(M)
    return prob


@pytest.mark.parametrize("M,nsamples", [(65, 300), (80, 1000), (100, "auto"), (127, 2000), (128, 4096)])
def test_device_plans_equal_the_sequential_loop_on_the_same_stream(M, nsamples):
    prob = _scaled_problem(M, n=3, N=8, seed=40 + M)
    eng = _engine(prob, seed=123, plan_mode="per_instance")
    got = eng.shap_values(prob["X"], nsamples=nsamples, l1_reg=False)
    assert eng.last_path()["general"] == "simt_wide"
    zb, w = eng.instance_plans()
    assert zb.shape[0] == 3 and zb.ndim == 3 and zb.shape[2] == 2
    Ms, _ = eng.varying(prob["X"])
    assert np.all(Ms == M)
    repeats = 0
    for i in range(3):
        want_z, want_w, Z = _expected_plan(M, nsamples, 123, i)
        S = len(want_w)
        np.testing.assert_array_equal(zb[i, :S], want_z, err_msg=f"instance {i}")
        np.testing.assert_allclose(w[i, :S], want_w, rtol=1e-13, atol=0)
        assert np.all(w[i, S:] == 0) and np.all(zb[i, S:] == 0)
        repeats += len(np.unique(w[i, 2 * M:S])) > 1          # some sampled mask was drawn more than once
        if i == 0 and M <= 100:
            orc = _oracle(prob)
            phi = orc.explain(prob["X"][:1], plan=(Z, want_w), nsamples=nsamples, l1_reg=False)
            for c in range(2):
                assert rel_err(got[c][0], phi[:, c]) < TOL
    if M == 65:
        assert repeats > 0                                     # small budget: size-2 draws repeat


def _cfg4(n, link, weights=False, predict="predict_proba"):
    from distributedkernelshap_b200 import datasets
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    d = datasets.dense_tabular(n=n, n_features=128, n_background=512, seed=4)
    w = np.random.default_rng(1).uniform(0.2, 1.0, 512) if weights else None
    args = (d["groups"],) + ((w,) if w is not None else ())
    dd = DenseData(d["background"], d["group_names"], *args)
    clf = d["predictor"]
    eng = GpuKernelExplainer(getattr(clf, predict), dd, link=link, seed=11, plan_mode="per_instance")
    head = "logistic" if predict == "predict_proba" else "identity"
    ref = LinearReference(clf.coef_, clf.intercept_, d["background"], d["groups"], w, head=head, link=link)
    return d, eng, ref


@pytest.mark.parametrize("link,weights,predict", [("logit", False, "predict_proba"), ("identity", False, "predict_proba"),
                                                   ("logit", True, "predict_proba"),
                                                   ("identity", True, "decision_function")])
def test_configs4_shape_matches_linear_reference(link, weights, predict):
    """configs[4] (M = 128, N = 512, S = 4096), 64 instances: phi from the device-drawn plans against the float64
    reference fed the same plans, under the baseline tests' max-norm and element-wise criteria."""
    d, eng, ref = _cfg4(64, link, weights, predict)
    got = eng.shap_values(d["X_explain"], nsamples=4096, l1_reg=False)
    got = got if isinstance(got, list) else [got]
    zb, w = eng.instance_plans()
    want = np.zeros((64, 128, ref.C))
    for i in range(64):
        want[i] = ref.explain(d["X_explain"][i], plan=(_dense(zb[i, :4096], 128), w[i, :4096]))
    worst = max(rel_err(got[c], want[:, :, c]) for c in range(ref.C))
    frac, mx = elementwise_excess(np.stack(got, axis=-1), want, rtol=TOL, atol=ATOL_ELEM)
    print(f"[cfg4 per-instance {link} w={weights} {predict}] max-norm {worst:.2e}, element-wise worst ratio {mx:.3f}")
    assert worst < TOL and frac == 0.0, (worst, frac, mx)
    if predict == "decision_function":
        # identity head: phi is exact for any plan -- XW - Bbar
        coef = np.asarray(d["predictor"].coef_).reshape(-1)
        ww = ref.weights
        exact = d["X_explain"] * coef[None, :] - (ww @ d["background"]) * coef[None, :]
        if link == "identity":
            np.testing.assert_allclose(got[0], exact, rtol=1e-9, atol=1e-9)


def test_results_do_not_depend_on_call_splits_or_entry_point(monkeypatch):
    import torch
    from distributedkernelshap_b200 import engine as engmod
    prob = _scaled_problem(70, n=24, N=16, seed=5)
    eng = _engine(prob, seed=3, plan_mode="per_instance")
    full = eng.shap_values(prob["X"], nsamples=600, l1_reg=False)
    part = eng.shap_values(prob["X"][7:19], nsamples=600, l1_reg=False, row_offset=7)
    for c in range(2):
        np.testing.assert_array_equal(part[c], full[c][7:19])
    monkeypatch.setattr(engmod, "MAX_ROWS_PER_CALL_WIDE_PER_INSTANCE", 5)      # five calls of <= 5 rows
    blocks = eng.shap_values(prob["X"], nsamples=600, l1_reg=False)
    for c in range(2):
        np.testing.assert_array_equal(blocks[c], full[c])
    # device-resident entry on a user stream: the second identical call is captured, later ones replay the graph
    stream = torch.cuda.Stream()
    out = []
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        eng.lib.dks_set_row_offset(eng._ctx, 0)
        X = torch.from_numpy(prob["X"]).cuda()
        phi = torch.zeros((2, 24, 70), dtype=torch.float64, device="cuda")
        for _ in range(4):
            phi.zero_()
            eng.explain_device(X.data_ptr(), 24, phi.data_ptr(), nsamples=600)
            eng.check_status()
            out.append(phi.cpu().numpy())
            assert eng.last_path()["general"] == "simt_wide"
        assert eng.graph_launches() >= 2
    eng.set_stream(0)
    for o in out:
        for c in range(2):
            np.testing.assert_array_equal(o[c], full[c])


def test_out_of_scope_cases_are_refused():
    from distributedkernelshap_b200._cabi import DksError
    prob = _scaled_problem(80, n=4, N=8, seed=6)
    refused = (NotImplementedError, DksError)
    # caller-supplied plans
    eng = _engine(prob, seed=1, plan_mode="per_instance")
    Z, w = np.ones((10, 80), dtype=np.uint8), np.full(10, 0.1)
    with pytest.raises(refused):
        eng.shap_values(prob["X"], nsamples=400, l1_reg=False, plans=[(Z, w)] * 4)
    # l1 selection on per-instance plans
    with pytest.raises(refused):
        eng.shap_values(prob["X"], nsamples=400, l1_reg="aic")
    # tensor-core / shared kernel
    for kernel in ("tcgen05", "shared"):
        e = _engine(prob, seed=1, plan_mode="per_instance", kernel=kernel)
        with pytest.raises(refused) as ei:
            e.shap_values(prob["X"], nsamples=400, l1_reg=False)
        assert not isinstance(ei.value, DksError) or ei.value.code == 3
    # a partial varying set
    part = dict(prob)
    part["X"] = prob["X"].copy()
    part["X"][:, 5] = part["bg"][0, 5]
    part["bg"] = prob["bg"].copy()
    part["bg"][:, 5] = part["bg"][0, 5]
    e = _engine(part, seed=1, plan_mode="per_instance")
    with pytest.raises(refused):
        e.shap_values(part["X"], nsamples=400, l1_reg=False)
    # softmax and one-vs-rest heads
    from distributedkernelshap_b200.predictors import LinearSoftmaxClassifier
    rng = np.random.default_rng(0)
    for mc in ("multinomial", "ovr"):
        p3 = dict(prob)
        p3["clf"] = LinearSoftmaxClassifier(rng.normal(0, 0.1, (3, 80)), rng.normal(0, 0.1, 3), multi_class=mc)
        e = _engine(p3, seed=1, plan_mode="per_instance")
        with pytest.raises(refused):
            e.shap_values(prob["X"], nsamples=400, l1_reg=False)
    # more than 128 groups
    wide = _scaled_problem(129, n=2, N=8, seed=7)
    e = _engine(wide, seed=1, plan_mode="per_instance")
    with pytest.raises(refused):
        e.shap_values(wide["X"], nsamples=600, l1_reg=False)
