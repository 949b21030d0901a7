"""Weighted backgrounds (k-means centroids weighted by cluster size, user weights) on the shared-plan kernels: the weighted
instantiations of explain_shared_fused_kernel and explain_shared_smem_kernel (dks_shared.cuh, DESIGN.md 5.0.1), at the
shape edges where their code changes, against the float64 reference of tests/linear_reference.py fed the engine's own
plans -- with the criteria of test_gpu_kernel_paths.py, and every case asserting through ``last_path()`` that it ran the
path it targets with ``bg_weights == "weighted"``.

Weights look like k-means output: integer cluster counts spread over more than two decades, some cases with a weight of
exactly 0."""
import numpy as np
import pytest

from conftest import rel_err
from test_gpu_kernel_paths import FUSED_N, _check, _device, _engine, _expect, _pmat_fits, _problem, _run, _spad

pytestmark = pytest.mark.gpu


def _counts(seed, N, zero=False):
    """Integer cluster counts, max / min >= 100 (N >= 2), one of them 0 with ``zero`` (N >= 3)."""
    rng = np.random.default_rng(seed)
    w = np.round(np.exp(rng.uniform(0.0, np.log(500.0), size=N)))
    if N >= 2:
        w[rng.integers(N)] = 1.0
        w[(rng.integers(N - 1) + 1 + np.argmin(w)) % N] = 400.0
    if zero and N >= 3:
        w[np.argsort(w)[N // 2]] = 0.0
    return w


def _wproblem(seed, G, N, n, zero=False, **kw):
    prob = _problem(seed, G=G, N=N, n=n, **kw)
    prob["weights"] = _counts(seed + 1, N, zero)
    return prob


def _wrun(prob, nsamples, kernel="auto", **want):
    eng, got, path = _run(prob, nsamples, kernel=kernel)
    if kernel == "auto":
        _expect(path, bg_weights="weighted", **want)
    return eng, got, path


# ---- fused kernel --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", FUSED_N)
def test_weighted_fused_background_sizes(N):
    """N = 1: a single background row has uniform weights whatever its count, and takes the uniform kernel."""
    prob = _wproblem(3000 + N, G=13, N=N, n=6, zero=N >= 3)
    eng, got, path = _run(prob, 400)
    _expect(path, shared="fused", solve="fused", chunks=1, fused_NI=1, bg_weights="weighted" if N > 1 else "uniform")
    _check(eng, prob, got, 400, "weighted fused N")


@pytest.mark.parametrize("G", [2, 13, 14, 16])
@pytest.mark.parametrize("N", [17, 100, 128])
def test_weighted_fused_group_counts(G, N):
    prob = _wproblem(3100 + 7 * G + N, G=G, N=N, n=5)
    eng, got, _ = _wrun(prob, 300, shared="fused", solve="fused")
    _check(eng, prob, got, 300, "weighted fused G")


@pytest.mark.parametrize("N", [64, 100, 128])
def test_weighted_fused_layouts_and_warp_caps(N):
    """Few row groups: several warps share a slice (kw > 1); warp caps down to the one-warp-per-slice layout (kw = 1) give
    the same bits (fixed-point accumulation), and the default stays within the weighted register budget (20 warps)."""
    prob = _wproblem(3200 + N, G=12, N=N, n=70, zero=True)
    eng = _engine(prob)
    want = np.stack(eng.shap_values(prob["X"], nsamples=2048, l1_reg=False), axis=-1)
    base = eng.last_path()
    _expect(base, shared="fused", bg_weights="weighted")
    assert base["cta_warps"] > base["warps"] and base["cta_warps"] <= 20, base
    _check(eng, prob, want, 2048, "weighted fused layouts")
    for cap in (2, 4, 12, 16):
        eng.set_option("fused_warps", cap)
        got = np.stack(eng.shap_values(prob["X"], nsamples=2048, l1_reg=False), axis=-1)
        path = eng.last_path()
        _expect(path, shared="fused", bg_weights="weighted")
        assert path["cta_warps"] <= cap, path
        assert np.array_equal(got, want), (cap, path, np.abs(got - want).max())
    eng.set_option("fused_warps", 0)


def test_weighted_fused_instance_counts_around_the_batch():
    probe_prob = _wproblem(3300, G=13, N=64, n=1)
    probe = _engine(probe_prob)
    probe.shap_values(probe_prob["X"], nsamples=200, l1_reg=False)
    B = probe.last_path()["fused_B"]
    assert B in (8, 16, 32)
    for n in (1, B - 1, B, B + 1):
        prob = _wproblem(3300 + n, G=13, N=64, n=n, zero=True)
        eng, got, _ = _wrun(prob, 200, shared="fused", fused_B=B)
        _check(eng, prob, got, 200, "weighted fused n")


def test_weighted_fused_to_unfused_boundary():
    """The weighted slice is twice the uniform one, so fewer row groups fit a CTA: the boundary is derived from the
    warps the engine reports for the weighted kernel, S_pad / 32 == sm_count * warps is the last fused plan."""
    sm, smem = _device()
    probe_prob = _wproblem(3400, G=16, N=128, n=1)
    probe = _engine(probe_prob)
    probe.shap_values(probe_prob["X"], nsamples=100, l1_reg=False)
    p0 = probe.last_path()
    _expect(p0, shared="fused", bg_weights="weighted")
    S = 32 * sm * p0["warps"]
    assert S <= 2 ** 16 - 2
    prob = _wproblem(3401, G=16, N=128, n=p0["fused_B"] + 3, zero=True)
    eng, got, _ = _wrun(prob, S, shared="fused", warps=p0["warps"], grid=sm)
    _check(eng, prob, got, S, "weighted fused boundary")
    eng, got, path = _wrun(prob, S + 1, shared="smem",
                           solve="pmat" if _pmat_fits(16, _spad(S + 1), smem) else "wls_shared")
    assert path["grid"] * path["warps"] >= _spad(S + 1) // 32
    _check(eng, prob, got, S + 1, "weighted fused boundary")


# ---- unfused kernel ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("G,solve", [(17, "pmat"), (25, "pmat"), (26, "wls_shared"), (64, "wls_shared")])
def test_weighted_unfused_solves(G, solve):
    prob = _wproblem(3500 + G, G=G, N=45, n=5, zero=True)
    eng, got, _ = _wrun(prob, 300, shared="smem", chunks=1, solve=solve)
    _check(eng, prob, got, 300, "weighted unfused")


@pytest.mark.parametrize("N", [21, 128, 129, 200])
def test_weighted_unfused_background_chunks(N):
    """Chunks of 128 background columns: each uses its own columns' weights; one column past a chunk puts a single
    weighted column in the last launch.  N = 21 and 129 leave an odd number of quads in a chunk (a zero quad pads it)."""
    prob = _wproblem(3600 + N, G=20, N=N, n=4, zero=True)
    eng, got, path = _wrun(prob, 200, shared="smem")
    assert path["chunks"] == -(-N // 128), path
    _check(eng, prob, got, 200, "weighted unfused chunks")


@pytest.mark.parametrize("G", [70, 128])
@pytest.mark.parametrize("N", [17, 130])
def test_weighted_two_word_rows(G, N):
    prob = _wproblem(3700 + G + N, G=G, N=N, n=3, zero=True)
    eng, got, _ = _wrun(prob, 600, shared="smem", solve="wls_shared", chunks=-(-N // 128))
    _check(eng, prob, got, 600, "weighted two-word rows")


@pytest.mark.parametrize("G", [129, 200])
@pytest.mark.parametrize("N", [17, 128, 130, 300])
def test_weighted_sixteen_word_rows(G, N):
    """More than 128 groups: chunks of 128 columns, A(i, s) handed from the first chunk's launch to the others."""
    prob = _wproblem(3800 + G + N, G=G, N=N, n=3, zero=True)
    eng, got, _ = _wrun(prob, 600, shared="smem", solve="wide", chunks=-(-N // 128))
    _check(eng, prob, got, 600, "weighted sixteen-word rows")


# ---- saturated scores ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,which", [(64, "fused"), (129, "smem")])
def test_weighted_near_saturated_scores(N, which):
    prob = _wproblem(3900 + N, G=8, N=N, n=8, intercept=-14.0, coef_sd=0.45, zero=True)
    eng, got, _ = _wrun(prob, 200, shared=which)
    _check(eng, prob, got, 200, "weighted saturated")


def _at_the_clamp_threshold(seed, N, n):
    """Every coalition row at the packed path's limit: kappa * score near -41 for every background row, so that
    Dm = 2^0.4 for every entry and A(i, s) = 2^(59 + a) with a in [0.5, 0.76] for most rows (A up to 0.97e18, just under
    the clamped path's 1e18), and the weight concentrated on the pair of columns (0, 2): W2 = w'0 + w'2 close to N, so
    that A^2 Dm0 Dm2 W2 passes the fp32 range whenever N is above about 200."""
    from distributedkernelshap_b200.predictors import LinearSoftmaxClassifier
    rng = np.random.default_rng(seed)
    G, scale = 8, -2.0 * np.log2(np.e)
    coef = np.full((1, G), 0.5)
    b = 59.4 / scale                                     # scale * intercept = 59.4: the row exponent is 59, Dm = 2^0.4
    bg = rng.normal(0.0, 0.002, size=(N, G))
    X = (0.094 - rng.uniform(0.0, 0.004, size=(n, G))) / (scale * 0.5)   # scale * x_k * c_k in [0.090, 0.094]
    w = np.ones(N)
    w[0], w[2] = 20000.0, 5000.0
    clf = LinearSoftmaxClassifier(coef, np.array([b]), multi_class="multinomial")
    a_max = (scale * X * 0.5).sum(axis=1).max()
    assert 59 + a_max < np.log2(1.0e18)
    return dict(X=X, bg=bg, groups=[[k] for k in range(G)], clf=clf, weights=w, kappa=2.0)


@pytest.mark.parametrize("N,which", [(128, "fused"), (300, "smem")])
def test_weighted_at_the_clamp_threshold_with_concentrated_weights(N, which):
    """The packed weighted path at its largest A with most of the weight on one pair of columns: the A^2 W2 Dma Dmb term
    of the p0 numerator is formed as (r q) W2, which stays finite where q W2 does not (N = 300: W2 = 296)."""
    prob = _at_the_clamp_threshold(3980 + N, N, 6)
    w = prob["weights"] / prob["weights"].sum() * N
    assert (2 ** (59 + 0.76)) ** 2 * 2 ** 0.8 * (w[0] + w[2]) > float(np.finfo(np.float32).max) or N <= 128
    eng, got, _ = _wrun(prob, 200, shared=which)
    _check(eng, prob, got, 200, "weighted at the clamp threshold")


@pytest.mark.parametrize("N,which", [(64, "fused"), (129, "smem")])
def test_weighted_past_the_clamp(N, which):
    """kappa * score <= -45 takes the clamped scalar path (A > 1e18, DESIGN.md 5.2), which bounds u at 2^60 and so does
    not reproduce the exact values there, weighted or not: finite values, antisymmetry and additivity with k-means
    weights; and with weights that differ from uniform by 1e-9 the weighted clamped path matches the uniform one."""
    prob = _wproblem(3950 + N, G=8, N=N, n=6, intercept=-30.0, coef_sd=0.45, zero=True)
    eng, got, _ = _wrun(prob, 200, shared=which)
    _check(eng, prob, got, 200, "weighted past the clamp", compare=False)
    prob["weights"] = None
    _, uniform, path = _run(prob, 200)
    _expect(path, shared=which, bg_weights="uniform")
    prob["weights"] = np.ones(N)
    prob["weights"][N // 2] += 1e-9
    eng, near, _ = _wrun(prob, 200, shared=which)
    _check(eng, prob, near, 200, "weighted past the clamp", compare=False)
    assert rel_err(near[..., 1], uniform[..., 1]) < 1e-5


# ---- l1 feature selection ------------------------------------------------------------------------------------------
def _l1_pair(prob, seed):
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from oracle.shap_kernel_oracle import DenseData as ODenseData, KernelExplainerOracle
    G = len(prob["groups"])
    names = [f"g{k}" for k in range(G)]
    eng = GpuKernelExplainer(prob["clf"].predict_proba, DenseData(prob["bg"], names, prob["groups"], prob["weights"]),
                             link="logit", seed=seed)
    orc = KernelExplainerOracle(prob["clf"].predict_proba, ODenseData(prob["bg"], names, prob["groups"], prob["weights"]),
                                link="logit")
    return eng, orc


@pytest.mark.parametrize("l1_reg", ["aic", "bic", "num_features(5)", "auto"])
@pytest.mark.parametrize("G,N,nsamples", [(16, 20, 300), (80, 40, 700)])
def test_weighted_l1_selection(l1_reg, G, N, nsamples):
    prob = _wproblem(4000 + G, G=G, N=N, n=5, zero=True)
    eng, orc = _l1_pair(prob, seed=3)
    got = eng.shap_values(prob["X"], nsamples=nsamples, l1_reg=l1_reg)
    _expect(eng.last_path(), shared="smem", solve="l1", bg_weights="weighted")
    plan = eng.shared_plan(G, nsamples)
    for i in range(prob["X"].shape[0]):
        want = orc.explain(prob["X"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=nsamples, l1_reg=l1_reg)
        np.testing.assert_array_equal(got[1][i] != 0, want[:, 1] != 0, err_msg=f"instance {i}: other features selected")
        for c in range(2):
            assert rel_err(got[c][i], want[:, c]) < 1e-5, (l1_reg, i, c)


def test_summarised_background_with_default_kwargs():
    """KernelShap.fit(summarise_background=True) clusters the background with k-means and weights each centroid by its
    cluster size; explain() with the default l1_reg='auto' selects features among 64 groups on the weighted kernels."""
    from distributedkernelshap_b200.datasets import dense_tabular
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    from oracle.shap_kernel_oracle import DenseData as ODenseData, KernelExplainerOracle
    d = dense_tabular(n=4, n_features=64, n_background=600, seed=11)
    ks = KernelShap(d["predictor"].predict_proba, link="logit", seed=4)
    ks.fit(d["background"], summarise_background=True)
    eng = ks._explainer
    w = np.asarray(eng.data.weights)
    assert eng.data.data.shape[0] == 300 and w.max() > w.min()
    exp = ks.explain(d["X_explain"], silent=True)
    _expect(eng.last_path(), shared="smem", solve="l1", bg_weights="weighted", chunks=3)
    plan = eng.shared_plan(64, "auto")
    orc = KernelExplainerOracle(d["predictor"].predict_proba,
                                ODenseData(eng.data.data, [f"f{k}" for k in range(64)], None, w), link="logit")
    for i in range(4):
        want = orc.explain(d["X_explain"][i:i + 1], plan=(plan.dense(), plan.weights))
        np.testing.assert_array_equal(exp.shap_values[1][i] != 0, want[:, 1] != 0)
        assert rel_err(exp.shap_values[1][i], want[:, 1]) < 1e-5


# ---- against the other kernels, uniform equivalents, graph replay --------------------------------------------------
@pytest.mark.parametrize("G,N", [(9, 50), (13, 100), (23, 77)])
def test_weighted_cross_kernel(G, N):
    """The weighted shared-plan kernels and the general kernels (which take the weights per background column) agree
    to the bar test_gpu_parity.py's randomized test holds every kernel to."""
    prob = _wproblem(4100 + G, G=G, N=N, n=6, zero=True)
    res = {}
    for kernel in ("auto", "tcgen05", "simt"):
        if kernel == "tcgen05" and G > 15:
            continue
        eng, got, path = _wrun(prob, 500, kernel=kernel)
        if kernel != "auto":
            _expect(path, shared="none")
        res[kernel] = got[..., 1]
    _expect(path, general="simt")
    for kernel, r in res.items():
        assert rel_err(r, res["simt"]) < 5e-6, kernel


@pytest.mark.parametrize("N,G", [(100, 12), (45, 30)])
def test_equal_weights_take_the_uniform_kernels(N, G):
    prob = _problem(4200 + N, G=G, N=N, n=5)
    eng, plain, path = _run(prob, 300)
    _expect(path, bg_weights="uniform")
    prob["weights"] = np.full(N, 3.0)
    eng, got, path = _run(prob, 300)
    _expect(path, bg_weights="uniform", shared="fused" if G <= 16 else "smem")
    assert np.array_equal(got, plain)


def test_weighted_graph_replay_is_bit_identical():
    import torch
    prob = _wproblem(4300, G=12, N=100, n=40, zero=True)
    eng = _engine(prob)
    want = eng.shap_values(prob["X"], nsamples=2048, l1_reg=False)[1]       # plans built + uploaded
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(prob["X"]).cuda()
        phi = torch.zeros((2, 40, 12), dtype=torch.float64, device="cuda")
        phis = []
        for _ in range(3):
            phi.zero_()
            eng.explain_device(X_dev.data_ptr(), 40, phi.data_ptr(), nsamples=2048)
            eng.check_status()
            phis.append(phi.cpu().numpy())
        assert eng.graph_launches() >= 1
        _expect(eng.last_path(), shared="fused", solve="fused", bg_weights="weighted")
    eng.set_stream(0)
    assert np.array_equal(phis[1], phis[0]) and np.array_equal(phis[2], phis[0])
    assert np.array_equal(phis[0][1], want)
    got = np.stack([phis[0][0], phis[0][1]], axis=-1)
    _check(eng, prob, got, 2048, "weighted graph replay")
