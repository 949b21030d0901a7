"""One small case per route of the explain dispatcher: what ``last_path()`` reports and how many kernels one plain call
(no CUDA graph) launches, pinned per route, and the refusals with their status code, message and launch count.  A
change to the host code that picks the kernels must leave every row as it is."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LINK = {"binary_logistic": "logit", "softmax": "logit", "ovr": "logit", "mixture": "logit", "identity": "identity",
        "exp": "identity"}


def _problem(seed, head, G, N, n, R=1, const=None, member=None, K=2):
    """One column per group.  ``const``: {group: rows of X} -- that group is constant in the background and equal to it
    in those rows, which therefore have a partial varying set."""
    rng = np.random.default_rng(seed)
    rows = K * R if head == "mixture" else R
    W = rng.normal(0, 1.2 / np.sqrt(G), (rows, G))
    b = rng.normal(0, 0.3, rows)
    bg, X = rng.standard_normal((N, G)), rng.standard_normal((n, G))
    for g, r in (const or {}).items():
        bg[:, g] = 0.25
        X[r, g] = 0.25
    pi = rng.uniform(0.2, 1.0, K) if head == "mixture" else None
    return dict(W=W, b=b, bg=bg, X=X, head=head, member=member, pi=None if pi is None else pi / pi.sum())


def _engine(prob, **kw):
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.predictors import LinearModelSpec
    head = prob["head"]
    spec = LinearModelSpec(prob["W"], prob["b"], head, pi=prob["pi"], member=prob["member"])
    G = prob["bg"].shape[1]
    data = DenseData(prob["bg"], [f"g{k}" for k in range(G)], [[k] for k in range(G)])
    eng = GpuKernelExplainer(spec, data, link=LINK[head], seed=5, **kw)
    eng.set_option("graph", 0)
    return eng


# name: (problem, engine options, nsamples, l1_reg)
CASES = {
    "binary_fused": (dict(seed=1, head="binary_logistic", G=13, N=64, n=6), {}, 400, False),
    "binary_smem_pmat": (dict(seed=2, head="binary_logistic", G=20, N=40, n=5), {}, 200, False),
    "binary_smem_pmat_chunks": (dict(seed=3, head="binary_logistic", G=13, N=257, n=5), {}, 300, False),
    "binary_wls_shared": (dict(seed=4, head="binary_logistic", G=26, N=40, n=5), {}, 300, False),
    "binary_two_word_flagged": (dict(seed=5, head="binary_logistic", G=70, N=40, n=3), {}, 600, False),
    "binary_wide": (dict(seed=6, head="binary_logistic", G=130, N=40, n=3), {}, 600, False),
    "binary_fused_and_tc": (dict(seed=7, head="binary_logistic", G=12, N=50, n=10, const={5: [5, 6, 7, 8, 9]}), {}, 500,
                            False),
    "binary_l1_full": (dict(seed=8, head="binary_logistic", G=12, N=30, n=5), {}, 300, "aic"),
    "binary_l1_general": (dict(seed=9, head="binary_logistic", G=12, N=30, n=8, const={3: [2, 3, 4]}), {}, 300, "aic"),
    "softmax": (dict(seed=10, head="softmax", G=10, N=40, n=5, R=3), {}, 300, False),
    "softmax_l1_full": (dict(seed=11, head="softmax", G=10, N=40, n=5, R=3), {}, 300, "aic"),
    "ovr": (dict(seed=12, head="ovr", G=10, N=40, n=5, R=3), {}, 300, False),
    "affine": (dict(seed=13, head="identity", G=10, N=40, n=5, R=2), {}, 300, False),
    "exp": (dict(seed=14, head="exp", G=10, N=40, n=5), {}, 300, False),
    "exp_partial_simt": (dict(seed=15, head="exp", G=10, N=40, n=6, const={2: [1, 2]}), {}, 300, False),
    "mixture_binary": (dict(seed=16, head="mixture", member="binary_logistic", G=10, N=40, n=5), {}, 300, False),
    "mixture_binary_l1_full": (dict(seed=17, head="mixture", member="binary_logistic", G=10, N=40, n=5), {}, 300, "aic"),
    "mixture_softmax": (dict(seed=18, head="mixture", member="softmax", R=3, G=10, N=40, n=5), {}, 300, False),
    "mixture_ovr_partial": (dict(seed=19, head="mixture", member="ovr", R=3, G=10, N=40, n=6, const={4: [0, 1]}), {}, 300,
                            False),
    "per_instance_64": (dict(seed=20, head="binary_logistic", G=64, N=30, n=4), {"plan_mode": "per_instance"}, 400, False),
    "per_instance_70": (dict(seed=21, head="binary_logistic", G=70, N=30, n=4), {"plan_mode": "per_instance"}, 400, False),
    "per_instance_small": (dict(seed=22, head="binary_logistic", G=9, N=30, n=4), {"plan_mode": "per_instance"}, 200,
                           False),
    "tc": (dict(seed=23, head="binary_logistic", G=9, N=50, n=6), {"kernel": "tcgen05"}, 300, False),
    "simt": (dict(seed=24, head="binary_logistic", G=9, N=50, n=6), {"kernel": "simt"}, 300, False),
}

# name: (last_path(), kernel_launches() of the second call)
EXPECTED = {
    "affine": ({"shared": "affine", "chunks": 0, "warps": 0, "grid": 0, "fused_B": 0, "fused_NI": 0, "solve": "wls_shared", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
              3),
    "binary_fused": ({"shared": "fused", "chunks": 1, "warps": 16, "grid": 132, "fused_B": 8, "fused_NI": 1, "solve": "fused", "pmat_kpad": 0, "general": "tc", "cta_warps": 16, "bg_weights": "uniform", "fused_table": 1, "general_l1": 0},
                    3),
    "binary_fused_and_tc": ({"shared": "fused", "chunks": 1, "warps": 19, "grid": 132, "fused_B": 8, "fused_NI": 1, "solve": "fused", "pmat_kpad": 0, "general": "tc", "cta_warps": 19, "bg_weights": "uniform", "fused_table": 1, "general_l1": 0},
                           3),
    # the l1 solve enqueues two kernels (moments, LARS); the dispatcher used to count one of them here
    "binary_l1_full": ({"shared": "smem", "chunks": 1, "warps": 20, "grid": 132, "fused_B": 0, "fused_NI": 0, "solve": "l1", "pmat_kpad": 0, "general": "tc", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                      5 + 1),
    # the l1 solve enqueues two kernels (moments, LARS); the dispatcher used to count one of them here
    "binary_l1_general": ({"shared": "smem", "chunks": 1, "warps": 20, "grid": 132, "fused_B": 0, "fused_NI": 0, "solve": "l1", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 1},
                         8 + 1),
    "binary_smem_pmat": ({"shared": "smem", "chunks": 1, "warps": 20, "grid": 132, "fused_B": 0, "fused_NI": 0, "solve": "pmat", "pmat_kpad": 20, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                        4),
    "binary_smem_pmat_chunks": ({"shared": "smem", "chunks": 3, "warps": 14, "grid": 132, "fused_B": 0, "fused_NI": 0, "solve": "pmat", "pmat_kpad": 12, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                               6),
    "binary_two_word_flagged": ({"shared": "smem", "chunks": 1, "warps": 20, "grid": 132, "fused_B": 0, "fused_NI": 0, "solve": "wls_shared", "pmat_kpad": 0, "general": "flagged", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                               4),
    "binary_wide": ({"shared": "smem", "chunks": 1, "warps": 20, "grid": 132, "fused_B": 0, "fused_NI": 0, "solve": "wide", "pmat_kpad": 0, "general": "flagged", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                   6),
    "binary_wls_shared": ({"shared": "smem", "chunks": 1, "warps": 20, "grid": 132, "fused_B": 0, "fused_NI": 0, "solve": "wls_shared", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                         4),
    "exp": ({"shared": "exp", "chunks": 0, "warps": 0, "grid": 0, "fused_B": 0, "fused_NI": 0, "solve": "wls_shared", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
           3),
    "exp_partial_simt": ({"shared": "exp", "chunks": 0, "warps": 0, "grid": 0, "fused_B": 0, "fused_NI": 0, "solve": "wls_shared", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                        3),
    "mixture_binary": ({"shared": "mixture", "chunks": 2, "warps": 20, "grid": 132, "fused_B": 0, "fused_NI": 0, "solve": "pmat", "pmat_kpad": 12, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                      7),
    # the l1 solve enqueues two kernels (moments, LARS); the dispatcher used to count one of them here
    "mixture_binary_l1_full": ({"shared": "mixture", "chunks": 2, "warps": 20, "grid": 132, "fused_B": 0, "fused_NI": 0, "solve": "l1", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                              8 + 1),
    "mixture_ovr_partial": ({"shared": "mixture", "chunks": 2, "warps": 8, "grid": 10, "fused_B": 0, "fused_NI": 0, "solve": "wls_shared", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                           7),
    "mixture_softmax": ({"shared": "mixture", "chunks": 2, "warps": 8, "grid": 10, "fused_B": 0, "fused_NI": 0, "solve": "wls_shared", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                       7),
    "ovr": ({"shared": "ovr", "chunks": 1, "warps": 8, "grid": 10, "fused_B": 0, "fused_NI": 0, "solve": "wls_shared", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
           4),
    "per_instance_64": ({"shared": "none", "chunks": 0, "warps": 0, "grid": 0, "fused_B": 0, "fused_NI": 0, "solve": "none", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                       4),
    "per_instance_70": ({"shared": "none", "chunks": 0, "warps": 0, "grid": 0, "fused_B": 0, "fused_NI": 0, "solve": "none", "pmat_kpad": 0, "general": "simt_wide", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                       5),
    "per_instance_small": ({"shared": "none", "chunks": 0, "warps": 0, "grid": 0, "fused_B": 0, "fused_NI": 0, "solve": "none", "pmat_kpad": 0, "general": "tc", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                          4),
    "simt": ({"shared": "none", "chunks": 0, "warps": 0, "grid": 0, "fused_B": 0, "fused_NI": 0, "solve": "none", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
            2),
    "softmax": ({"shared": "softmax", "chunks": 1, "warps": 8, "grid": 10, "fused_B": 0, "fused_NI": 0, "solve": "wls_shared", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
               4),
    "softmax_l1_full": ({"shared": "softmax", "chunks": 1, "warps": 8, "grid": 10, "fused_B": 0, "fused_NI": 0, "solve": "l1", "pmat_kpad": 0, "general": "simt", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
                       6),
    "tc": ({"shared": "none", "chunks": 0, "warps": 0, "grid": 0, "fused_B": 0, "fused_NI": 0, "solve": "none", "pmat_kpad": 0, "general": "tc", "cta_warps": 0, "bg_weights": "uniform", "fused_table": 0, "general_l1": 0},
          2),
}


def _observe(name):
    spec, opts, ns, l1 = CASES[name]
    eng = _engine(_problem(**spec), **opts)
    X = _problem(**spec)["X"]
    eng.shap_values(X, nsamples=ns, l1_reg=l1)              # uploads the plans and l1 tables this call needs
    before = eng.kernel_launches()
    eng.shap_values(X, nsamples=ns, l1_reg=l1)
    return eng.last_path(), eng.kernel_launches() - before


@pytest.mark.parametrize("name", sorted(CASES))
def test_route(name):
    path, launches = _observe(name)
    want_path, want_launches = EXPECTED[name]
    assert path == want_path
    assert launches == want_launches


# ---- refusals: status code, message and kernels launched by the refused call (stage 1 only) ----------------------------
def _raw_explain(eng, X, zb=None, w=None, stride=0):
    from distributedkernelshap_b200 import _cabi
    phi = np.zeros((eng.D, X.shape[0], eng.data.groups_size))
    X = np.ascontiguousarray(X)
    before = eng.kernel_launches()
    rc = eng.lib.dks_explain_host(eng._ctx, _cabi.ptr(X), X.shape[0], _cabi.ptr(phi), _cabi.ptr(zb), _cabi.ptr(w), stride)
    msg = eng.lib.dks_last_error().decode()
    return rc, msg, eng.kernel_launches() - before


def _upload_plans(eng, X, ns):
    from distributedkernelshap_b200 import _cabi
    eng._set_nsamples(ns)
    _cabi.check(eng.lib.dks_prepare_host(eng._ctx, _cabi.ptr(np.ascontiguousarray(X)), X.shape[0]))
    eng._ensure_shared_plans(eng.m_histogram(), ns)


def _refuse_shared_kernel_without_shared_route():
    prob = _problem(30, "softmax", G=130, N=20, n=2, R=3)
    eng = _engine(prob, kernel="shared")
    _upload_plans(eng, prob["X"], 600)
    return _raw_explain(eng, prob["X"])


def _refuse_l1_with_per_instance_plans():
    prob = _problem(31, "binary_logistic", G=10, N=20, n=3)
    eng = _engine(prob, plan_mode="per_instance")
    eng.shap_values(prob["X"], nsamples=200, l1_reg=False)
    from distributedkernelshap_b200 import _cabi
    _cabi.check(eng.lib.dks_set_l1(eng._ctx, 1, 0, C.c_uint64(1 << 9), C.c_uint64(0)))
    return _raw_explain(eng, prob["X"])


def _refuse_mixture_on_tc():
    prob = _problem(32, "mixture", G=8, N=20, n=2, member="binary_logistic")
    eng = _engine(prob, kernel="tcgen05")
    _upload_plans(eng, prob["X"], 200)
    return _raw_explain(eng, prob["X"])


def _refuse_caller_plans_beyond_64_groups():
    prob = _problem(33, "binary_logistic", G=70, N=20, n=2)
    eng = _engine(prob)
    stride = 8
    zb = np.zeros((2, stride, 2), dtype=np.uint64)
    w = np.zeros((2, stride))
    return _raw_explain(eng, prob["X"], zb, w, stride)


def _refuse_missing_plan_two_word():
    prob = _problem(34, "binary_logistic", G=70, N=20, n=2)
    return _raw_explain(_engine(prob), prob["X"])


def _refuse_missing_plan_softmax():
    prob = _problem(35, "softmax", G=100, N=200, n=2, R=3)
    eng = _engine(prob)
    eng._set_nsamples(4000)
    return _raw_explain(eng, prob["X"])


# name: (setup, status code, message substring, kernels launched: stage 1's only)
REFUSALS = {
    "shared_kernel_without_shared_route": (_refuse_shared_kernel_without_shared_route, 3,
                                           "shared-plan fast path needs the binary-logistic head", 1),
    # refused before the sampler draws the plans (it used to run the sampler's two kernels first)
    "l1_with_per_instance_plans": (_refuse_l1_with_per_instance_plans, 3, "l1 feature selection runs on shared plans only",
                                   1),
    "mixture_on_tc": (_refuse_mixture_on_tc, 3, "mixture head: no tensor-core kernel", 1),
    "caller_plans_beyond_64_groups": (_refuse_caller_plans_beyond_64_groups, 3,
                                      "caller-supplied per-instance plans are not supported", 1),
    "missing_plan_two_word": (_refuse_missing_plan_two_word, 4, "no shared plan for M=70", 1),
    "missing_plan_softmax": (_refuse_missing_plan_softmax, 4, "no shared plan for M=100", 1),
}


@pytest.mark.parametrize("name", sorted(REFUSALS))
def test_refusal(name):
    setup, code, text, launches = REFUSALS[name]
    rc, msg, got = setup()
    assert rc == code, (rc, msg)
    assert text in msg, msg
    assert got == launches


def test_replaced_plan_drops_its_sampling_state():
    """A plan replaced under another nsamples takes its sampling info with it, on the device too: a per-instance explain
    before the new info is uploaded reports the plan of that M as missing."""
    from distributedkernelshap_b200 import _cabi
    from distributedkernelshap_b200.plan import build_plan
    prob = _problem(40, "binary_logistic", G=10, N=20, n=3)
    eng = _engine(prob, plan_mode="per_instance")
    eng.shap_values(prob["X"], nsamples=200, l1_reg=False)          # plan of M = 10 and its sampling info
    plan = build_plan(10, 300, rng=np.random.RandomState(1))
    eng._set_nsamples(300)
    _cabi.check(eng.lib.dks_set_shared_plan(eng._ctx, 10, plan.S, _cabi.ptr(plan.zbits), _cabi.ptr(plan.weights)))
    rc, msg, _ = _raw_explain(eng, prob["X"])
    assert rc == _cabi.DKS_ERR_PLAN_MISSING, (rc, msg)
    assert "M=10" in msg, msg
