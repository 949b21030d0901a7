"""Runs one seeded matrix of explain calls on two builds of libdks.so and requires the same results bit for bit: phi,
expected_value, ``last_path()``, the ``kernel_launches()`` delta of each call, and the error of each refused call.  Use it
to check that a change which must not move any result (a refactor of the per-instance kernels or of the host dispatch)
does not.

Each library runs in a subprocess of its own (``DKS_LIB`` selects the build ``_cabi.load`` opens).  The matrix covers the
per-instance CUDA-core kernels -- linear heads (binary, identity, softmax, one-vs-rest, exp) on ``kernel='simt'``,
mixtures of binary and of softmax members, tree ensembles (sigmoid, softmax, identity and exp heads, and a forest behind a
per-column encoding) and kernel machines (identity and calibrated heads) -- each with shared plans, plans drawn on the
device and caller-supplied plans, and l1 selection on partial varying sets.  Needs a GPU.

    python scripts/lib_parity_probe.py --lib-a build/parent/libdks.so --lib-b distributedkernelshap_b200/libdks.so
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def _problem(seed, P, N, n, const=(2,)):
    """Background and instances; the columns in ``const`` are constant in the background and equal to it on every other
    instance, which therefore has a partial varying set."""
    rng = np.random.default_rng(seed)
    bg, X = rng.normal(size=(N, P)), rng.normal(size=(n, P))
    for c in const:
        bg[:, c] = 0.25
        X[::2, c] = 0.25
    return bg, X


def _linear(head, member=None, R=1, K=1):
    from distributedkernelshap_b200.predictors import LinearModelSpec
    rng = np.random.default_rng(len(head) + R + K)
    rows = K * R
    W, b = rng.normal(0, 0.4, (rows, 8)), rng.normal(0, 0.3, rows)
    pi = rng.uniform(0.2, 1.0, K) if head == "mixture" else None
    return LinearModelSpec(W, b, head, pi=None if pi is None else pi / pi.sum(), member=member)


def _trees(kind):
    from sklearn.ensemble import (GradientBoostingClassifier, GradientBoostingRegressor, HistGradientBoostingRegressor,
                                  RandomForestClassifier)
    rng = np.random.default_rng(3)
    X = rng.normal(size=(400, 8))
    s = X[:, 0] + 0.5 * X[:, 1] - 0.7 * X[:, 2] * X[:, 3]
    if kind == "sigmoid":
        return GradientBoostingClassifier(n_estimators=20, max_depth=3, random_state=0).fit(X, s > 0).predict_proba
    if kind == "softmax":
        return GradientBoostingClassifier(n_estimators=10, max_depth=2, random_state=0).fit(
            X, np.digitize(s, [-1.0, 0.0, 1.0])).predict_proba
    if kind == "identity":
        return GradientBoostingRegressor(n_estimators=20, random_state=0).fit(X, s).predict
    if kind == "exp":
        return HistGradientBoostingRegressor(max_iter=15, loss="poisson", random_state=0).fit(X, np.exp(0.5 * s)).predict
    # a forest behind a per-column encoding: column 7 is categorical
    from sklearn.compose import ColumnTransformer
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import OneHotEncoder, StandardScaler
    X[:, 7] = rng.integers(0, 3, 400)
    ct = ColumnTransformer([("num", StandardScaler(), list(range(7))), ("cat", OneHotEncoder(), [7])])
    return make_pipeline(ct, RandomForestClassifier(10, max_depth=5, random_state=0)).fit(X, s > 0).predict_proba


def _kmach(kind):
    from sklearn.calibration import CalibratedClassifierCV
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler
    from sklearn.svm import SVC, SVR
    rng = np.random.default_rng(4)
    X = rng.normal(size=(150, 8))
    s = X[:, 0] + 0.5 * X[:, 1] * X[:, 2]
    if kind == "identity":
        return make_pipeline(StandardScaler(), SVR()).fit(X, s).predict
    return CalibratedClassifierCV(make_pipeline(StandardScaler(), SVC()), ensemble=False, cv=3).fit(X, s > 0).predict_proba


def _models():
    """name -> (model factory, link, engine options)"""
    simt = {"kernel": "simt"}
    m = {
        "simt_binary": (lambda: _linear("binary_logistic"), "logit", simt),
        "simt_identity": (lambda: _linear("identity", R=2), "identity", simt),
        "simt_softmax": (lambda: _linear("softmax", R=3), "logit", simt),
        "simt_ovr": (lambda: _linear("ovr", R=3), "logit", simt),
        "simt_exp": (lambda: _linear("exp"), "identity", simt),
        "mix_binary": (lambda: _linear("mixture", member="binary_logistic", K=3), "logit", simt),
        "mix_softmax": (lambda: _linear("mixture", member="softmax", R=3, K=2), "logit", simt),
        "km_identity": (lambda: _kmach("identity"), "identity", {}),
        "km_calibrated": (lambda: _kmach("calibrated"), "logit", {}),
    }
    for kind, link in (("sigmoid", "logit"), ("softmax", "logit"), ("identity", "identity"), ("exp", "identity"),
                       ("encoded", "logit")):
        m["trees_" + kind] = (lambda kind=kind: _trees(kind), link, {})
    return m


def _run_case(model, link, opts, plans, l1_reg, bg, X, nsamples):
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    P = bg.shape[1]
    data = DenseData(bg, [f"g{k}" for k in range(P)], [[k] for k in range(P)])
    kw = dict(opts)
    if plans == "per_instance":
        kw["plan_mode"] = "per_instance"
    eng = GpuKernelExplainer(model, data, link=link, seed=11, **kw)
    eng.set_option("graph", 0)
    call = {"nsamples": nsamples, "l1_reg": l1_reg}
    if plans == "caller":
        M, _ = eng.varying(X)
        call["plans"] = [None if m < 2 else (eng.shared_plan(int(m), nsamples).zbits, eng.shared_plan(int(m), nsamples).weights)
                         for m in M]
    before = eng.kernel_launches()
    try:
        phi = eng.shap_values(X, **call)
    except Exception as e:          # a refusal is a result too: its type and message must agree
        return {"error": f"{type(e).__name__}: {e}", "launches": eng.kernel_launches() - before}, None
    out = {"launches": eng.kernel_launches() - before, "path": eng.last_path(),
           "expected_value": np.atleast_1d(eng.expected_value).tolist()}
    return out, np.stack(phi if isinstance(phi, list) else [phi])


def worker(out_dir):
    meta, arrays = {}, {}
    for name, (make, link, opts) in _models().items():
        model = make()
        bg, X = _problem(7, 8, 40, 10)
        if name == "trees_encoded":     # the encoded column takes the categories the encoder was fitted on
            bg[:, 7], X[:, 7] = np.arange(40) % 3, np.arange(10) % 3
        for plans in ("shared", "per_instance", "caller"):
            for l1_reg in ((False, "num_features(3)") if plans == "shared" else (False,)):
                key = f"{name}/{plans}/{l1_reg}"
                # l1: kernel 'auto', so the full-set instances take the shared-plan route (the only one that selects
                # for them) and the partial ones the L1 instantiation of the family's CUDA-core kernel
                info, phi = _run_case(model, link, {} if l1_reg else opts, plans, l1_reg, bg, X, 300)
                meta[key] = info
                if phi is not None:
                    arrays[key] = phi
                    arrays[key + "/ev"] = np.asarray(info["expected_value"])
                print(key, json.dumps({k: v for k, v in info.items() if k != "path"}), flush=True)
    np.savez(os.path.join(out_dir, "phi.npz"), **arrays)
    with open(os.path.join(out_dir, "meta.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-a", required=True)
    ap.add_argument("--lib-b", required=True)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args.worker)
    outs = []
    with tempfile.TemporaryDirectory() as tmp:
        for tag, lib in (("a", args.lib_a), ("b", args.lib_b)):
            d = os.path.join(tmp, tag)
            os.makedirs(d)
            env = dict(os.environ, DKS_LIB=os.path.abspath(lib))
            subprocess.run([sys.executable, os.path.abspath(__file__), "--lib-a", lib, "--lib-b", lib, "--worker", d],
                           env=env, cwd=REPO, check=True)
            with open(os.path.join(d, "meta.json")) as f:
                meta = json.load(f)
            with np.load(os.path.join(d, "phi.npz")) as z:
                outs.append((meta, {k: z[k] for k in z.files}))
    (ma, pa), (mb, pb) = outs
    bad = [k for k in sorted(set(ma) | set(mb)) if ma.get(k) != mb.get(k)]
    bad += [k for k in sorted(set(pa) | set(pb)) if k not in pa or k not in pb or not np.array_equal(pa[k], pb[k])]
    refused = sum("error" in v for v in ma.values())
    print(json.dumps({"cases": len(ma), "refused_in_both": refused, "arrays": len(pa), "mismatches": bad}))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
