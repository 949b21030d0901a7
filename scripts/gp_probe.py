"""Throughput of the kernel-machine route's program kernel (DESIGN.md §5.0.21) on the Adult-shaped problem: 2560
instances, a 100-row background, 12 groups over 49 columns, nsamples 2048, for three models fitted on 2000 rows:

  make_pipeline(StandardScaler(), GaussianProcessRegressor(ConstantKernel() * RBF(np.ones(49)) + WhiteKernel()))  predict
  make_pipeline(StandardScaler(), GaussianProcessRegressor(ConstantKernel() * Matern(nu=2.5) + WhiteKernel()))   predict
  make_pipeline(StandardScaler(), OneClassSVM())                                                     decision_function

The GPs are fitted to the problem predictor's probabilities with the hyperparameters as given (optimizer=None: the
optimiser's gradient over 51 length scales at 2000 rows is a 1.6 GB tensor per step; the explained model has the same
shape either way).  Per model: instances/s from the engine's device events (stage 1 to the end of the solve), the explain
stage's time, the kernel evaluations per instance (S N n_sv L) and, as the CPU figure, the oracle calling the real
scikit-learn method on the masked batch for a few instances.  The card name, power limit and SM clock are read in the same
run.

With ``--parent-lib``, the same call also times ``make_pipeline(StandardScaler(), SVC()).decision_function`` (the first
model of scripts/kernel_machine_probe.py) under that build of the library and under this one, alternating, each in its own
process: the existing kernels' speed next to the parent's.  Prints one JSON document; ``--out`` also writes it to a file.

    python scripts/gp_probe.py [--n 2560] [--fit-rows 2000] [--oracle-instances 1] [--parent-lib PATH] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.tree_probe import card  # noqa: E402


def _svc_run(a):
    """One timing of the scaled SVC's decision_function on the library DKS_LIB names (or this build)."""
    from distributedkernelshap_b200 import _cabi
    if os.environ.get("DKS_LIB"):               # the parent library predates the program kernel's entry point
        _cabi.SIGNATURES.pop("dks_set_kernel_program", None)
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler
    from sklearn.svm import SVC

    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.engine import GpuKernelExplainer

    d = adult_like(n_explain=max(a.n, 3000), n_background=100, seed=0)
    X_fit = d["X_explain"][:3000]
    p = d["predictor"].predict_proba(X_fit)[:, 1]
    y = (np.random.default_rng(1).random(len(p)) < p).astype(int)      # as scripts/kernel_machine_probe.py
    svc = make_pipeline(StandardScaler(), SVC()).fit(X_fit, y)
    eng = GpuKernelExplainer(svc.decision_function, DenseData(d["background"], d["group_names"], d["groups"]),
                             link="identity", seed=0)
    X_exp = d["X_explain"][:a.n]
    eng.shap_values(X_exp[:64], nsamples=a.nsamples, l1_reg=False)
    best = None
    for _ in range(3):
        phi = eng.shap_values(X_exp, nsamples=a.nsamples, l1_reg=False)
        tm = eng.last_timings_ms()
        best = tm["total"] if best is None else min(best, tm["total"])
    print(json.dumps({"total_ms": best, "instances_per_s": a.n / (best * 1e-3),
                      "phi_sum": float(np.sum(np.abs(np.asarray(phi)))), "general": eng.last_path()["general"]}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2560)
    ap.add_argument("--nsamples", type=int, default=2048)
    ap.add_argument("--fit-rows", type=int, default=2000)
    ap.add_argument("--oracle-instances", type=int, default=1)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--svc-only", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.svc_only:
        _svc_run(a)
        return

    import warnings

    from sklearn.gaussian_process import GaussianProcessRegressor
    from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern, WhiteKernel
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler
    from sklearn.svm import OneClassSVM

    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.kernel_machines import extract_kernel_machine_spec
    from oracle.shap_kernel_oracle import DenseData as ODense, KernelExplainerOracle

    d = adult_like(n_explain=max(a.n, a.fit_rows), n_background=100, seed=0)
    X_fit = d["X_explain"][:a.fit_rows]
    P = X_fit.shape[1]
    p = d["predictor"].predict_proba(X_fit)[:, 1]
    X_exp = d["X_explain"][:a.n]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gp_rbf = make_pipeline(StandardScaler(), GaussianProcessRegressor(
            ConstantKernel() * RBF(np.ones(P)) + WhiteKernel(), optimizer=None)).fit(X_fit, p)
        gp_mat = make_pipeline(StandardScaler(), GaussianProcessRegressor(
            ConstantKernel() * Matern(nu=2.5) + WhiteKernel(), optimizer=None)).fit(X_fit, p)
        ocsvm = make_pipeline(StandardScaler(), OneClassSVM()).fit(X_fit)
    models = {
        "make_pipeline(StandardScaler(), GaussianProcessRegressor(ConstantKernel() * RBF(np.ones(49)) + "
        "WhiteKernel())).predict": gp_rbf.predict,
        "make_pipeline(StandardScaler(), GaussianProcessRegressor(ConstantKernel() * Matern(nu=2.5) + "
        "WhiteKernel())).predict": gp_mat.predict,
        "make_pipeline(StandardScaler(), OneClassSVM()).decision_function": ocsvm.decision_function,
    }
    result = {"card": card(), "n": a.n, "N": 100, "groups": len(d["groups"]), "columns": P, "nsamples": a.nsamples,
              "fit_rows": a.fit_rows, "models": {}}
    data = DenseData(d["background"], d["group_names"], d["groups"])
    for name, fn in models.items():
        spec = extract_kernel_machine_spec(fn)
        L = spec.program.L if spec.program is not None else 1
        eng = GpuKernelExplainer(fn, data, link="identity", seed=0)
        M, _ = eng.varying(X_exp)
        S = int(eng.shared_plan(int(M.max()), a.nsamples).S)
        entry = {"kernel": spec.kernel, "statistics": L, "n_sv": spec.n_sv, "S_full_set": S,
                 "kernel_evaluations_per_instance": S * 100 * spec.n_sv, "statistic_rows_per_instance":
                 S * 100 * spec.n_sv * L}
        eng.shap_values(X_exp[:64], nsamples=a.nsamples, l1_reg=False)     # plans uploaded, kernels loaded
        t0 = time.perf_counter()
        eng.shap_values(X_exp, nsamples=a.nsamples, l1_reg=False)
        wall = time.perf_counter() - t0
        tm = eng.last_timings_ms()
        entry.update(total_ms=tm["total"], explain_stage_ms=tm["coalitions"], instances_per_s=a.n / (tm["total"] * 1e-3),
                     wall_s=wall, general=eng.last_path()["general"])
        print(name, entry, flush=True)
        orc = KernelExplainerOracle(fn, ODense(d["background"], d["group_names"], d["groups"]), link="identity")
        t0 = time.perf_counter()
        for i in range(a.oracle_instances):
            plan = eng.shared_plan(int(M[i]), a.nsamples)
            orc.explain(X_exp[i:i + 1], plan=(plan.dense(), plan.weights), nsamples=a.nsamples, l1_reg=False)
        entry["oracle_cpu_s_per_instance"] = (time.perf_counter() - t0) / a.oracle_instances
        entry["oracle_instances"] = a.oracle_instances
        result["models"][name] = entry
        eng.close()
    if a.parent_lib:
        runs = []
        for build in ("parent", "new", "parent", "new"):
            env = dict(os.environ)
            if build == "parent":
                env["DKS_LIB"] = os.path.abspath(a.parent_lib)
            else:
                env.pop("DKS_LIB", None)
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--svc-only", "--n", str(a.n),
                                  "--nsamples", str(a.nsamples)], env=env, capture_output=True, text=True, check=True)
            r = json.loads(out.stdout.strip().splitlines()[-1])
            r["build"] = build
            runs.append(r)
            print("svc", r, flush=True)
        result["svc_decision_function_parent_vs_new"] = runs
    result["card_after"] = card()
    text = json.dumps(result, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
