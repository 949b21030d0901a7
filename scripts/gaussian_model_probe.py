"""Throughput of the Gaussian route (DESIGN.md §5.0.23) on the Adult-shaped problem: 2560 instances, a 100-row background,
12 groups over 49 columns, nsamples 2048, for Gaussian generative models fitted on 2560 rows (labels drawn from the
problem's predictor probabilities):

  QuadraticDiscriminantAnalysis(reg_param=0.5).predict_proba      logit link (2 classes)
  GaussianNB().predict_proba                                      identity link
  GaussianMixture(5).score_samples / .predict_proba               identity link
  EllipticEnvelope().decision_function                            identity link

Per model: instances/s from the engine's device events (stage 1 to the end of the solve), the explain stage's time (CUDA
events), its FP64 operation count computed from the shapes -- per (coalition, background row, component) |z| (|z| + 1) / 2
table adds and one fma, per (background row, component) 2 r_k M (M + 1) / 2 for the tables -- and the rate that gives, and,
as the CPU figure, the oracle calling the real scikit-learn method on the masked batch for a few instances.  The card name,
power limit and SM clock are read in the same run.  Prints one JSON document; ``--out`` also writes it to a file.

    python scripts/gaussian_model_probe.py [--n 2560] [--fit-rows 2560] [--oracle-instances 2] [--out result.json]
"""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.tree_probe import card  # noqa: E402


def flops_per_instance(spec, plan, N, M):
    """FP64 operations of the explain kernel for one instance whose M groups all vary, from the plan's coalitions."""
    pc = np.asarray(plan.dense(), dtype=np.float64).sum(axis=1)
    ranks = np.array([Lk.shape[1] for Lk in spec.L], dtype=np.float64)
    coalitions = N * spec.K * float(np.sum(pc * (pc + 1) / 2 + 2))
    tables = N * float(np.sum(2 * ranks * M * (M + 1) / 2))
    return coalitions, tables


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2560)
    ap.add_argument("--nsamples", type=int, default=2048)
    ap.add_argument("--fit-rows", type=int, default=2560)
    ap.add_argument("--oracle-instances", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from sklearn.covariance import EllipticEnvelope
    from sklearn.discriminant_analysis import QuadraticDiscriminantAnalysis
    from sklearn.mixture import GaussianMixture
    from sklearn.naive_bayes import GaussianNB

    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.gaussian_models import extract_gaussian_spec
    from oracle.shap_kernel_oracle import DenseData as ODense, KernelExplainerOracle

    d = adult_like(n_explain=a.n + a.fit_rows, n_background=100, seed=0)
    X_fit = d["X_explain"][a.n:a.n + a.fit_rows]
    p = d["predictor"].predict_proba(X_fit)[:, 1]
    y = (np.random.default_rng(1).random(len(p)) < p).astype(int)
    X_exp = d["X_explain"][:a.n]
    result = {"card": card(), "n": a.n, "N": 100, "groups": len(d["groups"]), "columns": X_fit.shape[1],
              "nsamples": a.nsamples, "fit_rows": a.fit_rows, "models": {}}
    data = DenseData(d["background"], d["group_names"], d["groups"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        qda = QuadraticDiscriminantAnalysis(reg_param=0.5).fit(X_fit, y)
        nb = GaussianNB().fit(X_fit, y)
        gmm = GaussianMixture(5, random_state=0).fit(X_fit)
        env = EllipticEnvelope(random_state=0).fit(X_fit)
    models = [("QuadraticDiscriminantAnalysis(reg_param=0.5).predict_proba", qda.predict_proba, "logit"),
              ("GaussianNB().predict_proba", nb.predict_proba, "identity"),
              ("GaussianMixture(5).score_samples", gmm.score_samples, "identity"),
              ("GaussianMixture(5).predict_proba", gmm.predict_proba, "identity"),
              ("EllipticEnvelope().decision_function", env.decision_function, "identity")]
    for name, fn, link in models:
        spec = extract_gaussian_spec(fn)
        eng = GpuKernelExplainer(fn, data, link=link, seed=0)
        M, _ = eng.varying(X_exp)
        Mf = int(M.max())
        plan = eng.shared_plan(Mf, a.nsamples)
        S = int(plan.S)
        coal, tab = flops_per_instance(spec, plan, 100, Mf)
        entry = {"link": link, "K": spec.K, "ranks": [int(Lk.shape[1]) for Lk in spec.L], "head": spec.head,
                 "S_full_set": S, "instances_full_set": int((M == Mf).sum()),
                 "fp64_ops_per_instance_coalitions": coal, "fp64_ops_per_instance_tables": tab}
        eng.shap_values(X_exp[:64], nsamples=a.nsamples, l1_reg=False)      # plans uploaded, kernels loaded
        t0 = time.perf_counter()
        eng.shap_values(X_exp, nsamples=a.nsamples, l1_reg=False)
        wall = time.perf_counter() - t0
        tm = eng.last_timings_ms()
        ops = (coal + tab) * a.n
        entry.update({"total_ms": tm["total"], "explain_stage_ms": tm["coalitions"],
                      "instances_per_s": a.n / (tm["total"] * 1e-3), "wall_s": wall,
                      "fp64_ops_total_upper_bound": ops,
                      "fp64_gops_per_s_explain_stage": ops / (tm["coalitions"] * 1e-3) / 1e9,
                      "general": eng.last_path()["general"]})
        print(name, entry, flush=True)
        # CPU figure: the oracle with the real scikit-learn method on the engine's plans
        orc = KernelExplainerOracle(fn, ODense(d["background"], d["group_names"], d["groups"]), link=link)
        t0 = time.perf_counter()
        for i in range(a.oracle_instances):
            pl = eng.shared_plan(int(M[i]), a.nsamples)
            orc.explain(X_exp[i:i + 1], plan=(pl.dense(), pl.weights), nsamples=a.nsamples, l1_reg=False)
        entry["oracle_cpu_s_per_instance"] = (time.perf_counter() - t0) / a.oracle_instances
        result["models"][name] = entry
        eng.close()
    text = json.dumps(result, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
