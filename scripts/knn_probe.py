"""Throughput of the neighbour route (DESIGN.md §5.0.15) on the Adult-shaped problem: 2560 instances, a 100-row
background, 12 groups over 49 columns, nsamples 2048, for the default scaled k-nearest-neighbour classifier fitted on
2560 rows to labels drawn from the problem's predictor probabilities, with uniform and with distance weights:

  make_pipeline(StandardScaler(), KNeighborsClassifier(weights=w)).predict_proba     identity link

Per model: instances/s from the engine's device events (stage 1 to the end of the solve) and the explain stage's time,
the candidate (coalition, background row, training row) triples per instance (S N n_fit), and, as the CPU figure, the
oracle calling the real scikit-learn method on the masked batch for a few instances.  The engine is given the
scikit-learn method itself, so its fit check runs at this shape; the background rows whose k-th and (k + 1)-th neighbours
tie (checked against the engine's rule instead) are counted.  The card name, power limit and SM clock are read in the same
run.  Prints one JSON document; ``--out`` also writes it to a file.

    python scripts/knn_probe.py [--n 2560] [--fit-rows 2560] [--oracle-instances 2] [--out result.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.tree_probe import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2560)
    ap.add_argument("--nsamples", type=int, default=2048)
    ap.add_argument("--fit-rows", type=int, default=2560)
    ap.add_argument("--oracle-instances", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from sklearn.neighbors import KNeighborsClassifier
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler

    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.neighbors import extract_knn_spec
    from oracle.shap_kernel_oracle import DenseData as ODense, KernelExplainerOracle

    d = adult_like(n_explain=a.n + a.fit_rows, n_background=100, seed=0)
    X_fit = d["X_explain"][a.n:a.n + a.fit_rows]
    p = d["predictor"].predict_proba(X_fit)[:, 1]
    y = (np.random.default_rng(1).random(len(p)) < p).astype(int)
    X_exp = d["X_explain"][:a.n]
    result = {"card": card(), "n": a.n, "N": 100, "groups": len(d["groups"]), "columns": X_fit.shape[1],
              "nsamples": a.nsamples, "fit_rows": a.fit_rows, "models": {}}
    data = DenseData(d["background"], d["group_names"], d["groups"])
    for weights in ("uniform", "distance"):
        name = f"make_pipeline(StandardScaler(), KNeighborsClassifier(weights={weights!r})).predict_proba"
        fn = make_pipeline(StandardScaler(), KNeighborsClassifier(weights=weights)).fit(X_fit, y).predict_proba
        spec = extract_knn_spec(fn)
        eng = GpuKernelExplainer(fn, data, link="identity", seed=0)
        M, _ = eng.varying(X_exp)
        S = int(eng.shared_plan(int(M.max()), a.nsamples).S)
        entry = {"link": "identity", "k": spec.k, "n_fit": spec.n_fit, "S_full_set": S,
                 "candidates_per_instance": S * 100 * spec.n_fit,
                 "background_rows_with_boundary_ties": int(spec.boundary_ties(d["background"]).sum())}
        eng.shap_values(X_exp[:64], nsamples=a.nsamples, l1_reg=False)      # plans uploaded, kernels loaded
        t0 = time.perf_counter()
        eng.shap_values(X_exp, nsamples=a.nsamples, l1_reg=False)
        wall = time.perf_counter() - t0
        tm = eng.last_timings_ms()
        entry.update({"total_ms": tm["total"], "explain_stage_ms": tm["coalitions"],
                      "instances_per_s": a.n / (tm["total"] * 1e-3), "wall_s": wall,
                      "general": eng.last_path()["general"]})
        print(name, entry, flush=True)
        # CPU figure: the oracle with the real scikit-learn method on the engine's plans
        orc = KernelExplainerOracle(fn, ODense(d["background"], d["group_names"], d["groups"]), link="identity")
        t0 = time.perf_counter()
        for i in range(a.oracle_instances):
            plan = eng.shared_plan(int(M[i]), a.nsamples)
            orc.explain(X_exp[i:i + 1], plan=(plan.dense(), plan.weights), nsamples=a.nsamples, l1_reg=False)
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
