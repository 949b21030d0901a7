"""Throughput of the kernel-machine route (DESIGN.md §5.0.12) on the Adult-shaped problem: 2560 instances, a 100-row
background, 12 groups over 49 columns, nsamples 2048, for three kernel machines fitted to labels drawn from
the problem's predictor probabilities:

  make_pipeline(StandardScaler(), SVC())                                          decision_function, identity link
  CalibratedClassifierCV(make_pipeline(StandardScaler(), SVC()), ensemble=False)  predict_proba, logit link
  make_pipeline(StandardScaler(), SVR())                                          predict, identity link

Per model and l1_reg (False, 'auto'): instances/s from the engine's device events (stage 1 to the end of the solve) and
the explain stage's time, the support vector count and the kernel evaluations per instance (S N n_sv), and, as the CPU
figure, the oracle calling the real scikit-learn method on the masked batch for a few instances.  The card name, power
limit and SM clock are read in the same run.  Prints one JSON document; ``--out`` also writes it to a file.

    python scripts/kernel_machine_probe.py [--n 2560] [--fit-rows 3000] [--oracle-instances 2] [--out result.json]
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
    ap.add_argument("--fit-rows", type=int, default=3000)
    ap.add_argument("--oracle-instances", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from sklearn.calibration import CalibratedClassifierCV
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler
    from sklearn.svm import SVC, SVR

    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.kernel_machines import extract_kernel_machine_spec
    from oracle.shap_kernel_oracle import DenseData as ODense, KernelExplainerOracle

    d = adult_like(n_explain=max(a.n, a.fit_rows), n_background=100, seed=0)
    X_fit = d["X_explain"][:a.fit_rows]
    p = d["predictor"].predict_proba(X_fit)[:, 1]
    # labels drawn from the predictor's probabilities: its own predict() is a linear rule, on which a calibrated SVC
    # saturates (p1 == 1.0 in float64 for some rows, whose logit is infinite)
    y = (np.random.default_rng(1).random(len(p)) < p).astype(int)
    X_exp = d["X_explain"][:a.n]
    svc = make_pipeline(StandardScaler(), SVC()).fit(X_fit, y)
    cal = CalibratedClassifierCV(make_pipeline(StandardScaler(), SVC()), ensemble=False).fit(X_fit, y)
    svr = make_pipeline(StandardScaler(), SVR()).fit(X_fit, p)
    models = {
        "make_pipeline(StandardScaler(), SVC()).decision_function": (svc.decision_function, "identity"),
        "CalibratedClassifierCV(make_pipeline(StandardScaler(), SVC()), ensemble=False).predict_proba":
            (cal.predict_proba, "logit"),
        "make_pipeline(StandardScaler(), SVR()).predict": (svr.predict, "identity"),
    }
    result = {"card": card(), "n": a.n, "N": 100, "groups": len(d["groups"]), "columns": X_fit.shape[1],
              "nsamples": a.nsamples, "fit_rows": a.fit_rows, "models": {}}
    data = DenseData(d["background"], d["group_names"], d["groups"])
    for name, (fn, link) in models.items():
        spec = extract_kernel_machine_spec(fn)
        eng = GpuKernelExplainer(fn, data, link=link, seed=0)
        M, _ = eng.varying(X_exp)
        S = int(eng.shared_plan(int(M.max()), a.nsamples).S)
        entry = {"link": link, "n_sv": spec.n_sv, "S_full_set": S,
                 "kernel_evaluations_per_instance": S * 100 * spec.n_sv, "runs": {}}
        for l1 in (False, "auto"):
            eng.shap_values(X_exp[:64], nsamples=a.nsamples, l1_reg=l1)      # plans uploaded, kernels loaded
            t0 = time.perf_counter()
            eng.shap_values(X_exp, nsamples=a.nsamples, l1_reg=l1)
            wall = time.perf_counter() - t0
            tm = eng.last_timings_ms()
            path = eng.last_path()
            entry["runs"][str(l1)] = {"total_ms": tm["total"], "explain_stage_ms": tm["coalitions"],
                                      "instances_per_s": a.n / (tm["total"] * 1e-3), "wall_s": wall,
                                      "general": path["general"], "general_l1": path["general_l1"]}
            print(name, l1, entry["runs"][str(l1)], flush=True)
        # CPU figure: the oracle with the real scikit-learn method on the engine's plans
        orc = KernelExplainerOracle(fn, ODense(d["background"], d["group_names"], d["groups"]), link=link)
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
