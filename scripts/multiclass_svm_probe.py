"""Throughput of the one-vs-one head of the kernel-machine route (DESIGN.md §5.0.22) on the Adult-shaped problem: 2560
instances, a 100-row background, 12 groups over 49 columns, nsamples 2048.  Labels are drawn from a softmax of a seeded
random linear score over the standardised columns, with 4 and 8 classes, and the binary calibrated SVC is run in the same
process as the yardstick (labels from the problem's predictor probabilities, as scripts/kernel_machine_probe.py draws
them):

  CalibratedClassifierCV(make_pipeline(StandardScaler(), SVC()), ensemble=False).predict_proba, logit link

Per model: instances/s from the engine's device events (stage 1 to the end of the solve), the support vector count, the
kernel evaluations per instance (S N n_sv) and per second, and, as the CPU figure, the oracle calling the real
scikit-learn method on the masked batch for a few instances.  The card name, power limit and SM clock are read in the
same run.  Prints one JSON document; ``--out`` also writes it to a file.

    python scripts/multiclass_svm_probe.py [--n 2560] [--fit-rows 3000] [--oracle-instances 1] [--repeats 3] [--out r.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.tree_probe import card  # noqa: E402


def softmax_labels(X, classes, seed):
    rng = np.random.default_rng(seed)
    Z = (X - X.mean(0)) / (X.std(0) + 1e-12) @ rng.normal(size=(X.shape[1], classes))
    p = np.exp(Z - Z.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    return np.array([rng.choice(classes, p=q) for q in p])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2560)
    ap.add_argument("--nsamples", type=int, default=2048)
    ap.add_argument("--fit-rows", type=int, default=3000)
    ap.add_argument("--oracle-instances", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from sklearn.calibration import CalibratedClassifierCV
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler
    from sklearn.svm import SVC

    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.kernel_machines import extract_kernel_machine_spec
    from oracle.shap_kernel_oracle import DenseData as ODense, KernelExplainerOracle

    d = adult_like(n_explain=max(a.n, a.fit_rows), n_background=100, seed=0)
    X_fit = d["X_explain"][:a.fit_rows]
    X_exp = d["X_explain"][:a.n]
    p = d["predictor"].predict_proba(X_fit)[:, 1]
    y2 = (np.random.default_rng(1).random(len(p)) < p).astype(int)
    labels = {"binary": y2, "4 classes": softmax_labels(X_fit, 4, 4), "8 classes": softmax_labels(X_fit, 8, 8)}
    result = {"card": card(), "n": a.n, "N": 100, "groups": len(d["groups"]), "columns": X_fit.shape[1],
              "nsamples": a.nsamples, "fit_rows": a.fit_rows, "repeats": a.repeats,
              "model": "CalibratedClassifierCV(make_pipeline(StandardScaler(), SVC()), ensemble=False).predict_proba",
              "link": "logit", "models": {}}
    data = DenseData(d["background"], d["group_names"], d["groups"])
    for name, y in labels.items():
        cal = CalibratedClassifierCV(make_pipeline(StandardScaler(), SVC()), ensemble=False).fit(X_fit, y)
        fn = cal.predict_proba
        spec = extract_kernel_machine_spec(fn)
        eng = GpuKernelExplainer(fn, data, link="logit", seed=0)
        M, _ = eng.varying(X_exp)
        S = int(eng.shared_plan(int(M.max()), a.nsamples).S)
        evals = S * 100 * spec.n_sv
        entry = {"classes": len(cal.classes_), "head": spec.head, "n_sv": spec.n_sv, "S_full_set": S,
                 "kernel_evaluations_per_instance": evals}
        eng.shap_values(X_exp[:64], nsamples=a.nsamples, l1_reg=False)      # plans uploaded, kernels loaded
        totals = []
        for _ in range(a.repeats):
            eng.shap_values(X_exp, nsamples=a.nsamples, l1_reg=False)
            totals.append(eng.last_timings_ms()["total"])
        best = min(totals)
        entry.update({"total_ms": totals, "instances_per_s": a.n / (best * 1e-3),
                      "kernel_evaluations_per_s": evals * a.n / (best * 1e-3), "general": eng.last_path()["general"]})
        print(name, entry, flush=True)
        orc = KernelExplainerOracle(fn, ODense(d["background"], d["group_names"], d["groups"]), link="logit")
        t0 = time.perf_counter()
        for i in range(a.oracle_instances):
            plan = eng.shared_plan(int(M[i]), a.nsamples)
            orc.explain(X_exp[i:i + 1], plan=(plan.dense(), plan.weights), nsamples=a.nsamples, l1_reg=False)
        entry["oracle_cpu_s_per_instance"] = (time.perf_counter() - t0) / a.oracle_instances
        result["models"][name] = entry
        eng.close()
    base = result["models"]["binary"]["kernel_evaluations_per_s"]
    for name, entry in result["models"].items():
        entry["kernel_evaluations_per_s_vs_binary"] = entry["kernel_evaluations_per_s"] / base
    text = json.dumps(result, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
