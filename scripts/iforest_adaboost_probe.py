"""Throughput of the tree route (DESIGN.md §5.0.11, §5.0.18) for the anomaly head and SAMME AdaBoost on the Adult-shaped
problem: 2560 instances, a 100-row background, 12 groups over 49 columns, nsamples 2048, for two models with their
default settings:

  IsolationForest()        100 isolation trees of depth <= 8, decision_function, identity link
  AdaBoostClassifier()     50 stumps, predict_proba, logit link (fitted to the problem's labels)

Per model and l1_reg (False, 'auto'): instances/s from the engine's device events (stage 1 to the end of the solve) and
the explain stage's time, the node-step bound per instance computed from shapes (S N sum_t depth_t, before the
divergence reduction), and, as the CPU figure, the oracle calling the real scikit-learn model on the masked batch for a
few instances.  The card name, power limit and SM clock are read in the same run.  Prints one JSON document; ``--out``
also writes it to a file.

    python scripts/iforest_adaboost_probe.py [--n 2560] [--oracle-instances 2] [--out result.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from tree_probe import card, depth_sum  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2560)
    ap.add_argument("--nsamples", type=int, default=2048)
    ap.add_argument("--oracle-instances", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from sklearn.ensemble import AdaBoostClassifier, IsolationForest

    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.trees import extract_tree_spec
    from oracle.shap_kernel_oracle import DenseData as ODense, KernelExplainerOracle

    d = adult_like(n_explain=a.n, n_background=100, seed=0)
    X_all = np.concatenate([d["background"], d["X_explain"]])
    y = d["predictor"].predict(X_all)
    iso = IsolationForest(random_state=0).fit(X_all)
    ada = AdaBoostClassifier(random_state=0).fit(X_all, y)
    models = {"IsolationForest().decision_function": (iso.decision_function, "identity"),
              "AdaBoostClassifier().predict_proba": (ada.predict_proba, "logit")}
    result = {"card": card(), "n": a.n, "N": 100, "groups": len(d["groups"]), "columns": X_all.shape[1],
              "nsamples": a.nsamples, "models": {}}
    data = DenseData(d["background"], d["group_names"], d["groups"])
    for name, (fn, link) in models.items():
        spec = extract_tree_spec(fn)
        eng = GpuKernelExplainer(fn, data, link=link, seed=0)
        M, _ = eng.varying(d["X_explain"])
        S = int(eng.shared_plan(int(M.max()), a.nsamples).S)
        entry = {"link": link, "trees": spec.n_trees, "nodes": spec.n_nodes, "depth_sum": depth_sum(spec),
                 "S_full_set": S, "node_steps_bound_per_instance": S * 100 * depth_sum(spec), "runs": {}}
        for l1 in (False, "auto"):
            eng.shap_values(d["X_explain"][:64], nsamples=a.nsamples, l1_reg=l1)      # plans uploaded, kernels loaded
            t0 = time.perf_counter()
            eng.shap_values(d["X_explain"], nsamples=a.nsamples, l1_reg=l1)
            wall = time.perf_counter() - t0
            tm = eng.last_timings_ms()
            path = eng.last_path()
            entry["runs"][str(l1)] = {"total_ms": tm["total"], "explain_stage_ms": tm["coalitions"],
                                      "instances_per_s": a.n / (tm["total"] * 1e-3), "wall_s": wall,
                                      "general": path["general"], "general_l1": path["general_l1"]}
            print(name, l1, entry["runs"][str(l1)], flush=True)
        # CPU figure: the oracle with the real scikit-learn model on the engine's plans
        orc = KernelExplainerOracle(fn, ODense(d["background"], d["group_names"], d["groups"]), link=link)
        t0 = time.perf_counter()
        for i in range(a.oracle_instances):
            plan = eng.shared_plan(int(M[i]), a.nsamples)
            orc.explain(d["X_explain"][i:i + 1], plan=(plan.dense(), plan.weights), nsamples=a.nsamples, l1_reg=False)
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
