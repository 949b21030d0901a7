"""Throughput of the tree route (DESIGN.md §5.0.11) on the Adult-shaped problem: 2560 instances, a 100-row background,
12 groups over 49 columns, nsamples 2048, for three tree models fitted to the problem's labels:

  GradientBoostingClassifier()                          100 trees, depth 3
  HistGradientBoostingClassifier()                      100 iterations, up to 31 leaves
  RandomForestClassifier(n_estimators=100, max_depth=10)

Per model and l1_reg (False, 'auto'): instances/s from the engine's device events (stage 1 to the end of the solve) and
the explain stage's time, the node-step bound per instance computed from shapes (S N sum_t depth_t: every (coalition,
background row, tree) walked to its leaf, before the divergence reduction), and, as the CPU figure, the oracle calling the
real scikit-learn model on the masked batch for a few instances.  The card name, power limit and SM clock are read in the
same run.  Prints one JSON document; ``--out`` also writes it to a file.

    python scripts/tree_probe.py [--n 2560] [--oracle-instances 2] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    info = {}
    try:
        import torch
        info["name"] = torch.cuda.get_device_name(0)
    except Exception:                          # pragma: no cover
        pass
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=20)
        name, plim, sm, smax = [s.strip() for s in q.stdout.strip().split(",")]
        info.update(name=name, power_limit_w=float(plim), sm_clock_mhz=float(sm), sm_clock_max_mhz=float(smax))
    except Exception as e:                     # pragma: no cover
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def depth_sum(spec):
    """sum over trees of the deepest leaf's depth."""
    depth = np.zeros(spec.n_nodes, dtype=np.int64)
    for nd in range(spec.n_nodes):             # children follow their parent
        if spec.feature[nd] >= 0:
            depth[spec.left[nd]] = depth[nd] + 1
            depth[spec.right[nd]] = depth[nd] + 1
    roots = list(spec.roots) + [spec.n_nodes]
    return int(sum(depth[roots[k]:roots[k + 1]].max() for k in range(spec.n_trees)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2560)
    ap.add_argument("--nsamples", type=int, default=2048)
    ap.add_argument("--oracle-instances", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from sklearn.ensemble import GradientBoostingClassifier, HistGradientBoostingClassifier, RandomForestClassifier

    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.trees import extract_tree_spec
    from oracle.shap_kernel_oracle import DenseData as ODense, KernelExplainerOracle

    d = adult_like(n_explain=a.n, n_background=100, seed=0)
    X_all = np.concatenate([d["background"], d["X_explain"]])
    y = d["predictor"].predict(X_all)
    models = {
        "GradientBoostingClassifier()": GradientBoostingClassifier(random_state=0),
        "HistGradientBoostingClassifier()": HistGradientBoostingClassifier(random_state=0),
        "RandomForestClassifier(n_estimators=100, max_depth=10)": RandomForestClassifier(100, max_depth=10, random_state=0),
    }
    result = {"card": card(), "n": a.n, "N": 100, "groups": len(d["groups"]), "columns": X_all.shape[1],
              "nsamples": a.nsamples, "models": {}}
    data = DenseData(d["background"], d["group_names"], d["groups"])
    for name, m in models.items():
        m.fit(X_all, y)
        spec = extract_tree_spec(m.predict_proba)
        eng = GpuKernelExplainer(m.predict_proba, data, link="logit", seed=0)
        M, _ = eng.varying(d["X_explain"])
        S = int(eng.shared_plan(int(M.max()), a.nsamples).S)
        entry = {"trees": spec.n_trees, "nodes": spec.n_nodes, "depth_sum": depth_sum(spec), "S_full_set": S,
                 "node_steps_bound_per_instance": S * 100 * depth_sum(spec), "runs": {}}
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
        orc = KernelExplainerOracle(m.predict_proba, ODense(d["background"], d["group_names"], d["groups"]), link="logit")
        t0 = time.perf_counter()
        for i in range(a.oracle_instances):
            Mi = int(M[i])
            plan = eng.shared_plan(Mi, a.nsamples)
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
