"""Times l1 feature selection for instances whose varying set is partial (l1_reg='auto', the reference's default) against
the plain constrained WLS (l1_reg=False) on the same instances.

Cases: ungrouped Adult-like data (49 singleton groups, 100 background rows, 2560 instances, default kwargs: every instance
has 47 or 48 varying groups) and a BASELINE configs[2]-shaped problem (64 features, N = 512, two background columns made
constant and half the rows equal to them: M = 62 and 64).  For each: the host time of ``shap_values`` (the median of
``--reps`` synchronous calls after a warm-up), the split of the general list's selection from the engine's CUDA events
(the CUDA-core kernel that forms the moments, and the LARS kernel), the explain stage, the paths taken and the M
histogram.  Prints the GPU name, power limit and SM clock in the same run.  Needs an H100; there is no CPU fallback.

    python scripts/l1_partial_probe.py [--reps 5] [--n-configs2 512]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from multiclass_probe import gpu_info  # noqa: E402


def run(eng, X, l1_reg, reps):
    eng.shap_values(X, l1_reg=l1_reg)                    # plans, l1 tables and modules warm
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        phi = eng.shap_values(X, l1_reg=l1_reg)
        times.append((time.perf_counter() - t0) * 1e3)
    row = {"l1_reg": l1_reg, "host_ms": float(np.median(times)), "stage_ms": eng.last_timings_ms()["coalitions"],
           "path": eng.last_path()}
    if row["path"]["general_l1"]:
        row["general_l1_ms"] = eng.general_l1_timings_ms()
    return phi, row


def main():
    from distributedkernelshap_b200.datasets import adult_like, dense_tabular
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n-configs2", type=int, default=512)
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    d = adult_like(2560, 100, seed=0)
    c2 = dense_tabular(n=args.n_configs2, n_features=64, n_background=512, seed=0)
    c2["background"][:, [5, 40]] = 0.5
    c2["X_explain"][: args.n_configs2 // 2, [5, 40]] = 0.5
    for name, predictor, bg, X in [("adult_like_ungrouped", d["predictor"], d["background"], d["X_explain"]),
                                   ("configs2_partial", c2["predictor"], c2["background"], c2["X_explain"])]:
        eng = GpuKernelExplainer(predictor.predict_proba, bg, link="logit", seed=0)
        hist = {}
        M, _ = eng.varying(X)
        for m in M.tolist():
            hist[m] = hist.get(m, 0) + 1
        for l1_reg in ("auto", False):
            _, row = run(eng, X, l1_reg, args.reps)
            print(json.dumps({"case": name, "n": X.shape[0], "G": X.shape[1], "N": bg.shape[0], "M_hist": hist, **row}),
                  flush=True)
        eng.close()
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
