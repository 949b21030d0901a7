"""Times pipelines explained in raw feature space (column maps, DESIGN.md §5.0.9) next to the same model explained on
its encoded columns.

Two shapes, each as an encoded linear model with one group per categorical block and as the equivalent scikit-learn
pipeline over the raw columns (``datasets.raw_space_pipeline``), with the same seed and shared plans:
* the bench shape: Adult-like, 12 groups (4 standardised numeric columns + 8 one-hot blocks, ``drop='first'``), N = 100,
  S = 2048, 2560 instances;
* a wide categorical shape: BASELINE configs[3] decoded to 64 raw columns of 16 levels (``OneHotEncoder``), N = 256,
  S = 2048.
For each: stage 1 (``prep_kernel``: the engine's CUDA events around it, median over host calls), the explain stage after
it, and the device-resident step (``explain_device`` replayed as a CUDA graph, host clock around a synchronised batch).
Also checks that both readings give the same phi (max |d| / max |phi|).  Prints the GPU name, power limit and SM clock in
the same run.  Needs an H100; there is no CPU fallback.

    python scripts/pipeline_probe.py [--reps 20] [--n 2560]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from glm_probe import gpu_info  # noqa: E402
from multiclass_probe import time_route  # noqa: E402


def stage1_ms(eng, X, ns, reps):
    eng.shap_values(X, nsamples=ns, l1_reg=False)
    t = []
    for _ in range(reps):
        eng.shap_values(X, nsamples=ns, l1_reg=False)
        t.append(eng.last_timings_ms()["prepare"])
    return float(np.median(t))


def shapes(n):
    from distributedkernelshap_b200.datasets import (ADULT_ONEHOT_WIDTHS, adult_like, decode_onehot_blocks,
                                                     raw_space_pipeline, wide_onehot)
    d = adult_like(n_explain=n)
    raw_bg, raw_X = (decode_onehot_blocks(A, 4, ADULT_ONEHOT_WIDTHS, True) for A in (d["background"], d["X_explain"]))
    pipe = raw_space_pipeline(d["predictor"], np.vstack([raw_bg, raw_X]), 4, ADULT_ONEHOT_WIDTHS, True)
    yield ("bench", 2048, (d["predictor"].predict_proba, d["background"], d["X_explain"], d["groups"]),
           (pipe.predict_proba, raw_bg, raw_X, None))
    w = wide_onehot(n)
    widths = [16] * 64
    raw_bg, raw_X = (decode_onehot_blocks(A, 0, widths, False) for A in (w["background"], w["X_explain"]))
    pipe = raw_space_pipeline(w["predictor"], np.vstack([raw_bg, raw_X]), 0, widths, False)
    yield ("configs3_raw64", 2048, (w["predictor"].predict_proba, w["background"], w["X_explain"], w["groups"]),
           (pipe.predict_proba, raw_bg, raw_X, None))


def main():
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--n", type=int, default=2560)
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name, ns, encoded, raw in shapes(args.n):
        phis = {}
        for reading, (f, bg, X, groups) in (("encoded", encoded), ("raw_pipeline", raw)):
            data = bg if groups is None else DenseData(bg, [f"g{k}" for k in range(len(groups))], groups)
            eng = GpuKernelExplainer(f, data, link="logit", seed=0)
            prep = stage1_ms(eng, X, ns, args.reps)
            phi, stage, step, path = time_route(eng, X, ns, args.reps)
            phis[reading] = phi
            print(json.dumps({"shape": name, "reading": reading, "D": X.shape[1], "G": eng.data.groups_size,
                              "N": bg.shape[0], "S": ns, "n": X.shape[0], "stage1_ms": prep, "explain_stage_ms": stage,
                              "step_ms": step, "M_inst_per_s": X.shape[0] / step / 1e3,
                              "path": path["shared"] + "/" + path["solve"]}), flush=True)
            eng.close()
        a, b = phis["encoded"], phis["raw_pipeline"]
        print(json.dumps({"shape": name, "max_rel_diff": float(np.abs(a - b).max() / np.abs(a).max())}), flush=True)
    print(json.dumps({"gpu_after": gpu_info(), "time": time.strftime("%Y-%m-%d %H:%M:%S")}), flush=True)


if __name__ == "__main__":
    main()
