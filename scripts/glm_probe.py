"""Times the exp head (log-link GLM regressors, ``predict = exp(X w + b)``) next to the identity head.

For each shared-plan case: the explain stage (the engine's CUDA events: everything after stage 1) and the device-resident
step (``explain_device`` replayed as a CUDA graph, host clock around a synchronised batch of calls), at the bench shape
(Adult-like: 12 groups, N = 100, S = 2048, 2560 instances) and the BASELINE configs[2] shape (64 features, N = 512,
S = 4096).  Then one call whose instances have partial varying sets (the CUDA-core kernel) and the configs[4] shape with
per-instance plans (128 features, N = 512, S = 4096: the two-word CUDA-core kernel).  Prints the GPU name, power limit and
SM clock in the same run.  Needs an H100; there is no CPU fallback.

    python scripts/glm_probe.py [--reps 20] [--n 2560] [--n-wide 4096]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from multiclass_probe import time_route  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        return f"nvidia-smi unavailable: {e}"


def problem(G, N, n, seed):
    rng = np.random.default_rng(seed)
    return (rng.normal(0, 0.8 / np.sqrt(G), (1, G)), rng.normal(0, 0.3, 1), rng.standard_normal((N, G)),
            rng.standard_normal((n, G)))


def engine(W, b, bg, head, **kw):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.predictors import LinearModelSpec
    return GpuKernelExplainer(LinearModelSpec(W, b, head, scalar_out=True), bg, seed=1, **kw)


def host_call(eng, X, ns, reps):
    """Median device time of the explain stage and host time of a whole shap_values call."""
    eng.shap_values(X, nsamples=ns, l1_reg=False)
    stage, wall = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        eng.shap_values(X, nsamples=ns, l1_reg=False)
        wall.append((time.perf_counter() - t0) * 1e3)
        stage.append(eng.last_timings_ms()["coalitions"])
    return float(np.median(stage)), float(np.median(wall))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--n", type=int, default=2560)
    ap.add_argument("--n-wide", type=int, default=4096)
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name, G, N, ns in [("bench", 12, 100, 2048), ("configs2", 64, 512, 4096)]:
        W, b, bg, X = problem(G, N, args.n, seed=G)
        for head in ("exp", "identity"):
            eng = engine(W, b, bg, head)
            _, stage, step, path = time_route(eng, X, ns, args.reps)
            print(json.dumps({"shape": name, "G": G, "N": N, "S": ns, "n": args.n, "head": head, "stage_ms": stage,
                              "step_ms": step, "M_inst_per_s": args.n / step / 1e3,
                              "path": path["shared"] + "/" + path["solve"]}), flush=True)
            eng.close()
    # partial varying sets (groups 3 and 7 equal to a constant background column for every instance): CUDA-core kernel
    W, b, bg, X = problem(12, 100, args.n, seed=5)
    bg[:, [3, 7]] = 0.25
    X[:, [3, 7]] = 0.25
    for head in ("exp", "identity"):
        eng = engine(W, b, bg, head)
        stage, wall = host_call(eng, X, 2048, max(3, args.reps // 4))
        p = eng.last_path()
        print(json.dumps({"shape": "bench_partial", "G": 12, "M": 10, "N": 100, "S": 1022, "n": args.n, "head": head,
                          "stage_ms": stage, "host_call_ms": wall, "path": p["shared"] + "/" + p["general"]}), flush=True)
        eng.close()
    # configs[4] shape with per-instance plans (two-word rows)
    W, b, bg, X = problem(128, 512, args.n_wide, seed=128)
    for head in ("exp", "identity"):
        eng = engine(W, b, bg, head, plan_mode="per_instance")
        stage, wall = host_call(eng, X, 4096, 3)
        p = eng.last_path()
        print(json.dumps({"shape": "configs4_per_instance", "G": 128, "N": 512, "S": 4096, "n": args.n_wide, "head": head,
                          "stage_ms": stage, "host_call_ms": wall, "M_inst_per_s_stage": args.n_wide / stage / 1e3,
                          "path": p["general"]}), flush=True)
        eng.close()
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
