"""Times the softmax and identity heads on the shared-plan path against the CUDA-core (SIMT) kernel.

For each case: the explain stage (the engine's CUDA events: coalition kernels + solve), the device-resident step
(``explain_device`` replayed as a CUDA graph, host clock around a synchronised batch of calls) and the agreement of phi
between the two routes; plus one host call with l1_reg='auto'.  Shapes: the bench shape (Adult-like: 12 groups, N = 100,
S = 2048, 2560 instances) and BASELINE configs[2] (64 features, N = 512, S = 4096).  Prints the GPU name and power limit
with the numbers.  Needs an H100; there is no CPU fallback.

    python scripts/multiclass_probe.py [--reps 20] [--n 2560]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        out = f"nvidia-smi unavailable: {e}"
    return out


def problem(G, N, n, C, seed=0):
    rng = np.random.default_rng(seed)
    W = rng.normal(0, 2.0 / np.sqrt(G), (C, G))
    b = rng.normal(0, 0.5, C)
    return W, b, rng.standard_normal((N, G)), rng.standard_normal((n, G))


def engine(W, b, bg, head, link, kernel):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.predictors import LinearModelSpec
    return GpuKernelExplainer(LinearModelSpec(W, b, head), bg, link=link, seed=1, kernel=kernel)


def time_route(eng, X, ns, reps):
    import torch
    phi = eng.shap_values(X, nsamples=ns, l1_reg=False)
    phi = np.stack(phi if isinstance(phi, list) else [phi])
    stage = []
    for _ in range(reps):
        eng.shap_values(X, nsamples=ns, l1_reg=False)
        stage.append(eng.last_timings_ms()["coalitions"])
    path = eng.last_path()
    n = X.shape[0]
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        X_dev = torch.from_numpy(X).cuda()
        out = torch.zeros((phi.shape[0], n, X.shape[1]), dtype=torch.float64, device="cuda")
        for _ in range(3):
            eng.explain_device(X_dev.data_ptr(), n, out.data_ptr(), nsamples=ns)
        stream.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            eng.explain_device(X_dev.data_ptr(), n, out.data_ptr(), nsamples=ns)
        stream.synchronize()
        step = (time.perf_counter() - t0) / reps * 1e3
        eng.check_status()
    eng.set_stream(0)
    return phi, float(np.median(stage)), step, path


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--n", type=int, default=2560)
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}))
    cases = [("bench", 12, 100, 2048, args.n), ("configs2", 64, 512, 4096, args.n)]
    heads = [("softmax", 3), ("softmax", 4), ("softmax", 8), ("identity", 1)]
    for name, G, N, ns, n in cases:
        for head, C in heads:
            W, b, bg, X = problem(G, N, n, C, seed=G + C)
            link = "logit" if head == "softmax" else "identity"
            row = {"shape": name, "G": G, "N": N, "S": ns, "n": n, "head": head, "C": C}
            new = engine(W, b, bg, head, link, "auto")
            phi_new, row["stage_ms"], row["step_ms"], path = time_route(new, X, ns, args.reps)
            row["path"] = path["shared"] + "/" + path["solve"]
            row["M_inst_per_s"] = n / row["step_ms"] / 1e3
            try:
                old = engine(W, b, bg, head, link, "simt")
                phi_old, row["simt_stage_ms"], row["simt_step_ms"], _ = time_route(old, X, ns, max(2, args.reps // 10))
                scale = np.maximum(np.abs(phi_old).max(axis=-1, keepdims=True), 1e-12)
                row["max_rel_diff_vs_simt"] = float((np.abs(phi_new - phi_old) / scale).max())
            except Exception as e:
                row["simt"] = f"does not run: {str(e)[:100]}"
            print(json.dumps(row), flush=True)
            new.close()
    # one host call with the default l1_reg='auto' (64 features at S = 4096 of 2^64: the selection runs)
    W, b, bg, X = problem(64, 512, 256, 3, seed=7)
    eng = engine(W, b, bg, "softmax", "logit", "auto")
    eng.shap_values(X, nsamples=4096)
    t0 = time.perf_counter()
    eng.shap_values(X, nsamples=4096)
    print(json.dumps({"l1_auto_host_call": {"G": 64, "N": 512, "n": 256, "C": 3, "ms": (time.perf_counter() - t0) * 1e3,
                                            "path": eng.last_path()["shared"] + "/" + eng.last_path()["solve"]}}))


if __name__ == "__main__":
    main()
