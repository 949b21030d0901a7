"""Times the one-vs-rest head on the shared-plan path against the CUDA-core (SIMT) kernel, with the softmax head at the
same shapes for comparison.

For each case: the explain stage (the engine's CUDA events: coalition kernels + solve), the device-resident step
(``explain_device`` replayed as a CUDA graph, host clock around a synchronised batch of calls) and the largest difference
of phi against the SIMT kernel, relative to each instance's largest |phi|.  Shapes: the bench shape (Adult-like: 12
groups, N = 100, S = 2048, 2560 instances) and BASELINE configs[2] (64 features, N = 512, S = 4096).  Prints the GPU
name, power limit and SM clock with the numbers.  Needs an H100; there is no CPU fallback.

    python scripts/ovr_probe.py [--reps 20] [--n 2560]
"""
import argparse
import json

import numpy as np

from multiclass_probe import engine, gpu_info, problem, time_route


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--n", type=int, default=2560)
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}))
    cases = [("bench", 12, 100, 2048, args.n), ("configs2", 64, 512, 4096, args.n)]
    for name, G, N, ns, n in cases:
        for C in (3, 4, 8):
            for head in ("ovr", "softmax"):
                W, b, bg, X = problem(G, N, n, C, seed=G + C)
                row = {"shape": name, "G": G, "N": N, "S": ns, "n": n, "head": head, "C": C}
                new = engine(W, b, bg, head, "logit", "auto")
                phi_new, row["stage_ms"], row["step_ms"], path = time_route(new, X, ns, args.reps)
                row["path"] = path["shared"] + "/" + path["solve"]
                row["M_inst_per_s"] = n / row["step_ms"] / 1e3
                new.close()
                if head == "ovr":
                    try:
                        old = engine(W, b, bg, head, "logit", "simt")
                        phi_old, row["simt_stage_ms"], row["simt_step_ms"], _ = time_route(old, X, ns,
                                                                                          max(2, args.reps // 10))
                        scale = np.maximum(np.abs(phi_old).max(axis=-1, keepdims=True), 1e-12)
                        row["max_rel_diff_vs_simt"] = float((np.abs(phi_new - phi_old) / scale).max())
                        old.close()
                    except Exception as e:
                        row["simt"] = f"does not run: {str(e)[:100]}"
                print(json.dumps(row), flush=True)
    print(json.dumps({"gpu_after": gpu_info()}))


if __name__ == "__main__":
    main()
