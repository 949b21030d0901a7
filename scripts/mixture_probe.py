"""Times the mixture head (``sum_k pi_k h(z_k)``, DESIGN.md §5.0.10) on its shared-plan route (one pass of the member
head's coalition kernel per member) against K times the single-member head's shared-plan stage, measured in the same run,
and against the mixture's CUDA-core kernel (``kernel='simt'``).

For each case: the explain stage (the engine's CUDA events: coalition kernels + solve) and the device-resident step
(``explain_device`` replayed as a CUDA graph, host clock around a synchronised batch of calls), and the largest difference
of phi between the two routes relative to each instance's largest |phi|.  Shapes: the bench shape (Adult-like: 12 groups,
N = 100, S = 2048, 2560 instances) and BASELINE configs[2] (64 features, N = 512, S = 4096).  Models: binary members
K = 5 and K = 10, one-vs-rest members K = 5 over C = 3 classes.  Prints the GPU name, power limit and SM clock with the
numbers.  Needs an H100; there is no CPU fallback.

    python scripts/mixture_probe.py [--reps 10] [--n 2560]
"""
import argparse
import json

import numpy as np

from multiclass_probe import gpu_info, time_route


def _engine(W, b, bg, activation, kernel, **kw):
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.predictors import LinearModelSpec
    return GpuKernelExplainer(LinearModelSpec(W, b, activation, **kw), bg, link="logit", seed=1, kernel=kernel)


def _run(row, make, X, ns, reps, prefix=""):
    try:
        eng = make()
        phi, row[prefix + "stage_ms"], row[prefix + "step_ms"], path = time_route(eng, X, ns, reps)
        row[prefix + "path"] = path["shared"] + "/" + path["general"]
        eng.close()
        return phi
    except Exception as e:
        row[prefix + "error"] = str(e)[:120]
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--n", type=int, default=2560)
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}))
    shapes = [("bench", 12, 100, 2048), ("configs2", 64, 512, 4096)]
    models = [("binary_logistic", 1, 5), ("binary_logistic", 1, 10), ("ovr", 3, 5)]
    for name, G, N, ns in shapes:
        rng = np.random.default_rng(G)
        bg, X = rng.standard_normal((N, G)), rng.standard_normal((args.n, G))
        single = {}
        for member, Rm in (("binary_logistic", 1), ("ovr", 3)):
            W, b = rng.normal(0, 2.0 / np.sqrt(G), (Rm, G)), rng.normal(0, 0.5, Rm)
            row = {"shape": name, "G": G, "N": N, "S": ns, "n": args.n, "model": f"single {member}"}
            # the binary head's default route is the fused kernel; the unfused kernel is what a binary member's pass runs
            opts = [("fused", 0)] if member == "binary_logistic" else []

            def make(W=W, b=b, member=member, opts=opts):
                eng = _engine(W, b, bg, member, "auto")
                for o, v in opts:
                    eng.set_option(o, v)
                return eng
            _run(row, make, X, ns, args.reps)
            single[member] = row.get("stage_ms")
            print(json.dumps(row), flush=True)
        for member, Rm, K in models:
            W, b = rng.normal(0, 2.0 / np.sqrt(G), (K * Rm, G)), rng.normal(0, 0.5, K * Rm)
            pi = rng.uniform(0.2, 1.0, K)
            pi = pi / pi.sum()
            row = {"shape": name, "G": G, "N": N, "S": ns, "n": args.n, "model": f"mixture {member}", "K": K, "R_m": Rm}
            phi = _run(row, lambda: _engine(W, b, bg, "mixture", "auto", pi=pi, member=member), X, ns, args.reps)
            if phi is not None:
                row["M_inst_per_s"] = args.n / row["step_ms"] / 1e3
                if single.get(member):
                    row["K_x_single_stage_ms"] = K * single[member]
                    row["ratio"] = row["stage_ms"] / row["K_x_single_stage_ms"]
            old = _run(row, lambda: _engine(W, b, bg, "mixture", "simt", pi=pi, member=member), X, ns,
                       max(2, args.reps // 5), prefix="simt_")
            if phi is not None and old is not None:
                scale = np.maximum(np.abs(old).max(axis=-1, keepdims=True), 1e-12)
                row["max_rel_diff_vs_simt"] = float((np.abs(phi - old) / scale).max())
            print(json.dumps(row), flush=True)
    print(json.dumps({"gpu_after": gpu_info()}))


if __name__ == "__main__":
    main()
