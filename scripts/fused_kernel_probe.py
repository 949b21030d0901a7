#!/usr/bin/env python
"""Time the fused shared-plan coalition kernel on its own, on the bench.py workload, and sweep its warps per CTA and
the number of instances.

  python scripts/fused_kernel_probe.py [--launches 200] [--steps 50] [--warps 4,6,8,10,12] [--n 64,256,2560]
                                      [--fused-table 1] [--out FILE]

The workload is bench.py's: 2560 Adult-shaped instances, 12 groups, 100 background rows, nsamples = 2048, shared plans.
For the engine's default configuration and for every ``fused_warps`` value of the sweep it reports

  kernel_ms   the coalition stage (explain_shared_fused_kernel and its finish_fused_kernel) timed by the engine's own CUDA events
              (``last_timings_ms()["coalitions"]``, plain launches: ``graph`` 0), mean / min / max over ``--launches``
              launches, L2 flushed before each;
  step_ms     a whole device-resident step (CUDA graph replay, as bench.py's ``value`` times it), mean over ``--steps``,
              L2 flushed before each;
  path        what the engine reports it launched (``last_path()``).

The ``--n`` sweep explains the first n instances of the workload with the default configuration (few instances leave
most of the streaming warps with one or two instances each).

``--fused-table 0`` runs everything on the exact loop over the background instead of the plan's link table.

One JSON line on stdout, with the GPU name, its power limit and the SM clock sampled while the kernels ran.
"""
import argparse
import json
import os
import statistics
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

import bench  # noqa: E402  (the workload, NVML power limit and clock sampler of the benchmark)


def measure(engine, X_dev, n, phi_dev, flush, stream, launches, steps, warmup=5):
    import torch
    kernel = []
    engine.set_option("graph", 0)
    for k in range(warmup + launches):
        flush.zero_()
        engine.explain_device(X_dev.data_ptr(), n, phi_dev.data_ptr(), nsamples=bench.NSAMPLES)
        t = engine.last_timings_ms()["coalitions"]       # synchronises the engine's stream
        if k >= warmup:
            kernel.append(t)
    path = engine.last_path()
    engine.set_option("graph", 1)
    for _ in range(warmup):
        flush.zero_()
        engine.explain_device(X_dev.data_ptr(), n, phi_dev.data_ptr(), nsamples=bench.NSAMPLES)
    starts = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
    ends = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
    torch.cuda.synchronize()
    for k in range(steps):
        flush.zero_()
        starts[k].record(stream)
        engine.explain_device(X_dev.data_ptr(), n, phi_dev.data_ptr(), nsamples=bench.NSAMPLES)
        ends[k].record(stream)
    torch.cuda.synchronize()
    engine.check_status()
    step = [s.elapsed_time(e) for s, e in zip(starts, ends)]
    return {"kernel_ms": statistics.mean(kernel), "kernel_ms_min": min(kernel), "kernel_ms_max": max(kernel),
            "step_ms": statistics.mean(step), "kernel_share_of_step": statistics.mean(kernel) / statistics.mean(step),
            "path": {k: path[k] for k in ("shared", "warps", "grid", "fused_B", "fused_NI")} |
                    ({"cta_warps": path["cta_warps"]} if "cta_warps" in path else {}) |
                    ({"fused_table": path["fused_table"]} if "fused_table" in path else {})}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warps", default="4,6,8,10,12", help="fused_warps values to sweep (comma separated)")
    ap.add_argument("--n", default="64,256,2560", help="instance counts of the mapping sweep (comma separated)")
    ap.add_argument("--fused-table", type=int, default=1, help="the engine's fused_table option (0: exact loop only)")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("the probe needs a CUDA device")
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap

    wl = bench.workload()
    X = np.ascontiguousarray(wl["X_explain"], dtype=np.float64)
    n = X.shape[0]
    explainer = KernelShap(wl["predictor"].predict_proba, link="logit", feature_names=wl["group_names"], seed=0)
    explainer.fit(wl["data"]["background"]["X"]["preprocessed"], group_names=wl["group_names"], groups=wl["groups"])
    engine = explainer._explainer
    engine.get_explanation(X, nsamples=bench.NSAMPLES, l1_reg=False, silent=True)      # shared plans built + uploaded
    G, C = engine.data.groups_size, engine.D
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    engine.set_stream(stream.cuda_stream)
    engine.set_option("fused_table", args.fused_table)
    X_dev = torch.from_numpy(X).cuda()
    phi_dev = torch.empty((C, n, G), dtype=torch.float64, device="cuda")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")

    sampler = bench.ClockSampler(0)
    sampler.start()
    default = measure(engine, X_dev, n, phi_dev, flush, stream, args.launches, args.steps)
    phi_default = phi_dev.cpu().numpy()
    sweep = {}
    for w in [int(v) for v in args.warps.split(",") if v]:
        engine.set_option("fused_warps", w)
        sweep[str(w)] = measure(engine, X_dev, n, phi_dev, flush, stream, args.launches, args.steps)
        sweep[str(w)]["phi_equal_to_default"] = bool(np.array_equal(phi_dev.cpu().numpy(), phi_default))
    engine.set_option("fused_warps", 0)
    by_n = {}
    for m in [int(v) for v in args.n.split(",") if v]:
        m = min(m, n)
        phi_m = torch.empty((C, m, G), dtype=torch.float64, device="cuda")
        by_n[str(m)] = measure(engine, X_dev[:m], m, phi_m, flush, stream, args.launches, args.steps)
        by_n[str(m)]["phi_equal_to_default"] = bool(np.array_equal(phi_m.cpu().numpy(), phi_default[:, :m]))
    clocks = sampler.stop()
    engine.close()

    props = torch.cuda.get_device_properties(0)
    line = {"probe": "fused shared-plan kernel", "fused_table": args.fused_table, "workload": "bench.py: 2560 Adult-shaped instances, G = 12, N = 100, "
            "nsamples = 2048, shared plans", "launches": args.launches, "steps": args.steps,
            "default": default, "fused_warps_sweep": sweep, "n_sweep": by_n,
            "clocks": {"sm_mhz": clocks["sm_mhz"], "sm_max_mhz": clocks["sm_max_mhz"], "reasons": clocks["reasons"],
                       "samples": clocks["samples"]},
            "gpu": {"name": props.name, "sm_count": props.multi_processor_count, "power_limit_w": bench._power_limit_w(0)}}
    text = json.dumps(line)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
