"""Times per-instance coalition plans of 128 groups (two-word rows) at BASELINE configs[4]'s shape, device-resident.

Shape: ``datasets.dense_tabular(n, 128, 512)`` (M = 128, N = 512, binary-logistic head, logit link), nsamples 4096.  For
``plan_mode='per_instance'`` and, in the same run, ``plan_mode='shared'``: the plans are built by a small host call, then
``explain_device`` over all n rows on a user stream -- ``--warmup`` calls, then ``--reps`` calls each timed with CUDA
events after a 256 MB L2 flush (the device-resident call replays as a CUDA graph from the second call on).  A separate
pass under ``torch.profiler`` (graph replay off) splits the device time by kernel: stage 1 (prep_kernel), the plan
sampler, the per-instance inversion and the coalition kernel of each mode.  Prints one JSON line per mode and the GPU
name, power limit and SM clock read in the same run.  Needs an H100; there is no CPU fallback.

    python scripts/per_instance_wide_probe.py [--n 16384] [--reps 5] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from multiclass_probe import gpu_info  # noqa: E402

NSAMPLES = 4096
KERNELS = {"prep": "prep_kernel", "sampler": "sample_plans_kernel", "invert": "factor_wide_plans_kernel",
           "explain_wide": "explain_wide_instance_kernel"}


def kernel_split(eng, X_dev, n, phi, stream):
    """Device time per kernel (ms, one call) from torch.profiler, graph replay off."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    eng.set_option("graph", 0)
    with torch.cuda.stream(stream):
        eng.explain_device(X_dev.data_ptr(), n, phi.data_ptr(), nsamples=NSAMPLES)
        eng.check_status()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.explain_device(X_dev.data_ptr(), n, phi.data_ptr(), nsamples=NSAMPLES)
            eng.check_status()
    eng.set_option("graph", 1)
    split, total = {}, 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        ms = t / 1e3
        if ms <= 0:
            continue
        total += ms
        tag = next((k for k, v in KERNELS.items() if v in ev.key), None)
        if tag is None:
            tag = "other:" + ev.key[:60]
        split[tag] = split.get(tag, 0.0) + ms
    split["sum"] = total
    return split


def measure(mode, d, n, reps, warmup):
    import torch
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    eng = GpuKernelExplainer(d["predictor"].predict_proba, d["background"], link="logit", seed=0, plan_mode=mode)
    eng.shap_values(d["X_explain"][:8], nsamples=NSAMPLES, l1_reg=False)        # plans of M = 128 built and uploaded
    stream = torch.cuda.Stream()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    with torch.cuda.stream(stream):
        eng.set_stream(stream.cuda_stream)
        eng.lib.dks_set_row_offset(eng._ctx, 0)
        X_dev = torch.from_numpy(d["X_explain"]).cuda()
        phi = torch.zeros((2, n, 128), dtype=torch.float64, device="cuda")
        for _ in range(warmup):
            eng.explain_device(X_dev.data_ptr(), n, phi.data_ptr(), nsamples=NSAMPLES)
        eng.check_status()
        times = []
        for _ in range(reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            eng.explain_device(X_dev.data_ptr(), n, phi.data_ptr(), nsamples=NSAMPLES)
            e1.record(stream)
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        eng.check_status()
        path = eng.last_path()
    finite = bool(torch.isfinite(phi).all().item())
    split = kernel_split(eng, X_dev, n, phi, stream)
    eng.set_stream(0)
    med = float(np.median(times))
    return {"plan_mode": mode, "n": n, "M": 128, "N": 512, "nsamples": NSAMPLES, "ms_median": med,
            "ms_all": [round(t, 3) for t in times], "instances_per_s": n / (med / 1e3), "graph_launches": eng.graph_launches(),
            "path": {k: path[k] for k in ("shared", "solve", "general")}, "kernel_ms": split, "phi_finite": finite}


def main():
    from distributedkernelshap_b200.datasets import dense_tabular
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    d = dense_tabular(args.n, 128, 512, seed=4)
    rows = [{"gpu": gpu_info()}]
    print(json.dumps(rows[0]), flush=True)
    for mode in ("per_instance", "shared"):
        rows.append(measure(mode, d, args.n, args.reps, args.warmup))
        print(json.dumps(rows[-1]), flush=True)
    rows.append({"gpu_after": gpu_info()})
    print(json.dumps(rows[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
