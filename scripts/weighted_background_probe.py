#!/usr/bin/env python
"""Cost of weighted backgrounds (k-means centroids weighted by cluster size) on the shared-plan kernels, against uniform
backgrounds and against the general kernels that took weighted backgrounds before.

  python scripts/weighted_background_probe.py [--launches 20] [--steps 20] [--out FILE]

Shapes:
  bench     bench.py's workload: 2560 Adult-shaped instances, 12 groups, 100 background rows, nsamples = 2048;
  configs2  BASELINE.json configs[2]: 64 ungrouped features, 512 background rows, nsamples = 4096, 4096 instances.

Variants per shape: ``uniform`` (no weights), ``weighted`` (k-means-like integer cluster counts, max / min = 400, one of
them 0: the weighted shared-plan kernels) and ``weighted_old_route`` (the same weights forced onto the kernel that ran
them before: ``kernel="tcgen05"`` for bench, ``"simt"`` for configs2).  Each reports

  stage_ms  the explain stage (coalition kernels + solve) timed by the engine's own CUDA events
            (``last_timings_ms()["coalitions"]``), plain launches, mean over ``--launches``, L2 flushed before each;
  step_ms   a whole device-resident step (CUDA graph replay, as bench.py's ``value`` times it), mean over ``--steps``;
  path      what the engine reports it launched (``last_path()``);
and for configs2 ``l1_auto_ms``: one host-API call on 2048 instances with the reference's default ``l1_reg='auto'``
(median of three; the old route refuses it).

One JSON line on stdout, with the GPU name, its power limit and the SM clock sampled while the kernels ran.
"""
import argparse
import json
import os
import statistics
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

import bench  # noqa: E402  (the workload, NVML power limit and clock sampler of the benchmark)


def kmeans_like_counts(N, seed=0):
    """Integer cluster counts spread over more than two decades, one of them 0 (what k-means on skewed data gives)."""
    rng = np.random.default_rng(seed)
    w = np.round(np.exp(rng.uniform(0.0, np.log(400.0), size=N)))
    w[0], w[1], w[2] = 1.0, 400.0, 0.0
    return w


def measure(engine, X_dev, n, phi_dev, flush, stream, nsamples, launches, steps, warmup=3):
    import torch
    stage = []
    engine.set_option("graph", 0)
    for k in range(warmup + launches):
        flush.zero_()
        engine.explain_device(X_dev.data_ptr(), n, phi_dev.data_ptr(), nsamples=nsamples)
        t = engine.last_timings_ms()["coalitions"]       # synchronises the engine's stream
        if k >= warmup:
            stage.append(t)
    path = engine.last_path()
    engine.set_option("graph", 1)
    for _ in range(warmup):
        flush.zero_()
        engine.explain_device(X_dev.data_ptr(), n, phi_dev.data_ptr(), nsamples=nsamples)
    starts = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
    ends = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
    torch.cuda.synchronize()
    for k in range(steps):
        flush.zero_()
        starts[k].record(stream)
        engine.explain_device(X_dev.data_ptr(), n, phi_dev.data_ptr(), nsamples=nsamples)
        ends[k].record(stream)
    torch.cuda.synchronize()
    engine.check_status()
    step = [s.elapsed_time(e) for s, e in zip(starts, ends)]
    return {"stage_ms": statistics.mean(stage), "stage_ms_min": min(stage), "stage_ms_max": max(stage),
            "step_ms": statistics.mean(step), "instances_per_s": n / (statistics.mean(step) / 1e3),
            "path": {k: path[k] for k in ("shared", "chunks", "warps", "cta_warps", "solve", "general", "bg_weights")}}


def run_variant(predict, bg, groups, names, weights, X, nsamples, kernel, options, flush, args, l1_rows=0):
    import torch
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    eng = GpuKernelExplainer(predict, DenseData(bg, names, groups, *(() if weights is None else (weights,))),
                             link="logit", kernel=kernel, seed=0)
    for k, v in options.items():
        eng.set_option(k, v)
    n, G = X.shape[0], len(groups)
    eng.shap_values(X[:256], nsamples=nsamples, l1_reg=False)              # plans built + uploaded
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    eng.set_stream(stream.cuda_stream)
    X_dev = torch.from_numpy(X).cuda()
    phi = torch.empty((2, n, G), dtype=torch.float64, device="cuda")
    out = measure(eng, X_dev, n, phi, flush, stream, nsamples, args.launches, args.steps)
    if l1_rows:
        try:
            eng.shap_values(X[:64], nsamples=nsamples)                      # l1 tables uploaded
            dts = []
            for _ in range(3):
                t0 = time.perf_counter()
                eng.shap_values(X[:l1_rows], nsamples=nsamples)             # l1_reg='auto'
                dts.append(time.perf_counter() - t0)
            out["l1_auto_ms"] = 1e3 * statistics.median(dts)
            out["l1_auto_path"] = {k: eng.last_path()[k] for k in ("shared", "solve", "bg_weights")}
        except Exception as exc:                                            # the old route refuses it: reported
            out["l1_auto_ms"] = None
            out["l1_auto_error"] = repr(exc)[:200]
    eng.set_stream(0)
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("the probe needs a CUDA device")
    from distributedkernelshap_b200.datasets import dense_tabular

    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    wl = bench.workload()
    bg = wl["data"]["background"]["X"]["preprocessed"]
    bg = np.ascontiguousarray(bg.toarray() if hasattr(bg, "toarray") else bg, dtype=np.float64)
    shapes = {
        "bench": dict(predict=wl["predictor"].predict_proba, bg=bg, groups=wl["groups"], names=wl["group_names"],
                      X=np.ascontiguousarray(wl["X_explain"], dtype=np.float64), nsamples=bench.NSAMPLES,
                      old="tcgen05", l1_rows=0),
    }
    d = dense_tabular(4096, 64, 512, seed=0)
    shapes["configs2"] = dict(predict=d["predictor"].predict_proba, bg=d["background"], groups=d["groups"],
                              names=d["group_names"], X=np.ascontiguousarray(d["X_explain"]), nsamples=4096, old="simt",
                              l1_rows=2048)

    sampler = bench.ClockSampler(0)
    sampler.start()
    results = {}
    for name, s in shapes.items():
        w = kmeans_like_counts(s["bg"].shape[0])
        variants = {"uniform": (None, "auto", {}), "weighted": (w, "auto", {}), "weighted_old_route": (w, s["old"], {})}
        res = {}
        for vname, (weights, kernel, options) in variants.items():
            res[vname] = run_variant(s["predict"], s["bg"], s["groups"], s["names"], weights, s["X"], s["nsamples"], kernel,
                                     options, flush, args, s["l1_rows"])
        res["weighted_over_uniform_stage"] = res["weighted"]["stage_ms"] / res["uniform"]["stage_ms"]
        res["old_route_over_weighted_step"] = res["weighted_old_route"]["step_ms"] / res["weighted"]["step_ms"]
        results[name] = res
    clocks = sampler.stop()

    props = torch.cuda.get_device_properties(0)
    line = {"probe": "weighted backgrounds on the shared-plan kernels", "launches": args.launches, "steps": args.steps,
            "shapes": results,
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
