#!/usr/bin/env python
"""Attribute a device-resident shared-plan step node by node: where the time of bench.py's ``value`` goes.

  python scripts/step_profile.py [--n 2560,256,64] [--steps 30] [--warmup 5] [--out-dir DIR]

The workload is bench.py's (Adult-shaped instances, 12 groups, 100 background rows, nsamples = 2048, shared plans); the
``--n`` sweep explains its first n instances.  For each n the step runs as bench.py runs it -- the engine's CUDA graph
replayed on a user stream, the L2 flushed before each step -- first ``--steps`` times under CUDA events alone (``step_ms``),
then ``--steps`` times under ``torch.profiler`` with CUDA activities (a run of its own: the trace is written to
DIR/step_trace_n<n>.json).  From the trace, per step:

  nodes   the device time of every node of the replayed graph: the status/counter memset, stage 1 (``prep_kernel``), the
          fused shared-plan kernel, its finish kernel (``finish_fused_kernel``) and the general kernel(s) of the
          remaining instances;
  gaps    from the end of the memset to the start of stage 1, from the end of stage 1 to the start of the fused kernel,
          from the end of the fused kernel to the start of the finish kernel, and from the end of the fused kernel to
          the end of the step;
  stage1_plus_gaps   memset end -> fused kernel start, what stage 1 costs the step;
  span    memset start -> the end of the last node.

Medians over the profiled steps.  One JSON line on stdout (also DIR/step_profile.json) with the GPU name and its power
limit.  Needs a CUDA device.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

import bench  # noqa: E402  (the workload and the NVML power limit of the benchmark)

ROLES = (("prep", "prep_kernel"), ("fused", "explain_shared_fused_kernel"), ("finish", "finish_fused_kernel"))


def role_of(ev):
    if ev.get("cat") == "gpu_memset":
        return "memset"
    name = ev.get("name", "")
    for role, key in ROLES:
        if key in name:
            return role
    return "general"


def is_flush(ev):
    return ev.get("cat") == "kernel" and "fill" in ev.get("name", "").lower() and "dks" not in ev.get("name", "")


def split_steps(trace_path):
    """Device events of the trace, grouped into steps: a step is what runs between two L2 flushes."""
    with open(trace_path) as f:
        events = json.load(f)["traceEvents"]
    dev = sorted((e for e in events if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset")),
                 key=lambda e: float(e["ts"]))
    steps, cur = [], None
    for e in dev:
        if is_flush(e):
            if cur:
                steps.append(cur)
            cur = []
        elif cur is not None:
            cur.append(e)
    if cur:
        steps.append(cur)
    return steps


def attribute(step):
    """Per-node durations and the gaps between the nodes of one step (microseconds)."""
    t = {}
    for e in step:
        r = role_of(e)
        s, d = float(e["ts"]), float(e["dur"])
        if r in t:          # several general kernels: their union as one node
            t[r] = (min(t[r][0], s), max(t[r][1], s + d), t[r][2] + d)
        else:
            t[r] = (s, s + d, d)
    if not all(k in t for k in ("memset", "prep", "fused")):
        return None
    end = max(v[1] for v in t.values())
    out = {"nodes_us": {k: v[2] for k, v in t.items()},
           "gaps_us": {"memset->prep": t["prep"][0] - t["memset"][1], "prep->fused": t["fused"][0] - t["prep"][1],
                       "fused->step_end": end - t["fused"][1]},
           "stage1_plus_gaps_us": t["fused"][0] - t["memset"][1],
           "span_us": end - t["memset"][0]}
    if "finish" in t:
        out["gaps_us"]["fused->finish"] = t["finish"][0] - t["fused"][1]
    if "general" in t:
        out["gaps_us"]["prep->general"] = t["general"][0] - t["prep"][1]
    return out


def median_of(dicts):
    keys = dicts[0].keys()
    return {k: (median_of([d[k] for d in dicts]) if isinstance(dicts[0][k], dict)
                else statistics.median(d[k] for d in dicts)) for k in keys if all(k in d for d in dicts)}


def run_n(engine, X_dev, m, C, G, flush, stream, steps, warmup, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile
    phi = torch.empty((C, m, G), dtype=torch.float64, device="cuda")

    def step():
        flush.zero_()
        engine.explain_device(X_dev.data_ptr(), m, phi.data_ptr(), nsamples=bench.NSAMPLES)

    for _ in range(warmup):          # the second call captures the graph, the rest replay it
        step()
    torch.cuda.synchronize()
    engine.check_status()
    starts = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
    ends = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
    for k in range(steps):
        flush.zero_()
        starts[k].record(stream)
        engine.explain_device(X_dev.data_ptr(), m, phi.data_ptr(), nsamples=bench.NSAMPLES)
        ends[k].record(stream)
    torch.cuda.synchronize()
    step_ms = [s.elapsed_time(e) for s, e in zip(starts, ends)]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    engine.check_status()
    trace = os.path.join(out_dir, f"step_trace_n{m}.json")
    prof.export_chrome_trace(trace)
    per_step = [a for a in (attribute(s) for s in split_steps(trace)) if a is not None]
    if not per_step:
        raise SystemExit(f"n = {m}: no step with a memset, prep_kernel and the fused kernel in the trace")
    return {"step_ms": statistics.mean(step_ms), "step_ms_min": min(step_ms), "profiled_steps": len(per_step),
            **median_of(per_step), "path": {k: engine.last_path()[k] for k in ("shared", "general")}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", default="2560,256,64", help="instance counts (comma separated)")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "dks_step_profile"),
                    help="where the traces and the JSON line are written")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("the step profile needs a CUDA device")
    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    os.makedirs(args.out_dir, exist_ok=True)

    wl = bench.workload()
    X = np.ascontiguousarray(wl["X_explain"], dtype=np.float64)
    explainer = KernelShap(wl["predictor"].predict_proba, link="logit", feature_names=wl["group_names"], seed=0)
    explainer.fit(wl["data"]["background"]["X"]["preprocessed"], group_names=wl["group_names"], groups=wl["groups"])
    engine = explainer._explainer
    engine.get_explanation(X, nsamples=bench.NSAMPLES, l1_reg=False, silent=True)      # shared plans built + uploaded
    G, C = engine.data.groups_size, engine.D
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    engine.set_stream(stream.cuda_stream)
    X_dev = torch.from_numpy(X).cuda()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    by_n = {}
    for m in [int(v) for v in args.n.split(",") if v]:
        m = min(m, X.shape[0])
        by_n[str(m)] = run_n(engine, X_dev[:m], m, C, G, flush, stream, args.steps, args.warmup, args.out_dir)
    engine.close()

    props = torch.cuda.get_device_properties(0)
    line = {"probe": "shared-plan step attribution", "workload": "bench.py: Adult-shaped instances, G = 12, N = 100, "
            "nsamples = 2048, shared plans, CUDA graph replay, L2 flushed before each step", "steps": args.steps,
            "by_n": by_n, "gpu": {"name": props.name, "sm_count": props.multi_processor_count,
                                  "power_limit_w": bench._power_limit_w(0)}}
    text = json.dumps(line)
    print(text)
    with open(os.path.join(args.out_dir, "step_profile.json"), "w") as f:
        f.write(text + "\n")


if __name__ == "__main__":
    main()
