"""Throughput of the module route (DESIGN.md §5.0.19) on the Adult shape: a 100-row background, 12 columns (one group each),
nsamples 2048, and a float32 ``nn.Sequential`` 12 -> 256 -> 256 -> 2 with ReLU and a softmax head, explained under the
logit link.  Rows are drawn from a seeded normal distribution.

Reports: instances/s of ``shap_values`` (host clock around a call that ends in a synchronise), and, from CUDA events on
torch's stream around the same calls the engine makes, the time of the mask kernel, the module, the reduce kernel and the
tail (link + solve), with the mask and reduce kernels' bytes (mask: rows x D x 4 B stored; reduce: rows x C x 4 B read
plus the means written) over their time against 3.35 TB/s.  The comparison is the same network as a float64
``MLPClassifier`` on its own route (the engine's MLP kernels), and the CPU oracle calling that classifier on the masked
batch, in seconds per instance.  The card name, power limit and SM clock are read in the same run.

    python scripts/torch_model_probe.py [--n 4096] [--out result.json]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.tree_probe import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _module(torch, P, hidden, dev):
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Linear(P, hidden), torch.nn.ReLU(), torch.nn.Linear(hidden, hidden),
                               torch.nn.ReLU(), torch.nn.Linear(hidden, 2), torch.nn.Softmax(dim=1)).to(dev).eval()


def _phases(eng, X, nsamples, torch):
    """One explain call through the C ABI with CUDA events between the steps: mask, module, reduce (summed over blocks)
    and the tail (the engine's own events).  Mirrors GpuKernelExplainer._explain_module for one block of rows."""
    from distributedkernelshap_b200 import _cabi, torch_models
    from distributedkernelshap_b200.engine import _dtype_code
    spec, lib, ctx = eng.spec, eng.lib, eng._ctx
    dev = torch.device("cuda", eng.device)
    eng._set_nsamples(nsamples)
    eng._apply_l1(False, nsamples, None)
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    with torch.inference_mode():
        eng._bind_torch_stream()
        X_dev = torch.from_numpy(X).to(dev)
        fx = spec.outputs(X_dev.to(spec.dtype))
        _cabi.check(lib.dks_external_prepare(ctx, C.c_void_p(X_dev.data_ptr()), X.shape[0], C.c_void_p(fx.data_ptr()),
                                             _dtype_code(fx)))
        total = C.c_int64(0)
        _cabi.check(lib.dks_external_begin(ctx, None, None, 0, C.byref(total)))
        blocks = torch_models.plan_blocks(total.value, eng.N, eng.model_batch_rows)
        buf = torch.empty((blocks[0][1], eng.P), dtype=spec.dtype, device=dev)
        t = {"mask": 0.0, "module": 0.0, "reduce": 0.0}
        for row0, rows in blocks:
            e = [ev() for _ in range(4)]
            x = buf[:rows]
            e[0].record()
            _cabi.check(lib.dks_external_mask(ctx, row0, rows, C.c_void_p(x.data_ptr())))
            e[1].record()
            y = spec.outputs(x)
            e[2].record()
            _cabi.check(lib.dks_external_reduce(ctx, row0, rows, C.c_void_p(y.data_ptr()), _dtype_code(y)))
            e[3].record()
            torch.cuda.synchronize()
            t["mask"] += e[0].elapsed_time(e[1])
            t["module"] += e[1].elapsed_time(e[2])
            t["reduce"] += e[2].elapsed_time(e[3])
        phi = np.empty((eng.D, X.shape[0], eng.data.groups_size))
        _cabi.check(lib.dks_external_finish(ctx, _cabi.ptr(phi)))
        t["tail"] = eng.last_timings_ms()["coalitions"]
        t["stage1"] = eng.last_timings_ms()["prepare"]
    return t, total.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--n-mlp", type=int, default=256)
    ap.add_argument("--nsamples", type=int, default=2048)
    ap.add_argument("--oracle-instances", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    from sklearn.neural_network import MLPClassifier

    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from oracle.shap_kernel_oracle import DenseData as ODense, KernelExplainerOracle

    P, N, H = 12, 100, 256
    rng = np.random.default_rng(0)
    bg = rng.normal(size=(N, P))
    X = rng.normal(size=(a.n, P))
    names, groups = [f"x{k}" for k in range(P)], [[k] for k in range(P)]
    data = DenseData(bg, names, groups)
    dev = torch.device("cuda", 0)
    module = _module(torch, P, H, dev)

    result = {"card": card(), "n": a.n, "N": N, "columns": P, "groups": P, "nsamples": a.nsamples,
              "module": f"float32 nn.Sequential {P} -> {H} -> {H} -> 2, ReLU, softmax; link logit"}
    eng = GpuKernelExplainer(module, data, link="logit", seed=0)
    eng.shap_values(X[:64], nsamples=a.nsamples, l1_reg=False)            # plans uploaded, kernels loaded, warm
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eng.shap_values(X, nsamples=a.nsamples, l1_reg=False)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    assert eng.last_path()["general"] == "torch"
    n_ph = min(a.n, 1024)
    _phases(eng, X[:64], a.nsamples, torch)                               # warm the event path
    ph, rows = _phases(eng, X[:n_ph], a.nsamples, torch)
    step = sum(ph[k] for k in ("stage1", "mask", "module", "reduce", "tail"))
    mask_bytes = rows * P * 4
    reduce_bytes = rows * 2 * 4 + rows // N * 2 * 8
    result["torch_route"] = {
        "wall_s": wall, "instances_per_s": a.n / wall, "model_batch_rows": eng.model_batch_rows,
        "phases_instances": n_ph, "masked_rows": rows, "phase_ms": ph,
        "phase_share": {k: ph[k] / step for k in ph},
        "mask_bytes": mask_bytes, "mask_bytes_per_s": mask_bytes / (ph["mask"] * 1e-3),
        "mask_share_of_hbm": mask_bytes / (ph["mask"] * 1e-3) / HBM_BYTES_PER_S,
        "reduce_bytes": reduce_bytes, "reduce_bytes_per_s": reduce_bytes / (ph["reduce"] * 1e-3),
        "reduce_share_of_hbm": reduce_bytes / (ph["reduce"] * 1e-3) / HBM_BYTES_PER_S,
    }
    print(json.dumps(result["torch_route"], indent=1), flush=True)
    eng.close()

    # the same network in float64 on the engine's MLP route, and the CPU oracle calling it
    clf = MLPClassifier(hidden_layer_sizes=(H, H), max_iter=1)
    clf.fit(np.vstack([bg[:2], bg[:2]]), [0, 1, 0, 1])
    lin = [m for m in module if isinstance(m, torch.nn.Linear)]
    clf.coefs_ = [m.weight.detach().double().cpu().numpy().T.copy() for m in lin]
    clf.intercepts_ = [m.bias.detach().double().cpu().numpy().copy() for m in lin]
    W, b = clf.coefs_[-1], clf.intercepts_[-1]                            # 2-way softmax = logistic on the logit gap
    clf.coefs_[-1], clf.intercepts_[-1] = (W[:, 1] - W[:, 0])[:, None], np.array([b[1] - b[0]])
    clf.n_outputs_, clf.out_activation_ = 1, "logistic"
    mlp = GpuKernelExplainer(clf.predict_proba, data, link="logit", seed=0)
    mlp.shap_values(X[:16], nsamples=a.nsamples, l1_reg=False)
    t0 = time.perf_counter()
    mlp.shap_values(X[:a.n_mlp], nsamples=a.nsamples, l1_reg=False)
    mwall = time.perf_counter() - t0
    result["mlp_route_float64"] = {"instances": a.n_mlp, "wall_s": mwall, "instances_per_s": a.n_mlp / mwall,
                                   "general": mlp.last_path()["general"]}
    orc = KernelExplainerOracle(clf.predict_proba, ODense(bg, names, groups), link="logit")
    t0 = time.perf_counter()
    for i in range(a.oracle_instances):
        plan = mlp.shared_plan(P, a.nsamples)
        orc.explain(X[i:i + 1], plan=(plan.dense(), plan.weights), nsamples=a.nsamples, l1_reg=False)
    result["oracle_cpu_s_per_instance"] = (time.perf_counter() - t0) / a.oracle_instances
    mlp.close()
    text = json.dumps(result, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
