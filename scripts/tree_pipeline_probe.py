"""Tree models behind per-column preprocessing (DESIGN.md §5.0.13) on the Adult shape in raw form: 4 numeric and 8
categorical columns (``datasets.decode_onehot_blocks``), ``ColumnTransformer(StandardScaler, OneHotEncoder)``, 2560
instances, a 100-row background, nsamples 2048, link logit, for the three models of ``scripts/tree_probe.py`` behind
that preprocessing.  Per model:

  * instances/s of the pipeline route (raw rows in, the device encodes them) and of the same fitted trees explained on
    the encoded columns (one group per raw column's encoded block), alternated in one run, from the engine's device
    events (stage 1 to the end of the solve);
  * the device time of every stage-1 kernel, the encode kernel among them (torch.profiler, a run of its own);
  * max |d phi| between the two readings (expected 0).

The card name, power limit and SM clock are read in the same run.  Prints one JSON document; ``--out`` also writes it.

    python scripts/tree_pipeline_probe.py [--n 2560] [--reps 3] [--out result.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def encode_kernel_ms(eng, X, reps=20):
    """Device time of one encode_kernel launch over the rows X, from torch.profiler's CUDA activity records around
    stage 1 (dks_prepare_dev) on device-resident rows, in a run of its own after the timed ones."""
    import ctypes as C
    import torch
    from torch.profiler import ProfilerActivity, profile
    from distributedkernelshap_b200 import _cabi
    X_dev = torch.from_numpy(np.ascontiguousarray(X)).cuda()
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    _cabi.check(eng.lib.dks_prepare_dev(eng._ctx, C.c_void_p(X_dev.data_ptr()), X.shape[0]))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            _cabi.check(eng.lib.dks_prepare_dev(eng._ctx, C.c_void_p(X_dev.data_ptr()), X.shape[0]))
        torch.cuda.synchronize()
    eng.set_stream(0)
    out = {}
    for k in prof.key_averages():
        t = getattr(k, "device_time_total", None)
        t = k.cuda_time_total if t is None else t
        if k.count:
            out[k.key] = t / k.count / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2560)
    ap.add_argument("--nsamples", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from sklearn.compose import ColumnTransformer
    from sklearn.ensemble import GradientBoostingClassifier, HistGradientBoostingClassifier, RandomForestClassifier
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import OneHotEncoder, StandardScaler

    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import ADULT_ONEHOT_WIDTHS, adult_like, decode_onehot_blocks
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from tree_probe import card

    d = adult_like(n_explain=a.n, n_background=100, seed=0)
    raw_bg, raw_X = (decode_onehot_blocks(A, 4, ADULT_ONEHOT_WIDTHS, True) for A in (d["background"], d["X_explain"]))
    raw_all = np.vstack([raw_bg, raw_X])
    y = d["predictor"].predict(np.concatenate([d["background"], d["X_explain"]]))
    D = raw_all.shape[1]
    models = {
        "GradientBoostingClassifier()": GradientBoostingClassifier(random_state=0),
        "HistGradientBoostingClassifier()": HistGradientBoostingClassifier(random_state=0),
        "RandomForestClassifier(n_estimators=100, max_depth=10)": RandomForestClassifier(100, max_depth=10, random_state=0),
    }
    result = {"card": card(), "n": a.n, "N": 100, "raw_columns": D, "nsamples": a.nsamples, "link": "logit",
              "preprocessing": "ColumnTransformer([('num', StandardScaler(), [0..3]), ('cat', OneHotEncoder("
                               "handle_unknown='ignore'), [4..11])])", "models": {}}
    names = [f"c{k}" for k in range(D)]
    for name, m in models.items():
        pipe = make_pipeline(ColumnTransformer([("num", StandardScaler(), list(range(4))),
                                                ("cat", OneHotEncoder(handle_unknown="ignore", sparse_output=False),
                                                 list(range(4, D)))]), m).fit(raw_all, y)
        pipe_eng = GpuKernelExplainer(pipe.predict_proba, DenseData(raw_bg, names, [[k] for k in range(D)]),
                                      link="logit", seed=0)
        enc = pipe_eng.encoding
        groups = [[int(e) for e in np.nonzero(enc.sources == c)[0]] for c in range(D)]
        Zbg, ZX = (np.asarray(pipe[:-1].transform(A), dtype=np.float64) for A in (raw_bg, raw_X))
        enc_eng = GpuKernelExplainer(pipe[-1].predict_proba, DenseData(Zbg, names, groups), link="logit", seed=0)
        runs = {"pipeline": [], "encoded": []}
        phis = {}
        for eng, X, key in ((pipe_eng, raw_X, "pipeline"), (enc_eng, ZX, "encoded")):
            eng.shap_values(X[:64], nsamples=a.nsamples, l1_reg=False)          # plans uploaded, kernels loaded
        for r in range(a.reps):
            for eng, X, key in ((pipe_eng, raw_X, "pipeline"), (enc_eng, ZX, "encoded")):
                t0 = time.perf_counter()
                phi = eng.shap_values(X, nsamples=a.nsamples, l1_reg=False)
                wall = time.perf_counter() - t0
                tm = eng.last_timings_ms()
                assert eng.last_path()["general"] == "trees"
                runs[key].append({"total_ms": tm["total"], "prepare_ms": tm["prepare"], "explain_stage_ms": tm["coalitions"],
                                  "instances_per_s": a.n / (tm["total"] * 1e-3), "wall_s": wall})
                phis[key] = np.stack(phi)
        stage1 = encode_kernel_ms(pipe_eng, raw_X)
        enc_ms = [v for k, v in stage1.items() if "encode_kernel" in k]
        entry = {"encoded_columns": enc.E, "trees": pipe_eng.spec.n_trees, "runs": runs,
                 "stage1_kernel_ms_pipeline": stage1, "stage1_kernel_ms_encoded": encode_kernel_ms(enc_eng, ZX),
                 "encode_kernel_ms": enc_ms[0] if enc_ms else None,
                 "max_abs_dphi": float(np.abs(phis["pipeline"] - phis["encoded"]).max())}
        print(name, json.dumps(entry), flush=True)
        result["models"][name] = entry
        pipe_eng.close()
        enc_eng.close()
    text = json.dumps(result, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
