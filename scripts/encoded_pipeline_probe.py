"""Kernel machines, MLPs and k-nearest-neighbour models behind per-column preprocessing (DESIGN.md §5.0.16) on the Adult
shape in raw form: 4 numeric and 8 categorical columns (``datasets.decode_onehot_blocks``),
``ColumnTransformer(StandardScaler, OneHotEncoder(handle_unknown='ignore'))``, 2560 instances, a 100-row background,
nsamples 2048, for ``SVC().decision_function`` (identity link), ``MLPClassifier().predict_proba`` (logit link) and
``KNeighborsClassifier().predict_proba`` (identity link: uniform votes reach probabilities of exactly 0 and 1).  Per
model:

  * instances/s of the pipeline route (raw rows in, the device encodes them) and of the same fitted estimator explained
    on the encoded columns (one group per raw column's encoded block), alternated in one run, from the engine's device
    events (stage 1 to the end of the solve);
  * the device time of every stage-1 kernel, the encode kernel among them (torch.profiler, a run of its own);
  * max |d phi| between the two readings.

The card name, power limit and SM clock are read in the same run.  Prints one JSON document; ``--out`` also writes it.

    python scripts/encoded_pipeline_probe.py [--n 2560] [--reps 2] [--out result.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2560)
    ap.add_argument("--nsamples", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import warnings
    from sklearn.compose import ColumnTransformer
    from sklearn.neighbors import KNeighborsClassifier
    from sklearn.neural_network import MLPClassifier
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import OneHotEncoder, StandardScaler
    from sklearn.svm import SVC

    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import ADULT_ONEHOT_WIDTHS, adult_like, decode_onehot_blocks
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from tree_pipeline_probe import encode_kernel_ms
    from tree_probe import card

    d = adult_like(n_explain=a.n, n_background=100, seed=0)
    raw_bg, raw_X = (decode_onehot_blocks(A, 4, ADULT_ONEHOT_WIDTHS, True) for A in (d["background"], d["X_explain"]))
    raw_all = np.vstack([raw_bg, raw_X])
    p = d["predictor"].predict_proba(np.concatenate([d["background"], d["X_explain"]]))[:, 1]
    y = (np.random.default_rng(1).random(len(p)) < p).astype(int)    # labels drawn from the problem's probabilities
    D = raw_all.shape[1]
    models = {   # name: (estimator, method, link, route)
        "SVC().decision_function": (SVC(), "decision_function", "identity", "kmach"),
        "MLPClassifier().predict_proba": (MLPClassifier(random_state=0), "predict_proba", "logit", "mlp"),
        "KNeighborsClassifier().predict_proba": (KNeighborsClassifier(), "predict_proba", "identity", "knn"),
    }
    result = {"card": card(), "n": a.n, "N": 100, "raw_columns": D, "nsamples": a.nsamples, "fit_rows": len(raw_all),
              "preprocessing": "ColumnTransformer([('num', StandardScaler(), [0..3]), ('cat', OneHotEncoder("
                               "handle_unknown='ignore'), [4..11])])", "models": {}}
    names = [f"c{k}" for k in range(D)]
    for name, (m, method, link, route) in models.items():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            pipe = make_pipeline(ColumnTransformer([("num", StandardScaler(), list(range(4))),
                                                    ("cat", OneHotEncoder(handle_unknown="ignore"), list(range(4, D)))]),
                                 m).fit(raw_all, y)
        pipe_eng = GpuKernelExplainer(getattr(pipe, method), DenseData(raw_bg, names, [[k] for k in range(D)]),
                                      link=link, seed=0)
        enc = pipe_eng.encoding
        groups = [[int(e) for e in np.nonzero(enc.sources == c)[0]] for c in range(D)]
        Zbg, ZX = (pipe_eng.encode(A) for A in (raw_bg, raw_X))
        enc_eng = GpuKernelExplainer(getattr(pipe[-1], method), DenseData(Zbg, names, groups), link=link, seed=0)
        runs = {"pipeline": [], "encoded": []}
        phis = {}
        for eng, X in ((pipe_eng, raw_X), (enc_eng, ZX)):
            eng.shap_values(X[:64], nsamples=a.nsamples, l1_reg=False)          # plans uploaded, kernels loaded
        for r in range(a.reps):
            for eng, X, key in ((pipe_eng, raw_X, "pipeline"), (enc_eng, ZX, "encoded")):
                t0 = time.perf_counter()
                phi = eng.shap_values(X, nsamples=a.nsamples, l1_reg=False)
                wall = time.perf_counter() - t0
                tm = eng.last_timings_ms()
                assert eng.last_path()["general"] == route
                runs[key].append({"total_ms": tm["total"], "prepare_ms": tm["prepare"], "explain_stage_ms": tm["coalitions"],
                                  "instances_per_s": a.n / (tm["total"] * 1e-3), "wall_s": wall})
                phis[key] = np.stack(phi if isinstance(phi, list) else [phi])
        stage1 = encode_kernel_ms(pipe_eng, raw_X)
        enc_ms = [v for k, v in stage1.items() if "encode" in k]
        M = pipe_eng.varying(raw_X)[0]
        entry = {"link": link, "route": route, "encoded_columns": enc.E, "instances_with_M": {
                     str(int(k)): int((M == k).sum()) for k in np.unique(M)},
                 "varying_sets_equal": bool(np.array_equal(M, enc_eng.varying(ZX)[0])), "runs": runs,
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
