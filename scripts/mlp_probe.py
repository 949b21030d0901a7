"""Throughput of the MLP route (DESIGN.md §5.0.14) on the Adult-shaped problem: 2560 instances, a 100-row background, 12
groups over 49 columns, nsamples 2048, for three MLPs fitted to labels drawn from the problem's predictor probabilities
(so that the logit of a classifier's probabilities stays finite):

  make_pipeline(StandardScaler(), MLPClassifier())                                 predict_proba, logit link
  make_pipeline(StandardScaler(), MLPClassifier((100, 100), activation='tanh'))   predict_proba, identity link (logit
                                                                                  tried first: refused where it saturates)
  make_pipeline(StandardScaler(), MLPRegressor((64,)))                            predict, identity link

Per model and l1_reg (False, 'auto'): instances/s from the engine's device events (stage 1 to the end of the solve), the
explain kernel's time, the FP64 FLOP per instance computed from the shapes (2 S N sum_l K_l H_l over the layers, layer 1
with K = M; padded: K and H rounded up to the mma fragment shapes) and the achieved FLOP/s of the explain stage against
both, and, as the CPU figure, the oracle calling the real scikit-learn method on the masked batch for a few instances.  The
card name, power limit and SM clock are read in the same run.  Prints one JSON document; ``--out`` also writes it to a file.

    python scripts/mlp_probe.py [--n 2560] [--fit-rows 3000] [--oracle-instances 2] [--out result.json]
"""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.tree_probe import card  # noqa: E402


def _pad(v, m):
    return (v + m - 1) // m * m


def flop_per_instance(spec, M, S, N, padded):
    """FP64 FLOP of one instance's masked forward passes: 2 S N sum over layers of K_l H_l (layer 1: K = M)."""
    widths = spec.widths
    total = 0
    for l in range(len(widths) - 1):
        K = M if l == 0 else widths[l]
        H = widths[l + 1]
        last = l == len(widths) - 2
        if padded:
            K = _pad(K, 16)
            H = _pad(H, 8 if last else 16)
        total += K * H
    return 2 * S * N * total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2560)
    ap.add_argument("--nsamples", type=int, default=2048)
    ap.add_argument("--fit-rows", type=int, default=3000)
    ap.add_argument("--oracle-instances", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from sklearn.exceptions import ConvergenceWarning
    from sklearn.neural_network import MLPClassifier, MLPRegressor
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler

    from distributedkernelshap_b200._cabi import DksError
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import adult_like
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from distributedkernelshap_b200.mlp import extract_mlp_spec
    from oracle.shap_kernel_oracle import DenseData as ODense, KernelExplainerOracle

    d = adult_like(n_explain=max(a.n, a.fit_rows), n_background=100, seed=0)
    X_fit = d["X_explain"][:a.fit_rows]
    p = d["predictor"].predict_proba(X_fit)[:, 1]
    y = (np.random.default_rng(1).random(len(p)) < p).astype(int)
    X_exp = d["X_explain"][:a.n]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        clf = make_pipeline(StandardScaler(), MLPClassifier(random_state=0)).fit(X_fit, y)
        deep = make_pipeline(StandardScaler(), MLPClassifier(hidden_layer_sizes=(100, 100), activation="tanh",
                                                             random_state=0)).fit(X_fit, y)
        reg = make_pipeline(StandardScaler(), MLPRegressor(hidden_layer_sizes=(64,), random_state=0)).fit(X_fit, p)
    models = {
        "make_pipeline(StandardScaler(), MLPClassifier()).predict_proba": (clf.predict_proba, "logit"),
        # its probabilities reach exactly 0 or 1 in float64 on some rows, whose logit the engine refuses
        # (DKS_ERR_NUMERIC): the refusal is recorded and the model measured under the identity link
        "make_pipeline(StandardScaler(), MLPClassifier((100, 100), activation='tanh')).predict_proba":
            (deep.predict_proba, "identity"),
        "make_pipeline(StandardScaler(), MLPRegressor((64,))).predict": (reg.predict, "identity"),
    }
    result = {"card": card(), "n": a.n, "N": 100, "groups": len(d["groups"]), "columns": X_fit.shape[1],
              "nsamples": a.nsamples, "fit_rows": a.fit_rows, "models": {}}
    data = DenseData(d["background"], d["group_names"], d["groups"])
    for name, (fn, link) in models.items():
        spec = extract_mlp_spec(fn)
        if link == "identity" and spec.head != "identity":
            try:
                GpuKernelExplainer(fn, data, link="logit", seed=0).shap_values(X_exp, nsamples=a.nsamples, l1_reg=False)
                logit = "explained"
            except DksError as e:
                logit = f"refused: {e}"
        else:
            logit = None
        eng = GpuKernelExplainer(fn, data, link=link, seed=0)
        M, _ = eng.varying(X_exp)
        Mmax = int(M.max())
        S = int(eng.shared_plan(Mmax, a.nsamples).S)
        fl = flop_per_instance(spec, Mmax, S, 100, False)
        flp = flop_per_instance(spec, Mmax, S, 100, True)
        entry = {"link": link, "widths": spec.widths, "activation": spec.hidden_activation, "M_full_set": Mmax,
                 "logit_link": logit, "S_full_set": S, "fp64_flop_per_instance": fl,
                 "fp64_flop_per_instance_padded": flp, "runs": {}}
        for l1 in (False, "auto"):
            eng.shap_values(X_exp[:64], nsamples=a.nsamples, l1_reg=l1)      # plans uploaded, kernels loaded
            t0 = time.perf_counter()
            eng.shap_values(X_exp, nsamples=a.nsamples, l1_reg=l1)
            wall = time.perf_counter() - t0
            tm = eng.last_timings_ms()
            path = eng.last_path()
            run = {"total_ms": tm["total"], "explain_stage_ms": tm["coalitions"],
                   "instances_per_s": a.n / (tm["total"] * 1e-3), "wall_s": wall,
                   "general": path["general"], "general_l1": path["general_l1"]}
            if tm["coalitions"] > 0:
                # instances with M < Mmax do less work: the full-set figure bounds the stage's FLOP from above
                run["fp64_tflops_vs_unpadded"] = fl * a.n / (tm["coalitions"] * 1e-3) / 1e12
                run["fp64_tflops_vs_padded"] = flp * a.n / (tm["coalitions"] * 1e-3) / 1e12
            entry["runs"][str(l1)] = run
            print(name, l1, run, flush=True)
        orc = KernelExplainerOracle(fn, ODense(d["background"], d["group_names"], d["groups"]), link=link)
        t0 = time.perf_counter()
        for i in range(a.oracle_instances):
            plan = eng.shared_plan(int(M[i]), a.nsamples)
            orc.explain(X_exp[i:i + 1], plan=(plan.dense(), plan.weights), nsamples=a.nsamples, l1_reg=False)
        entry["oracle_cpu_s_per_instance"] = (time.perf_counter() - t0) / a.oracle_instances
        result["models"][name] = entry
        eng.close()
    text = json.dumps(result, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
