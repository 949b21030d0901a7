#!/usr/bin/env python
"""Accuracy of the fused kernel's link table on the bench.py workload: phi dumped by ``bench.py --dump-outputs`` from two
builds (or any [C, n, G] arrays) against the float64 reference fed the engine's own shared plans, all 2560 instances.

  python scripts/link_table_probe.py --phi NEW.npy [--base PARENT.npy] [--out FILE]

Reports per input the max |phi - phi_ref| and rel_err (as the GPU tests define it); with --base, the largest per-instance
max|phi_new - phi_base| / max|phi_base|; and, from an engine run of this tree, the table bytes of the 12-group plan, the
passes that fell back to the exact loop, the first call's wall time (plan upload and table build included) and the
path.  One JSON line on stdout.
"""
import argparse
import json
import os
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--phi", required=True)
    ap.add_argument("--base", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
    from conftest import rel_err
    from linear_reference import LinearReference

    wl = bench.workload()
    X = np.ascontiguousarray(wl["X_explain"], dtype=np.float64)
    bg = wl["data"]["background"]["X"]["preprocessed"]
    explainer = KernelShap(wl["predictor"].predict_proba, link="logit", feature_names=wl["group_names"], seed=0)
    explainer.fit(bg, group_names=wl["group_names"], groups=wl["groups"])
    eng = explainer._explainer
    t0 = time.perf_counter()
    eng.get_explanation(X, nsamples=bench.NSAMPLES, l1_reg=False, silent=True)
    first_call_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    eng.get_explanation(X, nsamples=bench.NSAMPLES, l1_reg=False, silent=True)
    second_call_s = time.perf_counter() - t0
    G = eng.data.groups_size
    info = eng.fused_table_info(G)
    path = eng.last_path()

    clf = wl["predictor"]
    ref = LinearReference(clf.coef_, clf.intercept_, wl["background"], wl["groups"], kappa=2.0, link="logit")
    plans = []
    for x in X:
        v = ref.varying(x)
        plan = eng.shared_plan(len(v), bench.NSAMPLES) if len(v) >= 2 else None
        plans.append(None if plan is None else (plan.dense(), plan.weights))
    want = ref.shap_values(X, plans)[..., 1]

    def stats(phi):
        got = phi[1]
        return {"max_abs_err": float(np.abs(got - want).max()), "rel_err": float(rel_err(got, want))}

    new = np.load(args.phi)
    out = {"probe": "fused link table accuracy", "instances": int(X.shape[0]), "new": stats(new),
           "table_bytes": info["bytes"], "fallback_passes_two_calls": info["fallback_passes"],
           "first_call_s": first_call_s, "second_call_s": second_call_s,
           "path": {k: path[k] for k in ("shared", "solve", "fused_table")}}
    if args.base:
        base = np.load(args.base)
        out["base"] = stats(base)
        d = np.abs(new[1] - base[1]).max(axis=1) / np.abs(base[1]).max(axis=1)
        out["max_instance_rel_diff_vs_base"] = float(d.max())
    eng.close()
    text = json.dumps(out)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
