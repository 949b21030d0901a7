"""Soft-voting ensembles on the device (DESIGN.md §5.0.17) on the Adult shape in raw form: 4 numeric and 8 categorical
columns (``datasets.decode_onehot_blocks``) encoded to 56 by ``ColumnTransformer(StandardScaler, OneHotEncoder(
handle_unknown='ignore'))``, 2560 instances, a 100-row background, nsamples 2048, logit link, for
``make_pipeline(ColumnTransformer(...), VotingClassifier([LogisticRegression, RandomForestClassifier(100, max_depth=10),
MLPClassifier, KNeighborsClassifier], voting='soft')).predict_proba``:

  * instances/s of the ensemble, from the engine's device events (stage 1 to the end of the solve);
  * instances/s of each member explained alone at the same shape (the fitted ColumnTransformer in front of it), and the
    ensemble's time over the sum of the members' times;
  * the CPU oracle's seconds per instance with the real ensemble's ``predict_proba`` on the engine's plans.

The card name, power limit and SM clock are read in the same run.  Prints one JSON document; ``--out`` also writes it.

    python scripts/ensemble_probe.py [--n 2560] [--reps 2] [--oracle-rows 1] [--out result.json]
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
    ap.add_argument("--oracle-rows", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import warnings
    from sklearn.compose import ColumnTransformer
    from sklearn.ensemble import RandomForestClassifier, VotingClassifier
    from sklearn.linear_model import LogisticRegression
    from sklearn.neighbors import KNeighborsClassifier
    from sklearn.neural_network import MLPClassifier
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import OneHotEncoder, StandardScaler

    from distributedkernelshap_b200._cabi import DksError
    from distributedkernelshap_b200.data import DenseData
    from distributedkernelshap_b200.datasets import ADULT_ONEHOT_WIDTHS, adult_like, decode_onehot_blocks
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from oracle.shap_kernel_oracle import DenseData as OracleData, KernelExplainerOracle
    from tree_probe import card

    d = adult_like(n_explain=a.n, n_background=100, seed=0)
    raw_bg, raw_X = (decode_onehot_blocks(A, 4, ADULT_ONEHOT_WIDTHS, True) for A in (d["background"], d["X_explain"]))
    raw_all = np.vstack([raw_bg, raw_X])
    p = d["predictor"].predict_proba(np.concatenate([d["background"], d["X_explain"]]))[:, 1]
    y = (np.random.default_rng(1).random(len(p)) < p).astype(int)    # labels drawn from the problem's probabilities
    D = raw_all.shape[1]
    names = [f"c{k}" for k in range(D)]
    ct = ColumnTransformer([("num", StandardScaler(), list(range(4))),
                            ("cat", OneHotEncoder(handle_unknown="ignore"), list(range(4, D)))])
    members = [("lr", LogisticRegression(max_iter=1000)),
               ("rf", RandomForestClassifier(100, max_depth=10, random_state=0)),
               ("mlp", MLPClassifier(random_state=0)), ("knn", KNeighborsClassifier())]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe = Pipeline([("ct", ct), ("vote", VotingClassifier(members, voting="soft"))]).fit(raw_all, y)
    fitted_ct, vote = pipe[0], pipe[-1]

    def engine(fn, link="logit"):
        return GpuKernelExplainer(fn, DenseData(raw_bg, names, [[k] for k in range(D)]), link=link, seed=0)

    def timed(eng, route):
        eng.shap_values(raw_X[:64], nsamples=a.nsamples, l1_reg=False)       # plans uploaded, kernels loaded
        runs = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            phi = eng.shap_values(raw_X, nsamples=a.nsamples, l1_reg=False)
            wall = time.perf_counter() - t0
            tm = eng.last_timings_ms()
            if route is not None:
                assert eng.last_path()["general"] == route, eng.last_path()
            runs.append({"total_ms": tm["total"], "instances_per_s": a.n / (tm["total"] * 1e-3), "wall_s": wall,
                         "general": eng.last_path()["general"]})
        return runs, phi

    eng = engine(pipe.predict_proba)
    ens_runs, phi = timed(eng, "ensemble")
    result = {"card": card(), "n": a.n, "N": 100, "raw_columns": D, "encoded_columns": eng.encoding.E,
              "nsamples": a.nsamples, "link": "logit", "fit_rows": len(raw_all),
              "model": "make_pipeline(ColumnTransformer([('num', StandardScaler(), [0..3]), ('cat', OneHotEncoder("
                       "handle_unknown='ignore'), [4..11])]), VotingClassifier([LogisticRegression(), "
                       "RandomForestClassifier(100, max_depth=10), MLPClassifier(), KNeighborsClassifier()], "
                       "voting='soft'))",
              "ensemble": {"runs": ens_runs, "kernel_launches_per_call": None}, "members": {}}
    before = eng.kernel_launches()
    eng.shap_values(raw_X[:64], nsamples=a.nsamples, l1_reg=False)
    result["ensemble"]["kernel_launches_per_call"] = eng.kernel_launches() - before
    best_ens = min(r["total_ms"] for r in ens_runs)
    member_sum = 0.0
    for name, est in vote.named_estimators_.items():
        fn = Pipeline([("ct", fitted_ct), ("m", est)]).predict_proba
        link = "logit"
        try:
            alone = engine(fn)
            runs, _ = timed(alone, None)
        except DksError as e:
            # a member alone can reach probabilities of exactly 0 or 1 (uniform k-NN votes), where the logit is
            # undefined: it is timed under the identity link, which runs the same kernels
            link = f"identity (logit refused: {e})"
            alone = engine(fn, "identity")
            runs, _ = timed(alone, None)
        best = min(r["total_ms"] for r in runs)
        member_sum += best
        result["members"][name] = {"link": link, "runs": runs, "best_ms": best}
        print(name, json.dumps(result["members"][name]), flush=True)
        alone.close()
    result["ensemble_over_member_sum"] = best_ens / member_sum
    orc = KernelExplainerOracle(pipe.predict_proba, OracleData(raw_bg, names, [[k] for k in range(D)]), link="logit")
    M, _ = eng.varying(raw_X[:a.oracle_rows])
    worst = 0.0
    t0 = time.perf_counter()
    for i in range(a.oracle_rows):
        plan = eng.shared_plan(int(M[i]), a.nsamples)
        want = orc.explain(raw_X[i:i + 1], plan=(plan.dense(), plan.weights), nsamples=a.nsamples, l1_reg=False)
        worst = max(worst, float(np.abs(phi[1][i] - want[:, 1]).max() / np.abs(want[:, 1]).max()))
    result["oracle_s_per_instance"] = (time.perf_counter() - t0) / a.oracle_rows
    result["oracle_max_rel_err"] = worst
    text = json.dumps(result, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
