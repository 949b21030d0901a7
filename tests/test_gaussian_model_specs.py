"""Gaussian generative models read into ``GaussianModelSpec`` (no GPU): every extractor's NumPy evaluation against the
scikit-learn method it was read from, bare, behind an affine scaler and behind a per-column pipeline; every refusal."""
import numpy as np
import pytest

sklearn = pytest.importorskip("sklearn")
from sklearn.compose import ColumnTransformer  # noqa: E402
from sklearn.covariance import EllipticEnvelope  # noqa: E402
from sklearn.discriminant_analysis import QuadraticDiscriminantAnalysis  # noqa: E402
from sklearn.ensemble import RandomForestClassifier, StackingClassifier, VotingClassifier  # noqa: E402
from sklearn.linear_model import LogisticRegression  # noqa: E402
from sklearn.mixture import BayesianGaussianMixture, GaussianMixture  # noqa: E402
from sklearn.naive_bayes import GaussianNB  # noqa: E402
from sklearn.pipeline import make_pipeline  # noqa: E402
from sklearn.preprocessing import (MinMaxScaler, OneHotEncoder, PolynomialFeatures, RobustScaler,  # noqa: E402
                                   StandardScaler)

from distributedkernelshap_b200.gaussian_models import (GaussianModelSpec, extract_gaussian_spec,  # noqa: E402
                                                        refuse_gaussian_members)
from distributedkernelshap_b200.trees import extract_encoded_pipeline_spec  # noqa: E402

RTOL = 1e-12


def _data(seed=0, n=300, P=5, classes=3):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)) * np.linspace(0.5, 3.0, P) + np.linspace(-1.0, 4.0, P)
    X[:, 1] += 0.6 * X[:, 0]
    s = X[:, 0] - X[:, 0].mean() + (X[:, 2] - X[:, 2].mean()) * 0.7
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, classes + 1)[1:-1]))
    Q = rng.normal(size=(80, P)) * np.linspace(0.5, 3.0, P) + np.linspace(-1.0, 4.0, P)
    return X, y, Q


def _close(spec, fn, Q):
    """To 1e-12, absolutely for the outputs near 0: a score l carries a rounding of about 1e-16 |l|, and a probability
    p(1 - p) times that, so the bound scales with the largest score (about 1e4 for rows far from every centre)."""
    got, want = spec(Q), fn(Q)
    assert got.shape == want.shape
    scale = max(100.0, float(np.max(np.abs(spec.scores(Q)))), float(np.max(np.abs(want))))
    np.testing.assert_allclose(got, want, rtol=RTOL, atol=1e-14 * scale)


MODELS = {
    "qda2": lambda: QuadraticDiscriminantAnalysis(reg_param=0.1),
    "qda5": lambda: QuadraticDiscriminantAnalysis(reg_param=0.05),
    "nb": lambda: GaussianNB(priors=[0.2, 0.5, 0.3]),
    "gmm_full": lambda: GaussianMixture(3, covariance_type="full", random_state=0),
    "gmm_tied": lambda: GaussianMixture(3, covariance_type="tied", random_state=0),
    "gmm_diag": lambda: GaussianMixture(4, covariance_type="diag", random_state=0),
    "gmm_spherical": lambda: GaussianMixture(2, covariance_type="spherical", random_state=0),
    "bgmm_full": lambda: BayesianGaussianMixture(n_components=3, random_state=0, max_iter=200),
    "bgmm_diag_dist": lambda: BayesianGaussianMixture(n_components=3, covariance_type="diag", random_state=0,
                                                      weight_concentration_prior_type="dirichlet_distribution"),
    "bgmm_tied": lambda: BayesianGaussianMixture(n_components=2, covariance_type="tied", random_state=0),
    "bgmm_spherical": lambda: BayesianGaussianMixture(n_components=3, covariance_type="spherical", random_state=0),
    "envelope": lambda: EllipticEnvelope(random_state=0),
}
METHODS = {"qda2": ("predict_proba", "decision_function"), "qda5": ("predict_proba", "decision_function"),
           "nb": ("predict_proba",), "envelope": ("decision_function", "score_samples")}
CLASSES = {"qda2": 2, "qda5": 5, "nb": 3}


def _fit(key, scaler=None, seed=0):
    X, y, Q = _data(seed, classes=CLASSES.get(key, 3))
    est = MODELS[key]()
    model = make_pipeline(scaler(), est) if scaler else est
    model.fit(X, y) if key in CLASSES else model.fit(X)
    return model, Q


@pytest.mark.parametrize("key", sorted(MODELS))
@pytest.mark.parametrize("scaler", [None, StandardScaler, MinMaxScaler, RobustScaler])
def test_every_model_and_method_matches_scikit_learn(key, scaler):
    model, Q = _fit(key, scaler)
    for method in METHODS.get(key, ("predict_proba", "score_samples")):
        fn = getattr(model, method)
        spec = extract_gaussian_spec(fn)
        assert isinstance(spec, GaussianModelSpec)
        _close(spec, fn, Q)
        _close(spec, fn, Q * 30.0 + 100.0)                  # rows far from every centre


def test_heads_and_shapes():
    m2, _ = _fit("qda2")
    m5, _ = _fit("qda5")
    assert extract_gaussian_spec(m2.decision_function).head == "diff"
    assert extract_gaussian_spec(m2.decision_function).scalar_out
    assert extract_gaussian_spec(m5.decision_function).head == "identity"
    assert extract_gaussian_spec(m5.predict_proba).n_outputs == 5
    g, _ = _fit("gmm_full")
    assert extract_gaussian_spec(g.score_samples).head == "logsumexp"
    assert extract_gaussian_spec(g.score_samples).n_outputs == 1
    e, _ = _fit("envelope")
    s = extract_gaussian_spec(e.decision_function)
    assert s.head == "identity" and s.K == 1 and s.scalar_out
    r_off, L = s.flat()
    assert r_off.tolist() == [0, 5] and L.shape == (5, 5)


def test_the_engine_sizes_row_blocks_from_the_spec():
    from distributedkernelshap_b200.engine import MAX_ROWS_PER_CALL, rows_per_call
    m5, _ = _fit("qda5")
    s = extract_gaussian_spec(m5.predict_proba)
    assert s.R == s.K == 5
    assert rows_per_call(s.act_code, s.n_outputs, "shared", 5, s.R) == MAX_ROWS_PER_CALL


@pytest.mark.parametrize("key", ["qda5", "nb", "gmm_diag", "bgmm_full", "envelope"])
def test_column_transformer_pipeline(key):
    X, y, Q = _data(4, classes=CLASSES.get(key, 3))
    Xc = np.concatenate([X, np.floor(np.abs(X[:, :1])) % 3], axis=1)
    Qc = np.concatenate([Q, np.floor(np.abs(Q[:, :1])) % 3], axis=1)
    pre = ColumnTransformer([("num", StandardScaler(), [0, 1, 2, 3, 4]),
                             ("cat", OneHotEncoder(sparse_output=False), [5])])
    est = MODELS[key]()
    if key == "qda5":
        est = QuadraticDiscriminantAnalysis(reg_param=0.3)
    pipe = make_pipeline(pre, est)
    pipe.fit(Xc, y) if key in CLASSES else pipe.fit(Xc)
    for method in METHODS.get(key, ("predict_proba", "score_samples")):
        fn = getattr(pipe, method)
        spec, enc = extract_encoded_pipeline_spec(fn)
        assert isinstance(spec, GaussianModelSpec) and spec.n_features == enc.D > 5
        _close(spec, getattr(pipe[-1], method), pipe[:-1].transform(Qc))


def test_refusals():
    X, y, Q = _data(2, classes=3)
    qda = QuadraticDiscriminantAnalysis(reg_param=0.1).fit(X, y)
    for bad in (qda.predict, qda.predict_log_proba):
        with pytest.raises(TypeError, match="not supported"):
            extract_gaussian_spec(bad)
    g = GaussianMixture(2, random_state=0).fit(X)
    for bad in (g.predict, g.predict_log_proba if hasattr(g, "predict_log_proba") else g.score):
        with pytest.raises(TypeError, match="not supported"):
            extract_gaussian_spec(bad)
    e = EllipticEnvelope(random_state=0).fit(X)
    with pytest.raises(TypeError, match="predict returns labels"):
        extract_gaussian_spec(e.predict)
    nb = GaussianNB().fit(X, y)
    with pytest.raises(TypeError, match="predict returns labels"):
        extract_gaussian_spec(nb.predict)
    with pytest.raises(TypeError, match="not supported"):
        extract_gaussian_spec(nb.predict_log_proba)
    # more than 8 classes / components
    y9 = np.arange(X.shape[0]) % 9
    with pytest.raises(NotImplementedError, match="at most 8"):
        extract_gaussian_spec(QuadraticDiscriminantAnalysis(reg_param=0.1).fit(X, y9).predict_proba)
    with pytest.raises(NotImplementedError, match="at most 8"):
        extract_gaussian_spec(GaussianNB().fit(X, y9).predict_proba)
    with pytest.raises(NotImplementedError, match="at most 8"):
        extract_gaussian_spec(GaussianMixture(9, random_state=0).fit(X).score_samples)
    # a singular QDA class: a zero (or non-finite) scaling
    for v in (0.0, np.nan):
        sing = QuadraticDiscriminantAnalysis(reg_param=0.1).fit(X, y)
        sing.scalings_[1] = sing.scalings_[1].copy()
        sing.scalings_[1][-1] = v
        with pytest.raises(NotImplementedError, match="zero or non-finite scaling"):
            extract_gaussian_spec(sing.predict_proba)
    # a materially negative precision eigenvalue
    e2 = EllipticEnvelope(random_state=0).fit(X)
    e2.precision_ = e2.precision_ - 2.0 * np.abs(np.linalg.eigvalsh(e2.precision_)).max() * np.eye(X.shape[1])
    with pytest.raises(NotImplementedError, match="negative eigenvalue"):
        extract_gaussian_spec(e2.decision_function)
    # a step that does not fold
    with pytest.raises(NotImplementedError, match="only StandardScaler"):
        extract_gaussian_spec(make_pipeline(PolynomialFeatures(2), GaussianNB()).fit(X, y).predict_proba)
    # Gaussian members of soft-voting and stacking ensembles
    vote = VotingClassifier([("q", QuadraticDiscriminantAnalysis(reg_param=0.1)),
                             ("rf", RandomForestClassifier(n_estimators=3, random_state=0))], voting="soft").fit(X, y)
    stack = StackingClassifier([("nb", GaussianNB()), ("lr", LogisticRegression())]).fit(X, y)
    for fn in (vote.predict_proba, stack.predict_proba, make_pipeline(StandardScaler(), vote).fit(X, y).predict_proba):
        with pytest.raises(NotImplementedError, match="inside an ensemble"):
            refuse_gaussian_members(fn)
        with pytest.raises(NotImplementedError, match="inside an ensemble"):
            extract_gaussian_spec(fn)
    # NaN or infinity in a row
    spec = extract_gaussian_spec(qda.predict_proba)
    for v in (np.nan, np.inf, -np.inf):
        Z = Q[:3].copy()
        Z[1, 2] = v
        with pytest.raises(ValueError, match="NaN or an infinity"):
            spec(Z)
    # anything else is not a Gaussian model
    assert extract_gaussian_spec(LogisticRegression().fit(X, y).predict_proba) is None
    assert extract_gaussian_spec(lambda Z: Z) is None
