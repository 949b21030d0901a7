"""Kernel machines of scikit-learn read into support vectors in raw feature space (``KernelMachineSpec``) for the device's
kernel-machine route.

A spec is what ``dks_set_kernel_machine`` takes (include/dks.h).  Every kernel is ``phi(t)`` of a statistic that adds up
over columns, ``t = sum_c h(x_c, v_c)``:

* ``rbf``: ``h = w_c (x_c - v_c)^2``, ``phi = exp(-gamma t)``;
* ``laplacian`` (KernelRidge only): ``h = w_c |x_c - v_c|``, ``phi = exp(-gamma t)``;
* ``poly``: ``h = w_c (x_c - o_c)(v_c - o_c)``, ``phi = (gamma t + coef0)^degree``;
* ``sigmoid``: the same ``h``, ``phi = tanh(gamma t + coef0)``.

Without preprocessing ``w_c = 1`` and ``o_c = 0``.  A ``Pipeline`` of per-column affine scalers in front of the model,
``x'_c = a_c x_c + b_c``, folds in exactly: the support vector is taken back to raw space, ``v_c = (v'_c - b_c) / a_c``,
and ``w_c = a_c^2`` (``|a_c|`` for the laplacian), ``o_c = -b_c / a_c``.  Each member of a calibrated ensemble has its own
support vectors, weights, origins and gamma.

Member score ``f_k = sum_v dual[v] phi(t(x, v)) + intercept_k``; heads:

* identity: ``SVC`` / ``NuSVC`` ``decision_function`` (two classes), ``SVR`` / ``NuSVR`` / ``KernelRidge`` ``predict``
  (1 to 8 targets);
* calibrated: ``CalibratedClassifierCV(SVC | NuSVC, method='sigmoid')`` ``predict_proba`` over two classes,
  ``p1 = sum_k pi_k expit(-(a_k f_k + b_k))`` with ``pi_k = 1 / K``, outputs ``[1 - p1, p1]``.

``KernelMachineSpec.__call__`` evaluates the same thing in NumPy.
"""
import numpy as np

MAX_OUTPUTS = 8
MAX_MEMBERS = 16
MAX_GROUPS = 64
KERNELS = ("rbf", "laplacian", "poly", "sigmoid")     # DKS_KM_KERNEL_* codes 0..3
HEADS = ("identity", "calibrated")                    # DKS_KM_HEAD_* codes 0..1

_SVM_CLASSIFIERS = {"SVC", "NuSVC"}
_SVM_REGRESSORS = {"SVR", "NuSVR"}
_KRR = {"KernelRidge"}
_KERNEL_MACHINES = _SVM_CLASSIFIERS | _SVM_REGRESSORS | _KRR
_SCALERS = {"StandardScaler", "MinMaxScaler", "MaxAbsScaler", "RobustScaler"}


class KernelMachineSpec:
    """Support vectors of a kernel machine in raw feature space, per member, and its head.

    sv [n_sv, D] float64, sv_off [K + 1] int32 (member k owns rows sv_off[k] .. sv_off[k + 1]), dual [n_sv, R],
    intercept [K, R], colw / colo [K, D] (column weights and origins), gamma [K], kernel in ``KERNELS``, degree, coef0,
    head in ``HEADS``; the calibrated head's cal_a, cal_b, pi [K]."""

    activation = "kmach"
    act_code = 7          # DKS_ACT_KMACH
    maps = None

    def __init__(self, sv, sv_off, dual, intercept, colw, colo, gamma, kernel, degree, coef0, head, n_features,
                 cal_a=None, cal_b=None, pi=None, scalar_out=False):
        self.sv = np.ascontiguousarray(np.atleast_2d(sv), dtype=np.float64)
        self.sv_off = np.ascontiguousarray(sv_off, dtype=np.int32)
        self.dual = np.ascontiguousarray(np.asarray(dual, dtype=np.float64).reshape(self.sv.shape[0], -1))
        self.K = len(self.sv_off) - 1
        self.R = self.dual.shape[1]
        self.intercept = np.ascontiguousarray(np.asarray(intercept, dtype=np.float64).reshape(self.K, self.R))
        self.colw = np.ascontiguousarray(np.asarray(colw, dtype=np.float64).reshape(self.K, -1))
        self.colo = np.ascontiguousarray(np.asarray(colo, dtype=np.float64).reshape(self.K, -1))
        self.gamma = np.ascontiguousarray(np.atleast_1d(gamma), dtype=np.float64)
        self.kernel = kernel
        self.degree = float(degree)
        self.coef0 = float(coef0)
        self.head = head
        self.n_features = int(n_features)
        self.scalar_out = bool(scalar_out)
        if kernel not in KERNELS:
            raise ValueError(f"unknown kernel {kernel!r}")
        if head not in HEADS:
            raise ValueError(f"unknown kernel-machine head {head!r}")
        if head == "calibrated":
            self.cal_a = np.ascontiguousarray(cal_a, dtype=np.float64)
            self.cal_b = np.ascontiguousarray(cal_b, dtype=np.float64)
            self.pi = np.ascontiguousarray(pi if pi is not None else np.full(self.K, 1.0 / self.K), dtype=np.float64)
        else:
            self.cal_a = self.cal_b = None
            self.pi = np.ones(self.K)
        self.n_outputs = 2 if head == "calibrated" else self.R
        if self.n_outputs > MAX_OUTPUTS:
            raise NotImplementedError(f"{self.n_outputs} model outputs: kernel machines are explained up to {MAX_OUTPUTS}")
        if self.K > MAX_MEMBERS:
            raise NotImplementedError(f"{self.K} calibrated members: kernel machines are explained up to {MAX_MEMBERS}")

    @property
    def kernel_code(self):
        return KERNELS.index(self.kernel)

    @property
    def head_code(self):
        return HEADS.index(self.head)

    @property
    def n_sv(self):
        return int(self.sv_off[-1])

    def statistic(self, X, k):
        """t [n, n_sv of member k] of the rows of X."""
        V = self.sv[self.sv_off[k]:self.sv_off[k + 1]]
        w, o = self.colw[k], self.colo[k]
        if self.kernel == "rbf":
            return ((X[:, None, :] - V[None, :, :]) ** 2 * w).sum(axis=2)
        if self.kernel == "laplacian":
            return (np.abs(X[:, None, :] - V[None, :, :]) * w).sum(axis=2)
        return ((X - o) * w) @ (V - o).T

    def kernel_values(self, t, k):
        if self.kernel in ("rbf", "laplacian"):
            return np.exp(-self.gamma[k] * t)
        u = self.gamma[k] * t + self.coef0
        return u ** self.degree if self.kernel == "poly" else np.tanh(u)

    def scores(self, X):
        """Member scores f [n, K, R]."""
        X = np.atleast_2d(np.asarray(X, dtype=np.float64))
        out = np.empty((X.shape[0], self.K, self.R))
        for k in range(self.K):
            Kv = self.kernel_values(self.statistic(X, k), k)
            out[:, k, :] = Kv @ self.dual[self.sv_off[k]:self.sv_off[k + 1]] + self.intercept[k]
        return out

    def __call__(self, X):
        """The scikit-learn method the spec was read from, in NumPy."""
        f = self.scores(X)
        if self.head == "calibrated":
            z = self.cal_a * f[:, :, 0] + self.cal_b
            p1 = (self.pi / (1.0 + np.exp(z))).sum(axis=1)
            p0 = (self.pi / (1.0 + np.exp(-z))).sum(axis=1)
            out = np.stack([p0, p1], axis=1)
        else:
            out = f[:, 0, :]
        return out[:, 0] if self.scalar_out else out


def _names(obj):
    return {c.__name__ for c in type(obj).__mro__ if c.__module__.startswith("sklearn.")}


def _final(est):
    """The last step of a Pipeline (the estimator itself otherwise)."""
    while "Pipeline" in _names(est):
        est = est.steps[-1][1]
    return est


def _is_kernel_machine(est):
    """A kernel machine with a non-linear kernel (linear SVMs stay on the linear route)."""
    est = _final(est)
    names = _names(est)
    if names & (_SVM_CLASSIFIERS | _SVM_REGRESSORS):
        return getattr(est, "kernel", None) != "linear"
    return bool(names & _KRR)


def _affine(step, family="kernel machine"):
    """(a, b) of a fitted per-column affine scaler: x' = a x + b.  ``family`` names the model in refusals."""
    name = type(step).__name__
    P = int(step.n_features_in_)
    a, b = np.ones(P), np.zeros(P)
    if name == "StandardScaler":
        if step.scale_ is not None:
            a = 1.0 / np.asarray(step.scale_, dtype=np.float64)
        if step.mean_ is not None and step.with_mean:
            b = -np.asarray(step.mean_, dtype=np.float64) * a
    elif name == "RobustScaler":
        if step.scale_ is not None:
            a = 1.0 / np.asarray(step.scale_, dtype=np.float64)
        if step.center_ is not None:
            b = -np.asarray(step.center_, dtype=np.float64) * a
    elif name == "MinMaxScaler":
        if step.clip:
            raise NotImplementedError(f"MinMaxScaler(clip=True) is not affine: {family}s fold affine scalers only")
        a, b = np.asarray(step.scale_, dtype=np.float64), np.asarray(step.min_, dtype=np.float64)
    elif name == "MaxAbsScaler":
        a = 1.0 / np.asarray(step.scale_, dtype=np.float64)
    return a, b


def _unwrap(est, P, family="kernel machine", target="its support vectors"):
    """(final estimator, a, b) with the pipeline's scalers composed into x' = a x + b.  ``family`` and ``target`` (what
    the scalers fold into) name the model in refusals."""
    a, b = np.ones(P), np.zeros(P)
    while "Pipeline" in _names(est):
        for name, step in est.steps[:-1]:
            if step is None or step == "passthrough":
                continue
            if type(step).__name__ not in _SCALERS:
                raise NotImplementedError(f"Pipeline step {name!r} ({type(step).__name__}) in front of a {family}: "
                                          "only StandardScaler, MinMaxScaler, MaxAbsScaler and RobustScaler fold into "
                                          f"{target}")
            sa, sb = _affine(step, family)
            a, b = sa * a, sa * b + sb
        est = est.steps[-1][1]
    if not (np.all(np.isfinite(a)) and np.all(np.isfinite(b)) and np.all(a != 0)):
        raise NotImplementedError(f"a scaler with a zero or non-finite scale cannot be folded into a {family}")
    return est, a, b


def _kernel_params(est, P):
    """(kernel, gamma, degree, coef0) resolved as scikit-learn evaluates them."""
    name = type(est).__name__
    kernel = est.kernel
    if callable(kernel) or kernel == "precomputed":
        raise NotImplementedError(f"{name}(kernel={'a callable' if callable(kernel) else repr(kernel)}) is not supported: "
                                  f"kernels {KERNELS[0]!r}, {KERNELS[2]!r}, {KERNELS[3]!r} (and 'laplacian' for "
                                  "KernelRidge) only")
    if kernel == "polynomial":
        kernel = "poly"
    allowed = KERNELS if name in _KRR else ("rbf", "poly", "sigmoid")
    if kernel not in allowed:
        raise NotImplementedError(f"{name}(kernel={kernel!r}) is not supported: kernels {', '.join(map(repr, allowed))}")
    if name in _KRR:
        if getattr(est, "kernel_params", None):
            raise NotImplementedError("KernelRidge with kernel_params is not supported")
        gamma = 1.0 / P if est.gamma is None else float(est.gamma)
        degree, coef0 = est.degree, float(est.coef0)
    else:
        gamma, degree, coef0 = float(est._gamma), est.degree, float(est.coef0)
    degree = float(degree)
    if kernel == "poly" and not (np.isfinite(degree) and degree >= 0 and degree == int(degree)):
        raise NotImplementedError(f"{name}(kernel='poly', degree={degree!r}): the polynomial degree must be an integer "
                                  ">= 0 (scikit-learn produces NaN for a fractional one)")
    return kernel, gamma, degree, coef0


def _dense(a):
    return np.asarray(a.toarray() if hasattr(a, "toarray") else a, dtype=np.float64)


def _member(est, P):
    """(kernel params, raw-space support vectors, dual [n_sv, R], intercept [R], colw, colo) of one fitted model behind
    its scalers."""
    est, a, b = _unwrap(est, P)
    names = _names(est)
    if not (names & _KERNEL_MACHINES):
        raise NotImplementedError(f"{type(est).__name__} is not a kernel machine")
    if not hasattr(est, "n_features_in_"):
        raise TypeError(f"{type(est).__name__} is not fitted")
    kernel, gamma, degree, coef0 = _kernel_params(est, P)
    if names & _KRR:
        Vt = _dense(est.X_fit_)
        dual = np.asarray(est.dual_coef_, dtype=np.float64)
        dual = dual.reshape(Vt.shape[0], -1)
        intercept = np.zeros(dual.shape[1])
    else:
        Vt = _dense(est.support_vectors_)
        dual = _dense(est.dual_coef_).T.copy()
        intercept = np.asarray(est.intercept_, dtype=np.float64).reshape(-1)
    V = (Vt - b) / a
    if kernel == "laplacian":
        colw, colo = np.abs(a), np.zeros(P)
    elif kernel == "rbf":
        colw, colo = a * a, np.zeros(P)
    else:
        colw, colo = a * a, -b / a
    return (kernel, gamma, degree, coef0), V, dual, intercept, colw, colo


def _svc_binary(est, what):
    clf = _final(est)
    n = len(clf.classes_)
    if n != 2:
        raise NotImplementedError(f"{what} over {n} classes: its one-vs-one votes are not a head the kernel-machine route "
                                  "evaluates; only two classes are supported")


def _calibrated_spec(owner, method, P, bare=False):
    """The calibrated head over the members' kernel machines; ``bare``: each member is read as its final estimator, its
    pipeline's steps being replayed in front of it (``trees.extract_encoded_pipeline_spec``)."""
    if method != "predict_proba":
        raise TypeError(f"CalibratedClassifierCV.{method} is not supported: pass predict_proba")
    if len(owner.classes_) != 2:
        raise NotImplementedError(f"CalibratedClassifierCV over {len(owner.classes_)} classes of a kernel machine: only "
                                  "two classes are supported")
    members = []
    for cc in owner.calibrated_classifiers_:
        if cc.method != "sigmoid":
            raise NotImplementedError(f"CalibratedClassifierCV(method={cc.method!r}) over a kernel machine: only "
                                      "method='sigmoid' is supported")
        if not (_names(_final(cc.estimator)) & _SVM_CLASSIFIERS):
            raise NotImplementedError(f"CalibratedClassifierCV over {type(_final(cc.estimator)).__name__}: the kernel-"
                                      "machine route calibrates SVC and NuSVC only")
        _svc_binary(cc.estimator, type(_final(cc.estimator)).__name__)
        params, V, dual, icpt, colw, colo = _member(_final(cc.estimator) if bare else cc.estimator, P)
        cal = cc.calibrators[0]
        members.append((params, V, dual, icpt, colw, colo, float(cal.a_), float(cal.b_)))
    kinds = {m[0][0] for m in members}
    if len(kinds) != 1 or len({(m[0][2], m[0][3]) for m in members}) != 1:
        raise NotImplementedError("calibrated members with different kernels, degrees or coef0")
    K = len(members)
    if K > MAX_MEMBERS:
        raise NotImplementedError(f"{K} calibrated members: kernel machines are explained up to {MAX_MEMBERS}")
    sv_off = np.concatenate([[0], np.cumsum([m[1].shape[0] for m in members])])
    return KernelMachineSpec(np.concatenate([m[1] for m in members]), sv_off, np.concatenate([m[2] for m in members]),
                             np.stack([m[3] for m in members]), np.stack([m[4] for m in members]),
                             np.stack([m[5] for m in members]), [m[0][1] for m in members], members[0][0][0],
                             members[0][0][2], members[0][0][3], "calibrated", P,
                             cal_a=[m[6] for m in members], cal_b=[m[7] for m in members], pi=np.full(K, 1.0 / K))


def _single_spec(owner, method, P):
    est = _final(owner)
    name = type(est).__name__
    names = _names(est)
    if names & _SVM_CLASSIFIERS:
        if method == "predict_proba":
            raise NotImplementedError(f"{name}(probability=True).predict_proba is not supported (its Platt scaling is "
                                      "deprecated in scikit-learn): explain CalibratedClassifierCV("
                                      f"{name}(), ensemble=False).predict_proba instead")
        if method != "decision_function":
            raise TypeError(f"{name}.{method} is not supported: pass decision_function (predict returns labels)")
        _svc_binary(est, name)
    elif method != "predict":
        raise TypeError(f"{name}.{method} is not supported: pass predict")
    params, V, dual, icpt, colw, colo = _member(owner, P)
    if dual.shape[1] > MAX_OUTPUTS:
        raise NotImplementedError(f"{dual.shape[1]} targets: kernel machines are explained up to {MAX_OUTPUTS} outputs")
    scalar = True
    if names & _KRR:
        scalar = np.ndim(est.dual_coef_) == 1
    kernel, gamma, degree, coef0 = params
    return KernelMachineSpec(V, [0, V.shape[0]], dual, icpt[None, :], colw[None, :], colo[None, :], [gamma], kernel,
                             degree, coef0, "identity", P, scalar_out=scalar)


def extract_kernel_machine_spec(predictor):
    """``KernelMachineSpec`` of a bound method of a fitted scikit-learn kernel machine -- ``SVC`` / ``NuSVC``
    ``decision_function``, ``SVR`` / ``NuSVR`` / ``KernelRidge`` ``predict``, ``CalibratedClassifierCV(SVC | NuSVC,
    method='sigmoid').predict_proba``, each possibly behind a ``Pipeline`` of per-column affine scalers -- and ``None``
    for anything else (linear SVMs included: the engine then reads a linear model).  A spec passes through.  Raises
    ``NotImplementedError`` / ``TypeError`` naming the reason for kernel machines the route does not cover: more than two
    classes, ``SVC(probability=True).predict_proba``, precomputed, callable and chi2 kernels, a non-integer or negative
    polynomial degree, pipeline steps other than the four affine scalers, calibration other than 'sigmoid'."""
    if isinstance(predictor, KernelMachineSpec):
        return predictor
    owner = getattr(predictor, "__self__", None)
    method = getattr(predictor, "__name__", None)
    if owner is None:
        return None
    outer = _final(owner)
    if "CalibratedClassifierCV" in _names(outer):
        ccs = getattr(outer, "calibrated_classifiers_", None)
        if not ccs or not any(_is_kernel_machine(cc.estimator) for cc in ccs):
            return None
        P = int(owner.n_features_in_)
        spec = _calibrated_spec(outer, method, P)
        if outer is not owner:                          # scalers in front of the calibrated classifier
            _, a, b = _unwrap(owner, P)
            spec = _fold_outer(spec, a, b)
        return spec
    if not _is_kernel_machine(owner):
        return None
    if callable(outer.kernel) or outer.kernel == "precomputed":
        _kernel_params(outer, 0)                        # raises, naming the kernel
    if not hasattr(outer, "n_features_in_"):
        raise TypeError(f"{type(outer).__name__} is not fitted")
    return _single_spec(owner, method, int(owner.n_features_in_))


def _fold_outer(spec, a, b):
    """The spec of the model behind one more affine map x' = a x + b of its raw columns."""
    if spec.kernel == "laplacian":
        colw = spec.colw * np.abs(a)
    else:
        colw = spec.colw * a * a
    colo = (spec.colo - b) / a
    return KernelMachineSpec((spec.sv - b) / a, spec.sv_off, spec.dual, spec.intercept, colw, colo, spec.gamma,
                             spec.kernel, spec.degree, spec.coef0, spec.head, spec.n_features, cal_a=spec.cal_a,
                             cal_b=spec.cal_b, pi=spec.pi, scalar_out=spec.scalar_out)
