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

Gaussian-process regressors (``predict``: ``K(x, X_train_) alpha_``, un-normalised), ``KernelRidge`` with a scikit-learn
``Kernel`` object and one-class SVMs (``decision_function``, ``score_samples``) share the identity head.  A one-class SVM
with ``rbf`` / ``poly`` / ``sigmoid`` takes the kernels above; a ``Kernel`` object (scikit-learn's kernel algebra) is read
into the ``program`` kernel: at most ``MAX_STATS`` additive statistics, each ``sqdist`` (``h = w_c (x_c - v_c)^2``) or
``dot`` (``h = w_c (x_c - o_c)(v_c - o_c)``) with its own column weights and origins, and a short postfix expression over
them (``KernelProgram``, ``dks_set_kernel_program``).

Multi-class ``SVC`` / ``NuSVC`` (3 to 8 classes) are read into ``MulticlassSvmSpec``, the one-vs-one head
(``dks_set_svc_multiclass``): support vectors in class blocks, ``dual [n_sv, classes - 1]`` and one intercept per class
pair.  Its outputs are the pair values of ``decision_function_shape='ovo'`` or the probabilities of
``CalibratedClassifierCV(SVC | NuSVC, method='sigmoid')``, which calibrates the ovr-vote decision function per class.

``KernelMachineSpec.__call__`` evaluates the same thing in NumPy.
"""
import numpy as np

MAX_OUTPUTS = 8
MAX_MEMBERS = 16
MAX_GROUPS = 64
KERNELS = ("rbf", "laplacian", "poly", "sigmoid", "program")  # DKS_KM_KERNEL_* codes 0..4
HEADS = ("identity", "calibrated")                    # DKS_KM_HEAD_* codes 0..1
STATS = ("sqdist", "dot")                             # DKS_KM_STAT_* codes 0..1
OPS = ("const", "stat", "exp", "matern05", "matern15", "matern25", "rq", "expsine", "add", "mul", "pow", "addc",
       "mulc")                                        # DKS_KM_OP_* codes 0..12
MAX_STATS = 4                                         # DKS_KM_MAX_STATS
MAX_OPS = 32                                          # DKS_KM_MAX_OPS
MAX_STACK = 4                                         # DKS_KM_MAX_STACK
OVO_MODES = ("ovo", "ovo_proba")                      # DKS_KM_OVO_* codes 0..1
OVO_HEAD = 2                                          # DKS_KM_HEAD_OVO
MAX_CLASSES = 8                                       # DKS_KM_OVO_MAX_CLASSES

_SVM_CLASSIFIERS = {"SVC", "NuSVC"}
_SVM_REGRESSORS = {"SVR", "NuSVR"}
_KRR = {"KernelRidge"}
_GPR = {"GaussianProcessRegressor"}
_OCSVM = {"OneClassSVM"}
_KERNEL_MACHINES = _SVM_CLASSIFIERS | _SVM_REGRESSORS | _KRR | _GPR | _OCSVM
# leaves and operators of scikit-learn's kernel algebra the program kernel reads
_GP_KERNELS = {"RBF", "Matern", "RationalQuadratic", "ExpSineSquared", "DotProduct", "ConstantKernel", "WhiteKernel", "Sum",
               "Product", "Exponentiation"}
_MATERN_OPS = {0.5: "matern05", 1.5: "matern15", 2.5: "matern25"}


class KernelProgram:
    """The kernel of a ``Kernel`` object as L <= ``MAX_STATS`` additive statistics and a postfix expression over them.

    kinds [L] in ``STATS``; colw / colo [L, D] (column weights and origins, scalers folded in); ops: a list of
    ``(op, arg, a, b)`` with op in ``OPS``.  Leaves push a value: ``const`` a; ``stat`` t_arg; ``exp`` exp(-a t);
    ``matern05/15/25`` scikit-learn's closed forms of r = sqrt(t); ``rq`` (1 + t)^a; ``expsine``
    exp(-2 (sin(pi r / a) / b)^2).  ``add`` / ``mul`` pop two, ``pow`` / ``addc`` / ``mulc`` apply a to the top."""

    def __init__(self, kinds, colw, colo, ops):
        self.kinds = list(kinds)
        self.colw = np.ascontiguousarray(np.asarray(colw, dtype=np.float64).reshape(len(self.kinds), -1))
        self.colo = np.ascontiguousarray(np.asarray(colo, dtype=np.float64).reshape(len(self.kinds), -1))
        self.ops = [(str(o), int(g), float(a), float(b)) for o, g, a, b in ops]
        if not 1 <= self.L <= MAX_STATS:
            raise NotImplementedError(f"a kernel of {self.L} statistics: the program kernel takes 1 to {MAX_STATS}")
        if len(self.ops) > MAX_OPS:
            raise NotImplementedError(f"a kernel expression of {len(self.ops)} operations: up to {MAX_OPS} are supported")
        if self.depth() > MAX_STACK:
            raise NotImplementedError(f"a kernel expression {self.depth()} operands deep: up to {MAX_STACK} are supported")

    @property
    def L(self):
        return len(self.kinds)

    def depth(self):
        d = top = 0
        for op, *_ in self.ops:
            top += 1 if op in ("const", "stat", "exp", "matern05", "matern15", "matern25", "rq", "expsine") else (
                -1 if op in ("add", "mul") else 0)
            d = max(d, top)
        return d

    @property
    def kind_codes(self):
        return np.asarray([STATS.index(k) for k in self.kinds], dtype=np.int32)

    def flat(self):
        """(op codes [n], args [n] int32, a [n], b [n] float64) for ``dks_set_kernel_program``."""
        return (np.asarray([OPS.index(o[0]) for o in self.ops], dtype=np.int32),
                np.asarray([o[1] for o in self.ops], dtype=np.int32),
                np.asarray([o[2] for o in self.ops], dtype=np.float64),
                np.asarray([o[3] for o in self.ops], dtype=np.float64))

    def statistics(self, X, V):
        """t_l [n, n_v] of the rows of X against the rows V, per statistic."""
        out = []
        for kind, w, o in zip(self.kinds, self.colw, self.colo):
            if kind == "sqdist":
                out.append(((X[:, None, :] - V[None, :, :]) ** 2 * w).sum(axis=2))
            else:
                out.append(((X - o) * w) @ (V - o).T)
        return out

    def __call__(self, t):
        """Kernel values of the statistics t (list of arrays), in the device's order."""
        st = []
        for op, g, a, b in self.ops:
            if op == "const":
                st.append(np.full(t[0].shape, a))
            elif op == "stat":
                st.append(t[g])
            elif op == "exp":
                st.append(np.exp(-a * t[g]))
            elif op in ("matern05", "matern15", "matern25", "expsine"):
                r = np.sqrt(np.maximum(t[g], 0.0))
                if op == "matern05":
                    st.append(np.exp(-r))
                elif op == "matern15":
                    k = r * np.sqrt(3.0)
                    st.append((1.0 + k) * np.exp(-k))
                elif op == "matern25":
                    k = r * np.sqrt(5.0)
                    st.append((1.0 + k + k * k / 3.0) * np.exp(-k))
                else:
                    st.append(np.exp(-2.0 * (np.sin(np.pi * r / a) / b) ** 2))
            elif op == "rq":
                st.append((1.0 + t[g]) ** a)
            elif op in ("add", "mul"):
                y = st.pop()
                st[-1] = st[-1] + y if op == "add" else st[-1] * y
            elif op == "pow":
                st[-1] = st[-1] ** a
            elif op == "addc":
                st[-1] = st[-1] + a
            else:
                st[-1] = st[-1] * a
        return st[0]

    def folded(self, a, b):
        """The program behind one more affine map x' = a x + b of its raw columns."""
        return KernelProgram(self.kinds, self.colw * a * a,
                             np.stack([(o - b) / a if k == "dot" else o for k, o in zip(self.kinds, self.colo)]),
                             self.ops)
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
                 cal_a=None, cal_b=None, pi=None, scalar_out=False, program=None):
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
        self.program = program
        if kernel not in KERNELS:
            raise ValueError(f"unknown kernel {kernel!r}")
        if (kernel == "program") != (program is not None) or (program is not None and (head != "identity" or self.K != 1)):
            raise ValueError("the program kernel takes a KernelProgram, one member and the identity head")
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
            if self.program is not None:
                Kv = self.program(self.program.statistics(X, self.sv[self.sv_off[k]:self.sv_off[k + 1]]))
            else:
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


class MulticlassSvmSpec(KernelMachineSpec):
    """A multi-class SVC / NuSVC (3 to ``MAX_CLASSES`` classes) under the one-vs-one head, per member (calibration fold).

    sv [n_sv, D], sv_off [K + 1]; cls_off [K, classes + 1] absolute rows of each member's class blocks; dual
    [n_sv, classes - 1] (``dual_coef_`` transposed), intercept [K, P] with P = classes (classes - 1) / 2; colw / colo
    [K, D], gamma [K], kernel ``rbf`` / ``poly`` / ``sigmoid``, degree, coef0.  head ``ovo``: one member, the P pair
    values of ``decision_function_shape='ovo'``; ``ovo_proba``: cal_a / cal_b [K, classes] and pi [K], the calibrated
    probabilities of ``CalibratedClassifierCV``."""

    def __init__(self, sv, sv_off, cls_off, dual, intercept, colw, colo, gamma, kernel, degree, coef0, head, n_features,
                 classes, cal_a=None, cal_b=None, pi=None, scalar_out=False):
        self.classes = int(classes)
        if not 3 <= self.classes <= MAX_CLASSES:
            raise NotImplementedError(f"a multi-class SVM over {self.classes} classes: 3 to {MAX_CLASSES} are supported")
        self.P = self.classes * (self.classes - 1) // 2
        self.sv = np.ascontiguousarray(np.atleast_2d(sv), dtype=np.float64)
        self.sv_off = np.ascontiguousarray(sv_off, dtype=np.int32)
        self.K = len(self.sv_off) - 1
        self.cls_off = np.ascontiguousarray(np.asarray(cls_off, dtype=np.int32).reshape(self.K, self.classes + 1))
        self.R = self.classes - 1
        self.dual = np.ascontiguousarray(np.asarray(dual, dtype=np.float64).reshape(self.sv.shape[0], self.R))
        self.intercept = np.ascontiguousarray(np.asarray(intercept, dtype=np.float64).reshape(self.K, self.P))
        self.colw = np.ascontiguousarray(np.asarray(colw, dtype=np.float64).reshape(self.K, -1))
        self.colo = np.ascontiguousarray(np.asarray(colo, dtype=np.float64).reshape(self.K, -1))
        self.gamma = np.ascontiguousarray(np.atleast_1d(gamma), dtype=np.float64)
        self.kernel = kernel
        self.degree = float(degree)
        self.coef0 = float(coef0)
        self.head = head
        self.n_features = int(n_features)
        self.scalar_out = bool(scalar_out)
        self.program = None
        if kernel not in ("rbf", "poly", "sigmoid"):
            raise ValueError(f"kernel {kernel!r}: the one-vs-one head takes 'rbf', 'poly' and 'sigmoid'")
        if head not in OVO_MODES:
            raise ValueError(f"unknown one-vs-one head {head!r}")
        if self.K > MAX_MEMBERS:
            raise NotImplementedError(f"{self.K} calibrated members: kernel machines are explained up to {MAX_MEMBERS}")
        if head == "ovo":
            if self.K != 1:
                raise ValueError("the pair values of decision_function_shape='ovo' take one member")
            if self.P > MAX_OUTPUTS:
                raise NotImplementedError(
                    f"SVC(decision_function_shape='ovo').decision_function over {self.classes} classes gives {self.P} "
                    f"pair values: up to {MAX_OUTPUTS} outputs (4 classes) are supported; explain "
                    "CalibratedClassifierCV(SVC(), ensemble=False).predict_proba instead")
            self.cal_a = self.cal_b = np.zeros((self.K, self.classes))
            self.pi = np.ones(self.K)
            self.n_outputs = self.P
        else:
            self.cal_a = np.ascontiguousarray(np.asarray(cal_a, dtype=np.float64).reshape(self.K, self.classes))
            self.cal_b = np.ascontiguousarray(np.asarray(cal_b, dtype=np.float64).reshape(self.K, self.classes))
            self.pi = np.ascontiguousarray(pi if pi is not None else np.full(self.K, 1.0 / self.K), dtype=np.float64)
            self.n_outputs = self.classes

    @property
    def head_code(self):
        return OVO_HEAD

    @property
    def mode_code(self):
        return OVO_MODES.index(self.head)

    def pairs(self):
        """[(i, j)] of the class pairs in scikit-learn's order."""
        return [(i, j) for i in range(self.classes) for j in range(i + 1, self.classes)]

    def pair_values(self, X):
        """dec [n, K, P] of every member, pairs in scikit-learn's order."""
        X = np.atleast_2d(np.asarray(X, dtype=np.float64))
        out = np.empty((X.shape[0], self.K, self.P))
        for m in range(self.K):
            Kv = self.kernel_values(self.statistic(X, m), m)
            o = self.cls_off[m] - self.sv_off[m]
            for k, (i, j) in enumerate(self.pairs()):
                bi, bj = slice(o[i], o[i + 1]), slice(o[j], o[j + 1])
                du = self.dual[self.sv_off[m]:self.sv_off[m + 1]]
                out[:, m, k] = Kv[:, bi] @ du[bi, j - 1] + Kv[:, bj] @ du[bj, i] + self.intercept[m, k]
        return out

    def __call__(self, X):
        """The scikit-learn method the spec was read from, in NumPy."""
        dec = self.pair_values(X)
        if self.head == "ovo":
            out = dec[:, 0, :]
        else:
            out = np.zeros((dec.shape[0], self.classes))
            for m in range(self.K):
                votes = np.zeros_like(out)
                conf = np.zeros_like(out)
                for k, (i, j) in enumerate(self.pairs()):
                    d = dec[:, m, k]
                    votes[:, i] += d >= 0
                    votes[:, j] += d < 0
                    conf[:, i] += d
                    conf[:, j] -= d
                f = votes + conf / (3.0 * (np.abs(conf) + 1.0))
                with np.errstate(over="ignore"):                # expit of a very negative argument is 0
                    e = 1.0 / (1.0 + np.exp(self.cal_a[m] * f + self.cal_b[m]))
                tot = e.sum(axis=1, keepdims=True)
                p = np.divide(e, tot, out=np.full_like(e, 1.0 / self.classes), where=tot != 0)
                p[(p > 1.0) & (p <= 1.0 + 1e-5)] = 1.0
                out += self.pi[m] * p
        return out[:, 0] if self.scalar_out else out


def _names(obj):
    return {c.__name__ for c in type(obj).__mro__ if c.__module__.startswith("sklearn.")}


def _final(est):
    """The last step of a Pipeline (the estimator itself otherwise)."""
    while "Pipeline" in _names(est):
        est = est.steps[-1][1]
    return est


def _is_kernel_machine(est):
    """A kernel machine with a non-linear kernel (linear SVMs stay on the linear route), a Gaussian process (classifiers
    included: the extractor refuses them by name) or a one-class SVM."""
    est = _final(est)
    names = _names(est)
    if names & (_SVM_CLASSIFIERS | _SVM_REGRESSORS):
        return getattr(est, "kernel", None) != "linear"
    return bool(names & (_KRR | _GPR | _OCSVM | {"GaussianProcessClassifier"}))


def _is_kernel_object(k):
    """A scikit-learn ``gaussian_process.kernels.Kernel`` (any subclass)."""
    return any(c.__name__ == "Kernel" and c.__module__ == "sklearn.gaussian_process.kernels" for c in type(k).__mro__)


def _kernel_tree(k, P, stats):
    """Expression tree of a scikit-learn kernel object over the columns it reads; ``stats`` collects the statistics
    ``(kind, colw)`` the leaves read (equal ones shared).  Constants fold."""
    name = type(k).__name__
    if type(k).__module__ != "sklearn.gaussian_process.kernels" or name not in _GP_KERNELS:
        what = "a user-defined kernel" if type(k).__module__ != "sklearn.gaussian_process.kernels" else name
        raise NotImplementedError(f"{what} ({name}) is not supported: the kernel-machine route reads "
                                  f"{', '.join(sorted(_GP_KERNELS))}")

    def stat(kind, w):
        w = np.ascontiguousarray(np.broadcast_to(np.asarray(w, dtype=np.float64), (P,)))
        for i, (kd, sw) in enumerate(stats):
            if kd == kind and np.array_equal(sw, w):
                return i
        stats.append((kind, w))
        return len(stats) - 1

    def scales(ls):
        ls = np.asarray(ls, dtype=np.float64)
        if ls.ndim > 0 and ls.size != P:
            raise NotImplementedError(f"{name} with {ls.size} length scales over {P} columns")
        return ls

    if name in ("Sum", "Product"):
        x, y = _kernel_tree(k.k1, P, stats), _kernel_tree(k.k2, P, stats)
        return _node_add(x, y) if name == "Sum" else _node_mul(x, y)
    if name == "Exponentiation":
        return _node_pow(_kernel_tree(k.kernel, P, stats), float(k.exponent))
    if name == "ConstantKernel":
        return ("c", float(k.constant_value))
    if name == "WhiteKernel":
        return ("c", 0.0)                               # k(X, Y) is zero whenever Y is given (every prediction)
    if name == "DotProduct":
        return _node_add(("leaf", "stat", stat("dot", 1.0), 0.0, 0.0), ("c", float(k.sigma_0) ** 2))
    if name == "ExpSineSquared":
        return ("leaf", "expsine", stat("sqdist", 1.0), float(k.periodicity), float(k.length_scale))
    if name == "RationalQuadratic":
        ls, al = float(k.length_scale), float(k.alpha)
        return ("leaf", "rq", stat("sqdist", 1.0 / (2.0 * al * ls ** 2)), -al, 0.0)
    ls = scales(k.length_scale)
    if name == "RBF":
        return ("leaf", "exp", stat("sqdist", 1.0 / ls ** 2), 0.5, 0.0)
    nu = float(k.nu)                                    # Matern
    if np.isinf(nu):
        return ("leaf", "exp", stat("sqdist", 1.0 / ls ** 2), 0.5, 0.0)
    if nu not in _MATERN_OPS:
        raise NotImplementedError(f"Matern(nu={nu!r}) is not supported: nu 0.5, 1.5, 2.5 and inf have closed forms, "
                                  "others need a Bessel function")
    return ("leaf", _MATERN_OPS[nu], stat("sqdist", 1.0 / ls ** 2), 0.0, 0.0)


def _node_add(x, y):
    if x[0] == "c" and y[0] == "c":
        return ("c", x[1] + y[1])
    if x[0] == "c":
        x, y = y, x
    if y[0] == "c":
        return x if y[1] == 0.0 else ("addc", x, y[1])
    return ("add", x, y)


def _node_mul(x, y):
    if x[0] == "c" and y[0] == "c":
        return ("c", x[1] * y[1])
    if x[0] == "c":
        x, y = y, x
    if y[0] == "c":
        return x if y[1] == 1.0 else (("c", 0.0) if y[1] == 0.0 else ("mulc", x, y[1]))
    return ("mul", x, y)


def _node_pow(x, e):
    if x[0] == "c":
        return ("c", x[1] ** e)
    return x if e == 1.0 else ("pow", x, e)


def _need(n):
    """Stack slots the postfix form of node n needs (Sethi-Ullman: the deeper operand goes first)."""
    if n[0] in ("c", "leaf"):
        return 1
    if n[0] in ("addc", "mulc", "pow"):
        return _need(n[1])
    a, b = _need(n[1]), _need(n[2])
    return a + 1 if a == b else max(a, b)


def _emit(n, out):
    if n[0] == "c":
        out.append(("const", 0, n[1], 0.0))
    elif n[0] == "leaf":
        out.append((n[1], n[2], n[3], n[4]))
    elif n[0] in ("addc", "mulc", "pow"):
        _emit(n[1], out)
        out.append((n[0], 0, n[2], 0.0))
    else:
        x, y = (n[1], n[2]) if _need(n[1]) >= _need(n[2]) else (n[2], n[1])
        _emit(x, out)
        _emit(y, out)
        out.append((n[0], 0, 0.0, 0.0))


def _kernel_program(kernel, P):
    """``KernelProgram`` of a scikit-learn kernel object over P columns (no scalers folded yet)."""
    stats = []
    tree = _kernel_tree(kernel, P, stats)
    if tree[0] == "c":
        raise NotImplementedError(f"the kernel {kernel!r} is constant on every prediction: the model does not depend on "
                                  "its input")
    if len(stats) > MAX_STATS:
        raise NotImplementedError(f"the kernel {kernel!r} reads {len(stats)} statistics: the program kernel takes up to "
                                  f"{MAX_STATS}")
    ops = []
    _emit(tree, ops)
    return KernelProgram([kd for kd, _ in stats], np.stack([w for _, w in stats]), np.zeros((len(stats), P)), ops)


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
    if name in _KRR and _is_kernel_object(kernel):
        if getattr(est, "kernel_params", None):
            raise NotImplementedError("KernelRidge with kernel_params is not supported")
        return "program", 0.0, 0.0, 0.0
    if _is_kernel_object(kernel):
        raise NotImplementedError(f"{name}(kernel={type(kernel).__name__}(...)) is not supported: kernel objects are read "
                                  "for GaussianProcessRegressor and KernelRidge only")
    if name in _OCSVM and kernel in ("linear", "precomputed"):
        raise NotImplementedError(f"OneClassSVM(kernel={kernel!r}) is not supported: kernels 'rbf', 'poly' and 'sigmoid'")
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
    """(kernel params, raw-space support vectors, dual [n_sv, R], intercept [R], colw, colo, program) of one fitted model
    behind its scalers (``program``: the ``KernelProgram`` of a kernel object, else None)."""
    est, a, b = _unwrap(est, P)
    names = _names(est)
    if not (names & _KERNEL_MACHINES):
        raise NotImplementedError(f"{type(est).__name__} is not a kernel machine")
    if names & _GPR:
        if not hasattr(est, "X_train_"):
            raise TypeError("GaussianProcessRegressor is not fitted (the prior mean is not explained)")
        Vt = _dense(est.X_train_)
        alpha = np.asarray(est.alpha_, dtype=np.float64).reshape(Vt.shape[0], -1)
        R = alpha.shape[1]
        std = np.broadcast_to(np.asarray(est._y_train_std, dtype=np.float64).reshape(-1), (R,))
        dual = alpha * std                              # predict: std (K alpha) + mean, as scikit-learn un-normalises
        intercept = np.broadcast_to(np.asarray(est._y_train_mean, dtype=np.float64).reshape(-1), (R,)).copy()
        params, program = ("program", 0.0, 0.0, 0.0), _kernel_program(est.kernel_, P)
    else:
        if not hasattr(est, "n_features_in_"):
            raise TypeError(f"{type(est).__name__} is not fitted")
        params = _kernel_params(est, P)
        program = _kernel_program(est.kernel, P) if params[0] == "program" else None
        if names & _KRR:
            Vt = _dense(est.X_fit_)
            dual = np.asarray(est.dual_coef_, dtype=np.float64)
            dual = dual.reshape(Vt.shape[0], -1)
            intercept = np.zeros(dual.shape[1])
        else:
            Vt = _dense(est.support_vectors_)
            dual = _dense(est.dual_coef_).T.copy()
            intercept = np.asarray(est.intercept_, dtype=np.float64).reshape(-1)
    kernel = params[0]
    V = (Vt - b) / a
    if program is not None:
        program = program.folded(a, b)
        colw, colo = np.ones(P), np.zeros(P)
    elif kernel == "laplacian":
        colw, colo = np.abs(a), np.zeros(P)
    elif kernel == "rbf":
        colw, colo = a * a, np.zeros(P)
    else:
        colw, colo = a * a, -b / a
    return params, V, dual, intercept, colw, colo, program


def _svc_classes(est, what):
    """The classes of a fitted SVC / NuSVC: 2, or 3 to ``MAX_CLASSES`` for the one-vs-one head."""
    n = len(_final(est).classes_)
    if n > MAX_CLASSES:
        raise NotImplementedError(f"{what} over {n} classes: the one-vs-one head of the kernel-machine route takes up to "
                                  f"{MAX_CLASSES} classes ({MAX_CLASSES * (MAX_CLASSES - 1) // 2} pairs)")
    return n


def _class_blocks(est, off):
    """cls_off [classes + 1] of a multi-class SVC whose support vectors start at row ``off``."""
    return off + np.concatenate([[0], np.cumsum(np.asarray(_final(est).n_support_, dtype=np.int64))])


def _calibrated_spec(owner, method, P, bare=False):
    """The calibrated head over the members' kernel machines; ``bare``: each member is read as its final estimator, its
    pipeline's steps being replayed in front of it (``trees.extract_encoded_pipeline_spec``)."""
    if method != "predict_proba":
        raise TypeError(f"CalibratedClassifierCV.{method} is not supported: pass predict_proba")
    nc = len(owner.classes_)
    if nc > MAX_CLASSES:
        raise NotImplementedError(f"CalibratedClassifierCV over {nc} classes of a kernel machine: up to {MAX_CLASSES} "
                                  "classes are supported")
    if nc > 2:
        return _calibrated_multiclass_spec(owner, P, bare)
    members = []
    for cc in owner.calibrated_classifiers_:
        if cc.method != "sigmoid":
            raise NotImplementedError(f"CalibratedClassifierCV(method={cc.method!r}) over a kernel machine: only "
                                      "method='sigmoid' is supported")
        if not (_names(_final(cc.estimator)) & _SVM_CLASSIFIERS):
            raise NotImplementedError(f"CalibratedClassifierCV over {type(_final(cc.estimator)).__name__}: the kernel-"
                                      "machine route calibrates SVC and NuSVC only")
        n = len(_final(cc.estimator).classes_)
        if n != 2:
            raise NotImplementedError(f"{type(_final(cc.estimator)).__name__} over {n} classes in a calibration fold of "
                                      "two classes: only folds that hold both classes are supported")
        params, V, dual, icpt, colw, colo, _ = _member(_final(cc.estimator) if bare else cc.estimator, P)
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


def _calibrated_multiclass_spec(owner, P, bare):
    """``_calibrated_spec`` over 3 to ``MAX_CLASSES`` classes: the one-vs-one head's calibrated probabilities."""
    nc = len(owner.classes_)
    members = []
    off = 0
    for cc in owner.calibrated_classifiers_:
        if cc.method != "sigmoid":
            raise NotImplementedError(f"CalibratedClassifierCV(method={cc.method!r}) over a kernel machine: only "
                                      "method='sigmoid' is supported")
        clf = _final(cc.estimator)
        name = type(clf).__name__
        if not (_names(clf) & _SVM_CLASSIFIERS):
            raise NotImplementedError(f"CalibratedClassifierCV over {name}: the kernel-machine route calibrates SVC and "
                                      "NuSVC only")
        if len(clf.classes_) != nc:
            raise NotImplementedError(f"CalibratedClassifierCV over {nc} classes with a fold whose {name} saw "
                                      f"{len(clf.classes_)}: a fold missing classes is not supported (use folds that "
                                      "hold every class)")
        if getattr(clf, "decision_function_shape", "ovr") != "ovr":
            raise NotImplementedError(f"CalibratedClassifierCV over {name}(decision_function_shape="
                                      f"{clf.decision_function_shape!r}): the calibrated probabilities are read from the "
                                      "default 'ovr' shape")
        params, V, dual, icpt, colw, colo, _ = _member(clf if bare else cc.estimator, P)
        cal_a = [float(c.a_) for c in cc.calibrators]
        cal_b = [float(c.b_) for c in cc.calibrators]
        members.append((params, V, dual, icpt, colw, colo, cal_a, cal_b, _class_blocks(clf, off)))
        off += V.shape[0]
    if len({m[0][0] for m in members}) != 1 or len({(m[0][2], m[0][3]) for m in members}) != 1:
        raise NotImplementedError("calibrated members with different kernels, degrees or coef0")
    K = len(members)
    if K > MAX_MEMBERS:
        raise NotImplementedError(f"{K} calibrated members: kernel machines are explained up to {MAX_MEMBERS}")
    sv_off = np.concatenate([[0], np.cumsum([m[1].shape[0] for m in members])])
    return MulticlassSvmSpec(np.concatenate([m[1] for m in members]), sv_off, np.stack([m[8] for m in members]),
                             np.concatenate([m[2] for m in members]), np.stack([m[3] for m in members]),
                             np.stack([m[4] for m in members]), np.stack([m[5] for m in members]),
                             [m[0][1] for m in members], members[0][0][0], members[0][0][2], members[0][0][3],
                             "ovo_proba", P, nc, cal_a=np.stack([m[6] for m in members]),
                             cal_b=np.stack([m[7] for m in members]), pi=np.full(K, 1.0 / K))


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
        nc = _svc_classes(est, name)
        if nc > 2 and est.decision_function_shape != "ovo":
            raise NotImplementedError(
                f"{name}.decision_function over {nc} classes with decision_function_shape='ovr': its integer part counts "
                "one-vs-one votes, a label-like step function the kernel-machine route does not explain; pass "
                f"{name}(decision_function_shape='ovo') for the pair values, or explain "
                f"CalibratedClassifierCV({name}(), ensemble=False).predict_proba")
        if nc > 2:
            params, V, dual, icpt, colw, colo, _ = _member(owner, P)
            kernel, gamma, degree, coef0 = params
            return MulticlassSvmSpec(V, [0, V.shape[0]], _class_blocks(est, 0)[None, :], dual, icpt[None, :],
                                     colw[None, :], colo[None, :], [gamma], kernel, degree, coef0, "ovo", P, nc)
    elif names & _OCSVM:
        if method not in ("decision_function", "score_samples"):
            raise TypeError(f"{name}.{method} is not supported: pass decision_function or score_samples (predict returns "
                            "labels)")
    elif method != "predict":
        raise TypeError(f"{name}.{method} is not supported: pass predict")
    params, V, dual, icpt, colw, colo, program = _member(owner, P)
    if dual.shape[1] > MAX_OUTPUTS:
        raise NotImplementedError(f"{dual.shape[1]} targets: kernel machines are explained up to {MAX_OUTPUTS} outputs")
    scalar = True
    if names & _KRR:
        scalar = np.ndim(est.dual_coef_) == 1
    elif names & _GPR:
        scalar = dual.shape[1] == 1                     # predict squeezes one target
    elif method == "score_samples":
        icpt = icpt + float(np.ravel(est.offset_)[0])
    kernel, gamma, degree, coef0 = params
    return KernelMachineSpec(V, [0, V.shape[0]], dual, icpt[None, :], colw[None, :], colo[None, :], [gamma], kernel,
                             degree, coef0, "identity", P, scalar_out=scalar, program=program)


def extract_kernel_machine_spec(predictor):
    """``KernelMachineSpec`` of a bound method of a fitted scikit-learn kernel machine -- ``SVC`` / ``NuSVC``
    ``decision_function``, ``SVR`` / ``NuSVR`` / ``KernelRidge`` (a ``Kernel`` object included) /
    ``GaussianProcessRegressor`` ``predict``, ``OneClassSVM`` ``decision_function`` / ``score_samples``,
    ``CalibratedClassifierCV(SVC | NuSVC, method='sigmoid').predict_proba``, each possibly behind a ``Pipeline`` of
    per-column affine scalers -- and ``None`` for anything else (linear SVMs included: the engine then reads a linear
    model).  Multi-class SVMs give a ``MulticlassSvmSpec`` (the one-vs-one head): ``SVC`` / ``NuSVC(decision_function_shape=
    'ovo').decision_function`` over 3 or 4 classes (the pair values) and the calibrated ``predict_proba`` over 3 to 8
    classes.  A spec passes through.  Raises ``NotImplementedError`` / ``TypeError`` naming the reason for kernel machines
    the route does not cover: the default ``'ovr'`` ``decision_function`` of a multi-class SVM (a vote count), ``'ovo'``
    with more than 8 pair values, more than 8 classes, a calibration fold that saw fewer classes than the calibrator,
    ``SVC(probability=True).predict_proba``, precomputed, callable and
    chi2 kernels, kernel objects on SVMs, kernel objects outside the program kernel (``Matern`` nu other than 0.5, 1.5,
    2.5, inf, ``PairwiseKernel``, ``CompoundKernel``, user-defined kernels, more than ``MAX_STATS`` statistics),
    ``GaussianProcessClassifier``, unfitted models, a non-integer or negative polynomial degree, pipeline steps other
    than the four affine scalers, calibration other than 'sigmoid'."""
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
    if "GaussianProcessClassifier" in _names(outer):
        raise NotImplementedError("GaussianProcessClassifier is not supported: its predict_proba needs the posterior "
                                  "variance (a triangular solve against every training row per masked row)")
    if not (_names(outer) & _GPR) and (callable(outer.kernel) or outer.kernel == "precomputed"):
        _kernel_params(outer, 0)                        # raises, naming the kernel (kernel objects: KernelRidge reads them)
    if (_names(outer) & _GPR) and not hasattr(outer, "X_train_"):
        raise TypeError("GaussianProcessRegressor is not fitted (the prior mean is not explained)")
    if (_names(outer) & _GPR) and not hasattr(owner, "n_features_in_"):
        return _single_spec(owner, method, int(np.shape(owner.X_train_)[1]))     # kernels on non-vector input
    if not hasattr(outer, "n_features_in_"):
        raise TypeError(f"{type(outer).__name__} is not fitted")
    return _single_spec(owner, method, int(owner.n_features_in_))


def _fold_outer(spec, a, b):
    """The spec of the model behind one more affine map x' = a x + b of its raw columns."""
    if isinstance(spec, MulticlassSvmSpec):
        return MulticlassSvmSpec((spec.sv - b) / a, spec.sv_off, spec.cls_off, spec.dual, spec.intercept,
                                 spec.colw * a * a, (spec.colo - b) / a, spec.gamma, spec.kernel, spec.degree, spec.coef0,
                                 spec.head, spec.n_features, spec.classes, cal_a=spec.cal_a, cal_b=spec.cal_b,
                                 pi=spec.pi, scalar_out=spec.scalar_out)
    program = spec.program.folded(a, b) if spec.program is not None else None
    if spec.kernel == "laplacian":
        colw = spec.colw * np.abs(a)
    else:
        colw = spec.colw * a * a
    colo = (spec.colo - b) / a
    return KernelMachineSpec((spec.sv - b) / a, spec.sv_off, spec.dual, spec.intercept, colw, colo, spec.gamma,
                             spec.kernel, spec.degree, spec.coef0, spec.head, spec.n_features, cal_a=spec.cal_a,
                             cal_b=spec.cal_b, pi=spec.pi, scalar_out=spec.scalar_out, program=program)
