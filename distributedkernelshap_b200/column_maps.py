"""Column maps: a linear model behind per-column preprocessing, read in raw feature space.

A fitted scikit-learn ``Pipeline`` whose transformers each act on one column at a time (scalers, encoders, binning,
imputation, ``ColumnTransformer`` routing) followed by a linear estimator has a score that is still a sum over the RAW
columns::

    score_r(x) = b_r + sum_col f_{r,col}(x_col)

so the engine's algebra (DESIGN.md §3) applies with ``XW_i[k] = sum_{col in group k} f_col(x_i[col])``.  This module owns
the representation of ``f`` and its compiler.  For each raw column, ``f`` is one of two kinds:

* piecewise affine: sorted breakpoints ``t[0..m-2]``; the piece is ``k = searchsorted(t, x, side='right')`` (a value on
  a breakpoint belongs to the piece on its right) and ``f_r(x) = a[k][r] x + c[k][r]``;
* categorical: sorted float64 keys; an exact match gives that key's row, no match the unknown row (or the policy
  "error").

For both kinds a NaN gives the NaN row, or the policy "error".  "error" means scikit-learn's pipeline raises for that
input (an encoder's ``handle_unknown='error'``, or a NaN reaching the estimator); the engine raises ``ValueError`` too.

Packed form (what ``dks_set_column_maps`` reads), ``R`` score rows, ``D`` raw columns:

* ``hdr`` int32 [D][4] = {flags, m, key offset, value offset}; flags: ``CATEGORICAL``, ``NAN_ERROR``, ``UNKNOWN_ERROR``;
* ``keys`` float64: the ``m - 1`` breakpoints (affine) or ``m`` keys (categorical) of each column;
* ``vals`` float64: affine ``[m][2][R]`` (the ``a`` row then the ``c`` row of each piece), then the NaN row ``[R]``;
  categorical ``[m][R]``, the unknown row ``[R]``, then the NaN row ``[R]``.  Rows under the policy "error" are zero.

The tables are built by calling the fitted transformers themselves (on their own categories, bin representatives, one
unseen value and NaN), so ``drop``, infrequent categories and unknown handling come from scikit-learn.  Scalers and
imputers are folded analytically.  Anything that mixes columns or is not piecewise affine per column raises
``TypeError`` naming the step.

The same walk also builds, per encoded column, an exact program of the steps' own arithmetic (``_Prog``): a tree model
compares encoded values exactly, which folded maps cannot reproduce.  ``compile_encoding`` packs those programs
(``ColumnEncoding``, what ``dks_set_column_encoding`` reads; DESIGN.md §5.0.13)."""
import warnings

import numpy as np

CATEGORICAL = 1
NAN_ERROR = 2
UNKNOWN_ERROR = 4

ERR = None          # a value for which the pipeline raises

# ops of a column encoding (ColumnEncoding, dks_set_column_encoding): DKS_ENC_OP_* in include/dks.h
OP_SUB, OP_DIV, OP_MUL, OP_ADD, OP_CLIP, OP_NANFILL, OP_ISNAN, OP_PIECES, OP_TABLE = range(9)


class ColumnMaps:
    """Packed per-column maps of ``R`` score rows over ``D`` raw columns (module docstring), evaluated in NumPy by
    ``contributions``."""

    def __init__(self, hdr, keys, vals, R):
        self.hdr = np.ascontiguousarray(np.asarray(hdr, dtype=np.int32).reshape(-1, 4))
        self.keys = np.ascontiguousarray(np.asarray(keys, dtype=np.float64).reshape(-1))
        self.vals = np.ascontiguousarray(np.asarray(vals, dtype=np.float64).reshape(-1))
        self.R = int(R)
        self.D = self.hdr.shape[0]

    def column(self, col):
        """``(flags, keys, rows)`` of one column: rows [m][2][R] (affine) or [m + 1][R] (categorical, unknown row last),
        and the NaN row [R] as ``rows_nan``."""
        flags, m, ko, vo = (int(v) for v in self.hdr[col])
        R = self.R
        if flags & CATEGORICAL:
            keys = self.keys[ko:ko + m]
            rows = self.vals[vo:vo + (m + 1) * R].reshape(m + 1, R)
            nan_row = self.vals[vo + (m + 1) * R:vo + (m + 2) * R]
        else:
            keys = self.keys[ko:ko + m - 1]
            rows = self.vals[vo:vo + 2 * m * R].reshape(m, 2, R)
            nan_row = self.vals[vo + 2 * m * R:vo + (2 * m + 1) * R]
        return flags, keys, rows, nan_row

    def column_contribution(self, col, x):
        """``f_col(x)`` [n, R] for raw values ``x`` [n]; raises ``ValueError`` where the policy is "error"."""
        x = np.asarray(x, dtype=np.float64)
        flags, keys, rows, nan_row = self.column(col)
        out = np.empty((x.shape[0], self.R))
        nan = np.isnan(x)
        if nan.any() and flags & NAN_ERROR:
            raise ValueError(f"raw column {col} holds NaN, which the pipeline does not accept")
        out[nan] = nan_row
        xv = x[~nan]
        if flags & CATEGORICAL:
            k = np.searchsorted(keys, xv, side="left")
            hit = (k < len(keys)) & (keys[np.minimum(k, len(keys) - 1)] == xv)
            if not hit.all() and flags & UNKNOWN_ERROR:
                raise ValueError(f"raw column {col} holds a category unseen at fit time ({xv[~hit][0]!r})")
            out[~nan] = rows[np.where(hit, k, len(keys))]
        else:
            k = np.searchsorted(keys, xv, side="right")
            out[~nan] = rows[k, 0] * xv[:, None] + rows[k, 1]
        return out

    def contributions(self, X):
        """``sum_col f_col(X[:, col])`` [n, R]."""
        X = np.atleast_2d(np.asarray(X, dtype=np.float64))
        if X.shape[1] != self.D:
            raise ValueError(f"X has {X.shape[1]} columns, the column maps {self.D}")
        z = np.zeros((X.shape[0], self.R))
        for col in range(self.D):
            z += self.column_contribution(col, X[:, col])
        return z


# ---- features in flight: scalar functions of one raw column ---------------------------------------------------------
class _Affine:
    """Piecewise affine in the raw value; ``nan``: the value a raw NaN gives (float, NaN, or ERR)."""

    def __init__(self, src, t, a, c, nan, prog=None):
        self.src, self.t = src, np.asarray(t, dtype=np.float64)
        self.a, self.c = np.asarray(a, dtype=np.float64), np.asarray(c, dtype=np.float64)
        self.nan = nan
        self.prog = prog if prog is not None else _Prog(src)

    def is_raw(self):
        return len(self.a) == 1 and self.a[0] == 1.0 and self.c[0] == 0.0

    def is_constant(self):
        return bool(np.all(self.a == 0.0))

    def values(self):
        return list(self.c) + [self.nan]

    def map_values(self, g, prog):
        """Piecewise constant feature through the scalar function ``g`` (ERR in, ERR out); ``prog`` its exact program."""
        return _Affine(self.src, self.t, np.zeros_like(self.c), [_apply(g, v) for v in self.c], _apply(g, self.nan), prog)


class _Table:
    """Categorical in the raw value: ``vals[k]`` at ``keys[k]``, else ``unknown``; a raw NaN gives ``nan``."""

    def __init__(self, src, keys, vals, unknown, nan, prog):
        self.src, self.keys, self.vals = src, np.asarray(keys, dtype=np.float64), list(vals)
        self.unknown, self.nan = unknown, nan
        self.prog = prog

    def values(self):
        return self.vals + [self.unknown, self.nan]

    def map_values(self, g, prog):
        return _Table(self.src, self.keys, [_apply(g, v) for v in self.vals], _apply(g, self.unknown), _apply(g, self.nan),
                      prog)


def _apply(g, v):
    return ERR if v is ERR else g(float(v))


# ---- exact programs: what pipe[:-1].transform does to one encoded column, op by op (ColumnEncoding) ------------------
def _scalar(op, v):
    """One scalar op on a float64 value, with the arithmetic of the scikit-learn step it stands for."""
    code, c0, c1 = op
    v = np.float64(v)
    if code == OP_SUB:
        return float(v - c0)
    if code == OP_DIV:
        return float(v / np.float64(c0))
    if code == OP_MUL:
        return float(v * c0)
    if code == OP_ADD:
        return float(v + c0)
    if code == OP_CLIP:
        return float(np.clip(v, c0, c1))
    if code == OP_NANFILL:
        return float(c0) if np.isnan(v) else float(v)
    if code == OP_ISNAN:
        return 1.0 if np.isnan(v) else 0.0
    raise AssertionError(code)


class _Lookup:
    """The piecewise-constant end of a program: ``OP_PIECES`` (sorted edges, one output per bin, bin = numpy
    searchsorted(edges, v, side='right')) or ``OP_TABLE`` (sorted keys, one output per key, ``unknown`` on no exact
    match).  A NaN gives ``nan``.  Outputs may be ERR (the pipeline raises)."""

    def __init__(self, code, keys, outs, unknown, nan):
        self.code, self.keys, self.outs = code, np.asarray(keys, dtype=np.float64), list(outs)
        self.unknown, self.nan = unknown, nan

    def map(self, g):
        return _Lookup(self.code, self.keys, [_apply(g, v) for v in self.outs],
                       _apply(g, self.unknown) if self.code == OP_TABLE else None, _apply(g, self.nan))


class _Prog:
    """Exact program of one encoded column: scalar ops on raw column ``src``, optionally ending in a ``_Lookup``.  An op
    that follows the lookup is folded into its outputs, so a program is always ``ops`` then at most one lookup."""

    def __init__(self, src, ops=(), look=None):
        self.src, self.ops, self.look = src, tuple(ops), look

    def then(self, *ops):
        p = self
        for op in ops:
            p = _Prog(p.src, p.ops + (op,)) if p.look is None else _Prog(p.src, p.ops, p.look.map(lambda v: _scalar(op, v)))
        return p

    def lookup(self, look):
        """``look`` applied to this program's value (the program must not end in a lookup yet)."""
        assert self.look is None
        return _Prog(self.src, self.ops, look)

    def values(self):
        """``(sorted distinct finite values, whether NaN is one)`` of a piecewise-constant program: its lookup's outputs,
        or what the ops after its last ``OP_ISNAN`` make of 0 and 1."""
        if self.look is not None:
            vs = self.look.outs + [self.look.unknown if self.look.code == OP_TABLE else ERR, self.look.nan]
        else:
            last = max(k for k, op in enumerate(self.ops) if op[0] == OP_ISNAN)
            vs = []
            for v in (0.0, 1.0):
                for op in self.ops[last + 1:]:
                    v = _scalar(op, v)
                vs.append(v)
        vs = [v for v in vs if v is not ERR]
        return sorted({float(v) for v in vs if not np.isnan(v)}), any(np.isnan(v) for v in vs)

    def compose(self, g, keys, has_nan):
        """This program through ``g`` (a scalar function defined on the program's finite values ``keys`` and, with
        ``has_nan``, on NaN): the lookup's outputs mapped, or a table over ``keys`` appended."""
        if self.look is not None:
            return _Prog(self.src, self.ops, self.look.map(g))
        return self.lookup(_Lookup(OP_TABLE, keys, [g(k) for k in keys], ERR, g(np.nan) if has_nan else ERR))


def _name(step):
    return type(step).__name__


# ---- per-step compilers -------------------------------------------------------------------------------------------
def _affine_step(feats, mul, add, name, exact, clip=None):
    """y = x * mul + add per feature (add applied after mul), then optionally clipped to ``clip`` -- the order of the
    scalers' own arithmetic, so that tables come out bit-identical to ``transform``.  ``exact[i]``: the ops the step
    itself performs on feature i (its program's continuation)."""
    out = []
    for f, s, o, ops in zip(feats, mul, add, exact):
        def g(v, s=s, o=o):
            y = v * s + o
            return float(np.clip(y, clip[0], clip[1])) if clip is not None else y
        prog = f.prog.then(*ops)
        if isinstance(f, _Table) or f.is_constant():
            out.append(f.map_values(g, prog))
            continue
        a, c = f.a * s, f.c * s + o
        nan = _apply(g, f.nan)
        if clip is None:
            out.append(_Affine(f.src, f.t, a, c, nan, prog))
            continue
        if len(a) != 1:
            raise TypeError(f"{name}(clip=True) after a piecewise transformer is not supported")
        lo, hi = float(clip[0]), float(clip[1])
        x_lo, x_hi = (lo - c[0]) / a[0], (hi - c[0]) / a[0]
        if a[0] > 0:
            out.append(_Affine(f.src, [x_lo, x_hi], [0.0, a[0], 0.0], [lo, c[0], hi], nan, prog))
        else:
            out.append(_Affine(f.src, [x_hi, x_lo], [0.0, a[0], 0.0], [hi, c[0], lo], nan, prog))
    return out


def _scaler(step, feats):
    from sklearn import preprocessing as pp
    k = len(feats)
    one, zero = np.ones(k), np.zeros(k)

    def ops(code, vals, on=True):
        return [[(code, float(v), 0.0)] if on else [] for v in np.broadcast_to(np.asarray(vals, dtype=np.float64), (k,))]
    if isinstance(step, pp.StandardScaler):
        with_mean = step.with_mean and step.mean_ is not None
        mean = step.mean_ if with_mean else zero
        scale = step.scale_ if step.with_std and step.scale_ is not None else one
        # (x - mean) / scale
        feats = _affine_step(feats, one, -np.asarray(mean, dtype=np.float64), "StandardScaler",
                             ops(OP_SUB, mean, with_mean))
        return _affine_step(feats, 1.0 / np.asarray(scale, dtype=np.float64), zero, "StandardScaler",
                            ops(OP_DIV, scale)) if step.with_std else feats
    if isinstance(step, pp.RobustScaler):
        if step.with_centering:
            feats = _affine_step(feats, one, -np.asarray(step.center_, dtype=np.float64), "RobustScaler",
                                 ops(OP_SUB, step.center_))
        if step.with_scaling:
            feats = _affine_step(feats, 1.0 / np.asarray(step.scale_, dtype=np.float64), zero, "RobustScaler",
                                 ops(OP_DIV, step.scale_))
        return feats
    if isinstance(step, pp.MaxAbsScaler):
        return _affine_step(feats, 1.0 / np.asarray(step.scale_, dtype=np.float64), zero, "MaxAbsScaler",
                            ops(OP_DIV, step.scale_))
    if isinstance(step, pp.MinMaxScaler):
        exact = [m + a for m, a in zip(ops(OP_MUL, step.scale_), ops(OP_ADD, step.min_))]
        if step.clip:
            lo, hi = (float(v) for v in step.feature_range)
            exact = [e + [(OP_CLIP, lo, hi)] for e in exact]
        return _affine_step(feats, np.asarray(step.scale_, dtype=np.float64), np.asarray(step.min_, dtype=np.float64),
                            "MinMaxScaler", exact, clip=step.feature_range if step.clip else None)
    raise AssertionError


def _imputer(step, feats):
    missing = step.missing_values
    if not (isinstance(missing, float) and np.isnan(missing)):
        raise TypeError(f"SimpleImputer(missing_values={missing!r}): only NaN as the missing value is supported")
    stats = np.asarray(step.statistics_, dtype=np.float64)
    if np.isnan(stats).any() and not getattr(step, "keep_empty_features", False):
        raise TypeError("SimpleImputer drops columns that were empty at fit time: not supported")
    out = []
    for f, fill in zip(feats, stats):
        def g(v, fill=fill):
            return float(fill) if np.isnan(v) else v
        prog = f.prog.then((OP_NANFILL, float(fill), 0.0))
        if isinstance(f, _Affine) and not f.is_constant():
            out.append(_Affine(f.src, f.t, f.a, f.c, _apply(g, f.nan), prog))
        else:
            out.append(f.map_values(g, prog))
    ind = getattr(step, "indicator_", None)
    if step.add_indicator and ind is not None:
        for i in ind.features_:
            f = feats[i]

            def h(v):
                return 1.0 if np.isnan(v) else 0.0
            prog = f.prog.then((OP_ISNAN, 0.0, 0.0))
            if isinstance(f, _Affine) and not f.is_constant():
                out.append(_Affine(f.src, [], [0.0], [0.0], _apply(h, f.nan), prog))
            else:
                out.append(f.map_values(h, prog))
    return out


def _transform_row_outputs(step, P):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = step.transform(P)
    if hasattr(out, "toarray"):
        out = out.toarray()
    return np.asarray(out, dtype=np.float64)


def _output_owner(step, k):
    """Input index of every output column of a transformer that encodes each input on its own."""
    names = step.get_feature_names_out(np.asarray([f"c{i}#" for i in range(k)], dtype=object))
    return np.asarray([int(str(nm).split("#")[0][1:]) for nm in names])


def _valuewise(step, feats):
    """Encoders and binning: evaluated by calling ``step.transform`` on probe values of each input."""
    from sklearn import preprocessing as pp
    name = _name(step)
    k = len(feats)
    is_bins = isinstance(step, pp.KBinsDiscretizer)
    if not is_bins:
        for cats in step.categories_:
            if not np.issubdtype(np.asarray(cats).dtype, np.number):
                raise TypeError(f"{name}: string categories are not supported (numeric categories only)")
    owner = _output_owner(step, k)

    # a value every input accepts, for the inputs not being probed
    safe = []
    for i, f in enumerate(feats):
        if is_bins:
            cand = [float(step.bin_edges_[i][0])] if isinstance(f, _Affine) and f.is_raw() else f.values()
        else:
            cats = np.asarray(step.categories_[i], dtype=np.float64)
            cand = list(cats[~np.isnan(cats)]) if isinstance(f, _Affine) and f.is_raw() else f.values()
        cand = [v for v in cand if v is not ERR and not np.isnan(v)]
        safe.append(cand[0] if cand else 0.0)

    def probe(i, values):
        """Outputs of input i's columns at each value (a list of [n_out_i] arrays, ERR where transform raises)."""
        res = []
        for v in values:
            if v is ERR:
                res.append(ERR)
                continue
            row = np.asarray(safe, dtype=np.float64)[None, :].copy()
            row[0, i] = v
            try:
                res.append(_transform_row_outputs(step, row)[0, owner == i])
            except ValueError:
                res.append(ERR)
        return res

    def col(o, j):
        return ERR if o is ERR else float(o[j])

    out = []
    for i, f in enumerate(feats):
        n_out = int((owner == i).sum())
        if isinstance(f, _Affine) and f.is_raw():
            nan_out = probe(i, [f.nan])[0]
            # the program replays the steps before this one, so its lookup sees what the step sees: a NaN only when no
            # imputer filled it
            nan_look = nan_out if f.nan is not ERR and np.isnan(f.nan) else probe(i, [np.nan])[0]
            if is_bins:
                t = np.asarray(step.bin_edges_[i][1:-1], dtype=np.float64)
                reps = [float(step.bin_edges_[i][0]) if len(t) == 0 else float(np.nextafter(t[0], -np.inf))]
                reps += [float(v) for v in t]
                outs = probe(i, reps)
                for j in range(n_out):
                    look = _Lookup(OP_PIECES, t, [col(o, j) for o in outs], None, col(nan_look, j))
                    out.append(_Affine(f.src, t, np.zeros(len(reps)), [o[j] for o in outs],
                                       ERR if nan_out is ERR else nan_out[j], f.prog.lookup(look)))
            else:
                cats = np.asarray(step.categories_[i], dtype=np.float64)
                keys = np.unique(cats[~np.isnan(cats)])
                outs = probe(i, list(keys))
                unseen = float(keys.max() + 1.0) if len(keys) else 0.0
                unk = probe(i, [unseen])[0]
                for j in range(n_out):
                    look = _Lookup(OP_TABLE, keys, [col(o, j) for o in outs], col(unk, j), col(nan_look, j))
                    out.append(_Table(f.src, keys, [o[j] for o in outs], ERR if unk is ERR else unk[j],
                                      ERR if nan_out is ERR else nan_out[j], f.prog.lookup(look)))
        elif isinstance(f, _Table) or f.is_constant():
            vals = sorted({float(v) for v in f.values() if v is not ERR and not np.isnan(v)})
            has_nan = any(v is not ERR and np.isnan(v) for v in f.values())
            outs = dict(zip(vals, probe(i, vals)))
            nan_out = probe(i, [np.nan])[0] if has_nan else ERR
            # the program's own values (exact arithmetic; the folded ones above may differ in the last bit)
            pvals, p_nan = f.prog.values()
            pouts = dict(zip(pvals, probe(i, pvals)))
            p_nan_out = probe(i, [np.nan])[0] if p_nan else ERR
            for j in range(n_out):
                def g(v, j=j):
                    o = nan_out if np.isnan(v) else outs[v]
                    return ERR if o is ERR else float(o[j])

                def gp(v, j=j):
                    return col(p_nan_out if np.isnan(v) else pouts[v], j)
                out.append(f.map_values(g, f.prog.compose(gp, pvals, p_nan)))
        else:
            raise TypeError(f"{name} after a transformer that is not the identity or piecewise constant on its column "
                            "is not supported")
    # outputs of one input are contiguous and in input order for every encoder scikit-learn ships
    order = np.argsort(owner, kind="stable")
    if not np.array_equal(order, np.arange(len(owner))):
        raise TypeError(f"{name}: output columns are not grouped by input column")
    return out


def _compile_step(step, feats):
    from sklearn import compose, impute, pipeline, preprocessing as pp
    if step is None or (isinstance(step, str) and step == "passthrough"):
        return feats
    if isinstance(step, pp.FunctionTransformer) and step.func is None:
        return feats                        # how a fitted ColumnTransformer stores 'passthrough
    if isinstance(step, pipeline.Pipeline):
        for _, s in step.steps:
            feats = _compile_step(s, feats)
        return feats
    if isinstance(step, compose.ColumnTransformer):
        return _column_transformer(step, feats)
    if isinstance(step, (pp.StandardScaler, pp.MinMaxScaler, pp.MaxAbsScaler, pp.RobustScaler)):
        return _scaler(step, feats)
    if isinstance(step, impute.SimpleImputer):
        return _imputer(step, feats)
    if isinstance(step, (pp.OneHotEncoder, pp.OrdinalEncoder, pp.KBinsDiscretizer)):
        return _valuewise(step, feats)
    raise TypeError(f"{_name(step)} is not supported in a pipeline the CUDA engine explains: only per-column scalers, "
                    "encoders, KBinsDiscretizer and SimpleImputer (steps that mix columns or are not piecewise affine per "
                    "column are refused)")


def _selected(columns, n, owner_name):
    """Indices a ColumnTransformer selector picks among ``n`` inputs: integers, a slice or a boolean mask."""
    if callable(columns):
        raise TypeError(f"ColumnTransformer '{owner_name}': callable column selectors are not supported")
    if isinstance(columns, slice):
        if isinstance(columns.start, str) or isinstance(columns.stop, str):
            raise TypeError(f"ColumnTransformer '{owner_name}': column selection by name is not supported")
        return list(range(n))[columns]
    cols = np.atleast_1d(np.asarray(columns))
    if cols.size == 0:
        return []
    if cols.dtype == bool:
        return [int(i) for i in np.nonzero(cols)[0]]
    if not np.issubdtype(cols.dtype, np.integer):
        raise TypeError(f"ColumnTransformer '{owner_name}': column selection by name is not supported")
    return [int(i) % n for i in cols]


def _column_transformer(ct, feats):
    out = []
    for name, trans, columns in ct.transformers_:
        idx = _selected(columns, len(feats), name)
        if not idx or (isinstance(trans, str) and trans == "drop"):
            continue
        out.extend(_compile_step(trans, [feats[i] for i in idx]))
    return out


# ---- final assembly -----------------------------------------------------------------------------------------------
def _merge_column(col, feats, weights, R):
    """One raw column's map from its features ``feats`` and their coefficient columns ``weights`` [len(feats)][R]:
    returns (flags, keys, value rows flattened)."""
    def nan_row(fs):
        vals = [f.nan for f in fs]
        if any(v is ERR or np.isnan(v) for v in vals):
            return 0, np.zeros(R)
        return 1, sum(w * v for w, v in zip(weights, vals))

    if not feats:
        return 0, [], np.zeros(3 * R)           # dropped column: one zero piece, NaN row zero
    nan_ok, nrow = nan_row(feats)
    flags = 0 if nan_ok else NAN_ERROR
    tables = [f for f in feats if isinstance(f, _Table)]
    if not tables:
        T = np.unique(np.concatenate([f.t for f in feats]))
        rows = np.zeros((len(T) + 1, 2, R))
        for K in range(len(T) + 1):
            for f, w in zip(feats, weights):
                p = 0 if K == 0 else int(np.searchsorted(f.t, T[K - 1], side="right"))
                rows[K, 0] += w * f.a[p]
                rows[K, 1] += w * f.c[p]
        return flags, T, np.concatenate([rows.reshape(-1), nrow])
    for f in feats:
        if isinstance(f, _Affine) and not (f.is_constant() and len(f.a) == 1):
            raise TypeError(f"raw column {col} feeds both an encoder and a numeric transformer: not supported")
    keys = np.unique(np.concatenate([f.keys for f in tables]))

    def value_at(f, key):
        if isinstance(f, _Affine):
            return f.c[0]
        hit = np.nonzero(f.keys == key)[0]
        return f.vals[hit[0]] if len(hit) else f.unknown

    rows = np.zeros((len(keys) + 1, R))
    for kk, key in enumerate(keys):
        for f, w in zip(feats, weights):
            v = value_at(f, key)
            if v is ERR or np.isnan(v):
                raise TypeError(f"raw column {col}: category {key!r} is known to one encoder and refused by another")
            rows[kk] += w * v
    unk = [f.c[0] if isinstance(f, _Affine) else f.unknown for f in feats]
    if any(v is ERR or np.isnan(v) for v in unk):
        flags |= UNKNOWN_ERROR
    else:
        rows[-1] = sum(w * v for w, v in zip(weights, unk))
    return flags | CATEGORICAL, keys, np.concatenate([rows.reshape(-1), nrow])


def compile_maps(steps, n_raw, W):
    """Column maps of the fitted transformer ``steps`` (applied in order; each a transformer, Pipeline or
    ColumnTransformer) over ``n_raw`` raw columns, followed by the score rows ``W`` [R, E] of the final estimator (E
    encoded columns)."""
    W = np.atleast_2d(np.asarray(W, dtype=np.float64))
    R = W.shape[0]
    feats = [_Affine(c, [], [1.0], [0.0], np.nan) for c in range(n_raw)]
    for step in steps:
        feats = _compile_step(step, feats)
    if len(feats) != W.shape[1]:
        raise TypeError(f"the preprocessing yields {len(feats)} columns but the estimator has {W.shape[1]} coefficients")
    hdr, keys, vals = [], [], []
    nk = nv = 0
    for col in range(n_raw):
        js = [j for j, f in enumerate(feats) if f.src == col]
        flags, k, v = _merge_column(col, [feats[j] for j in js], [W[:, j] for j in js], R)
        m = len(k) if flags & CATEGORICAL else len(k) + 1
        hdr.append((flags, m, nk, nv))
        keys.append(np.asarray(k, dtype=np.float64))
        vals.append(np.asarray(v, dtype=np.float64))
        nk += len(k)
        nv += len(v)
    return ColumnMaps(hdr, np.concatenate(keys), np.concatenate(vals), R)


class ColumnEncoding:
    """Packed exact programs of ``E`` encoded columns over ``D`` raw columns (what ``dks_set_column_encoding`` reads):
    ``pipe[:-1].transform`` replayed column by column, bit for bit.

    * ``hdr`` int32 [E][3] = {raw source column, first op, op count};
    * ``ops`` int32 [n_ops][4] = {code ``OP_*``, flags ``NAN_ERROR`` | ``UNKNOWN_ERROR``, m, table offset};
    * ``opvals`` float64 [n_ops][2]: the constants of the scalar ops (``OP_CLIP``: lo, hi);
    * ``tab`` float64: per lookup, its m sorted edges (``OP_PIECES``) or keys (``OP_TABLE``), then its outputs -- m + 1
      bins, or m keys and the unknown output --, then the NaN output: 2 m + 2 values.  Outputs under the policy "error"
      are 0 and flagged instead.

    A lookup can only end a program.  ``transform`` evaluates the encoding in NumPy."""

    def __init__(self, D, hdr, ops, opvals, tab):
        self.D = int(D)
        self.hdr = np.ascontiguousarray(np.asarray(hdr, dtype=np.int32).reshape(-1, 3))
        self.ops = np.ascontiguousarray(np.asarray(ops, dtype=np.int32).reshape(-1, 4))
        self.opvals = np.ascontiguousarray(np.asarray(opvals, dtype=np.float64).reshape(-1, 2))
        self.tab = np.ascontiguousarray(np.asarray(tab, dtype=np.float64).reshape(-1))
        self.E = self.hdr.shape[0]

    @property
    def sources(self):
        return self.hdr[:, 0].copy()

    def column(self, e, x):
        """Encoded column ``e`` [n] of the raw values ``x`` [n] of its source; raises ``ValueError`` naming the first row
        whose value the pipeline refuses."""
        v = np.array(x, dtype=np.float64)
        _, first, count = (int(u) for u in self.hdr[e])
        for k in range(first, first + count):
            code, flags, m, off = (int(u) for u in self.ops[k])
            c0, c1 = self.opvals[k]
            if code == OP_SUB:
                v = v - c0
            elif code == OP_DIV:
                v = v / c0
            elif code == OP_MUL:
                v = v * c0
            elif code == OP_ADD:
                v = v + c0
            elif code == OP_CLIP:
                v = np.clip(v, c0, c1)
            elif code == OP_NANFILL:
                v = np.where(np.isnan(v), c0, v)
            elif code == OP_ISNAN:
                v = np.isnan(v).astype(np.float64)
            else:
                keys = self.tab[off:off + m]
                outs = self.tab[off + m:off + 2 * m + 1]
                nan_out = self.tab[off + 2 * m + 1]
                nan = np.isnan(v)
                if code == OP_PIECES:
                    idx = np.searchsorted(keys, v, side="right")
                    bad = nan & bool(flags & NAN_ERROR)
                else:
                    pos = np.minimum(np.searchsorted(keys, v, side="left"), max(m - 1, 0))
                    hit = (m > 0) & (keys[pos] == v) if m else np.zeros(v.shape, dtype=bool)
                    idx = np.where(hit, pos, m)
                    bad = (nan & bool(flags & NAN_ERROR)) | (~nan & ~hit & bool(flags & UNKNOWN_ERROR))
                if bad.any():
                    r = int(np.nonzero(bad)[0][0])
                    raise ValueError(f"row {r}: raw column {int(self.hdr[e, 0])} holds {x[r]!r}, which the pipeline "
                                     "refuses (NaN, or a category unseen at fit time)")
                v = np.where(nan, nan_out, outs[np.minimum(idx, len(outs) - 1)])
        return v

    def transform(self, X):
        """``pipe[:-1].transform(X)`` [n, E] float64, densified."""
        X = np.atleast_2d(np.asarray(X, dtype=np.float64))
        if X.shape[1] != self.D:
            raise ValueError(f"X has {X.shape[1]} columns, the encoding {self.D}")
        out = np.empty((X.shape[0], self.E))
        for e in range(self.E):
            out[:, e] = self.column(e, X[:, int(self.hdr[e, 0])])
        return out


def _encoders(step):
    """Every encoder or KBinsDiscretizer inside a fitted transformer (Pipelines and ColumnTransformers walked)."""
    from sklearn import compose, pipeline, preprocessing as pp
    if isinstance(step, pipeline.Pipeline):
        return [e for _, s in step.steps for e in _encoders(s)]
    if isinstance(step, compose.ColumnTransformer):
        return [e for _, t, _ in step.transformers_ for e in _encoders(t)]
    return [step] if isinstance(step, (pp.OneHotEncoder, pp.OrdinalEncoder, pp.KBinsDiscretizer)) else []


def compile_encoding(steps, n_raw, n_out, model="a tree model"):
    """Exact per-column programs (``ColumnEncoding``) of the fitted transformer ``steps`` (applied in order) over
    ``n_raw`` raw columns, for an estimator (``model``, as refusals name it) reading ``n_out`` encoded columns: a tree
    model, which compares their values, or a kernel machine, MLP or neighbour model, which sum over them.  Accepts what
    ``compile_maps`` accepts, less its rule that a raw column may not feed both an encoder and a numeric transformer
    (the linear maps need it: they fold every step into one function per raw column; an exact program per encoded
    column does not); refuses encoders whose output dtype is not float64 (the estimator would read rounded values)."""
    for enc in _encoders_of(steps):
        dt = getattr(enc, "dtype", None)
        if dt is not None and np.dtype(dt) != np.float64:
            raise TypeError(f"{_name(enc)}(dtype={np.dtype(dt).name}): only float64 encoder output is supported behind "
                            f"{model}")
    feats = [_Affine(c, [], [1.0], [0.0], np.nan) for c in range(n_raw)]
    for step in steps:
        feats = _compile_step(step, feats)
    if len(feats) != n_out:
        raise TypeError(f"the preprocessing yields {len(feats)} columns but the estimator reads {n_out}")
    hdr, ops, opvals, tab = [], [], [], []
    for e, f in enumerate(feats):
        p = f.prog
        hdr.append((p.src, len(ops), len(p.ops) + (p.look is not None)))
        for code, c0, c1 in p.ops:
            ops.append((code, 0, 0, 0))
            opvals.append((c0, c1))
        if p.look is None:
            continue
        lk = p.look
        outs = lk.outs + ([lk.unknown] if lk.code == OP_TABLE else [])
        if any(v is ERR for v in lk.outs):
            raise TypeError(f"encoded column {e}: a value known to one encoder is refused by a later step: not supported")
        flags = (NAN_ERROR if lk.nan is ERR else 0) | (UNKNOWN_ERROR if lk.code == OP_TABLE and lk.unknown is ERR else 0)
        ops.append((lk.code, flags, len(lk.keys), len(tab)))
        opvals.append((0.0, 0.0))
        tab.extend(float(k) for k in lk.keys)
        tab.extend(0.0 if v is ERR else float(v) for v in outs + [lk.nan])
    enc = ColumnEncoding(n_raw, hdr, ops, opvals, tab)
    enc.steps = list(steps)         # what the encoding replays: the engine checks it against their own transform
    return enc


def _encoders_of(steps):
    return [e for s in steps for e in _encoders(s)]


def pipeline_parts(pipe):
    """``(preprocessor steps, final estimator)`` of a fitted Pipeline, nested final pipelines flattened."""
    pre = []
    while True:
        steps = list(pipe.steps)
        pre.extend(s for _, s in steps[:-1])
        final = steps[-1][1]
        if type(final).__name__ == "Pipeline" and hasattr(final, "steps"):
            pipe = final
            continue
        return pre, final
