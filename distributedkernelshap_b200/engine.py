"""``GpuKernelExplainer``: the object that sits in ``KernelShap._explainer``.

In the reference that slot holds ``KernelExplainerWrapper`` (explainers/kernel_shap.py:217-261), a subclass of
``shap.KernelExplainer``; ``KernelShap`` only needs ``get_explanation(X, **kwargs)``, ``.expected_value`` and
``.vector_out`` from it (kernel_shap.py:789-790, :880-887).  This class keeps that constructor shape
``(predictor, background_data, link=..., seed=...)`` and those members, and runs the per-instance hot path
(varying groups -> coalition plan -> mask/impute -> predict -> background mean -> link -> constrained WLS) in
CUDA through the C ABI of ``include/dks.h``.  No CPU fallback: without ``libdks.so`` and an H100 it raises.
"""
import ctypes as C
import logging

import numpy as np

from . import _cabi
from .data import DenseData, convert_to_data, convert_to_link
from .ensembles import MAX_GROUPS as ENSEMBLE_MAX_GROUPS, EnsembleSpec, extract_ensemble_spec
from .plan import build_plan, l1_tables, pack_dense_plan, projection, resolve_nsamples, sampling_info
from .kernel_machines import MAX_GROUPS as KMACH_MAX_GROUPS, KernelMachineSpec, extract_kernel_machine_spec
from .mlp import MAX_GROUPS as MLP_MAX_GROUPS, MlpSpec, extract_mlp_spec
from .neighbors import MAX_GROUPS as KNN_MAX_GROUPS, KnnSpec, extract_knn_spec
from .predictors import LinearModelSpec, extract_linear_spec
from .stacking import MAX_GROUPS as STACKING_MAX_GROUPS, StackingSpec, extract_stacking_spec
from . import torch_models
from .torch_models import TorchModelSpec
from .trees import MAX_GROUPS as TREE_MAX_GROUPS, TreeEnsembleSpec, extract_encoded_pipeline_spec, \
    extract_tree_pipeline_spec, extract_tree_spec

logger = logging.getLogger(__name__)

MODEL_CHECK_RTOL = 1e-9
MAX_ROWS_PER_CALL = 65536     # rows per C-ABI call: bounds the engine's per-call workspace (n x S x 8 B on the fast path)
# per-instance plans of 65..128 groups keep, per row, the plan (S x 16 B words + S x 8 B weights) and the inverse of its
# (M-1) x (M-1) normal matrix: about 222 KB at M = 128, S = 4096.  Row blocks of 4096 bound that workspace by ~0.9 GB.
MAX_ROWS_PER_CALL_WIDE_PER_INSTANCE = 4096
MAX_SAMPLED_SIZES = 64        # subset sizes the device sampler draws from (csrc/dks_sampler.cuh, MAX_SIZES)
# a model behind a column encoding keeps the encoded rows of a call on the device (n x E x 8 B): row blocks bound them
MAX_ENCODED_BYTES_PER_CALL = 256 << 20
# a soft-voting ensemble keeps its members' weighted background means of a call on the device (n x C x S x 8 B): row
# blocks bound them
MAX_ENSEMBLE_BYTES_PER_CALL = 1 << 30
# a stacking ensemble keeps its members' outputs of every masked row of one background chunk on the device
# (n x F x chunk x S x 8 B): the library splits the background into the fewest chunks within this budget
MAX_STACKING_BYTES_PER_CALL = 1 << 30


def per_instance_workspace_bytes(M, S):
    """Device workspace one row of ``plan_mode='per_instance'`` holds for a plan of S rows over M groups: the plan's
    words and weights and one (M-1) x (M-1) float64 matrix (two of them, factor and inverse, up to 64 groups)."""
    words = 1 if M <= 64 else 2
    mats = 2 if M <= 64 else 1
    return S * (8 * words + 8) + mats * 8 * (M - 1) ** 2


def device_sampling_supported(M, n_sizes):
    """Whether the device sampler draws the per-instance plans of M groups whose sampled part has ``n_sizes`` subset
    sizes: up to 128 groups (one- and two-word rows) and 64 sizes (M <= 128 has at most 63)."""
    return M <= 128 and n_sizes <= MAX_SAMPLED_SIZES


def rows_per_call(act_code, n_outputs, plan_mode, G, score_rows=1):
    """Rows per C-ABI call.  The softmax and one-vs-rest heads' shared-plan path keeps C per-class sums per coalition
    where the binary head keeps two: their row blocks are 2 / C as long, so that the per-call workspace stays the binary
    path's.  The mixture head keeps ``score_rows`` = K R_m nibble tables per instance and, on its shared-plan route, a
    member's sums next to the mixture's: its blocks are 1 / (K R_m) as long.  Tree ensembles, kernel machines and MLPs keep
    no per-instance workspace beyond phi and f(x) (their kernels hold an instance's coalitions in shared memory): full
    blocks.  Per-instance plans of more than 64 groups: ``MAX_ROWS_PER_CALL_WIDE_PER_INSTANCE`` (plans
    are keyed by the global row, so results do not depend on the block size)."""
    if act_code == _cabi.ACT_MIX:
        return MAX_ROWS_PER_CALL // max(1, score_rows)
    if act_code in (_cabi.ACT_SOFTMAX, _cabi.ACT_OVR) and n_outputs > 2:
        return MAX_ROWS_PER_CALL * 2 // n_outputs
    if plan_mode == "per_instance" and G > 64:
        return MAX_ROWS_PER_CALL_WIDE_PER_INSTANCE
    return MAX_ROWS_PER_CALL


def refuse_partial_sets_beyond_64_groups(G, hist):
    """Multi-word coalition rows (more than 64 groups) exist on the shared-plan path only, which takes the instances whose
    groups ALL vary.  ``hist[M]`` = instances with M varying groups: anything below G is refused here, before plans (and,
    beyond 128 groups, their projections) are built for sizes no kernel would evaluate -- the library reports the same
    condition as status 3 (unsupported)."""
    if G <= 64:
        return
    partial = [M for M in range(0, G) if hist[M] > 0]
    if partial:
        raise NotImplementedError(
            f"{int(sum(hist[M] for M in partial))} instance(s) have a partial varying set (M in {partial[:8]}"
            f"{'...' if len(partial) > 8 else ''} of {G} groups): more than 64 groups run on the shared-plan path, which "
            "needs every group to vary (unsupported otherwise)")


def _explicit_l1(l1_reg):
    """``(mode, k)`` of ``dks_set_l1`` for an ``l1_reg`` that selects whatever the sampled fraction ('aic', 'bic',
    'num_features(k)'), None for 'auto'; a fixed Lasso strength is refused."""
    if l1_reg in ("aic", "bic"):
        return (1 if l1_reg == "aic" else 2, 0)
    if isinstance(l1_reg, str) and l1_reg.startswith("num_features("):
        return (3, int(l1_reg[len("num_features("):-1]))
    if l1_reg != "auto":
        raise NotImplementedError(f"l1_reg={l1_reg!r}: a fixed Lasso strength is not implemented in the CUDA engine; "
                                  "use 'auto', 'aic', 'bic', 'num_features(k)' or False")
    return None


def _auto_selects(M, nsamples):
    """l1_reg='auto': upstream selects when less than 20% of the coalition space of M groups is evaluated."""
    S, max_s = resolve_nsamples(M, nsamples)
    return S / max_s < 0.2


def l1_selecting_sizes(l1_reg, nsamples, G, hist):
    """Which instances run upstream's l1 feature selection before the constrained WLS (``solve``): all of them under
    'aic' / 'bic' / 'num_features(k)', and under 'auto' those whose coalition plan covers less than 20% of the coalition
    space -- a property of their number M of varying groups.  ``hist[M]`` = instances with M varying groups.  Returns
    ``(mode, k, sizes)``: the ``dks_set_l1`` mode and k, and the sorted M (>= 2, present in ``hist``) that select; mode 0
    and no sizes when none does.  Raises for what the engine does not cover: a fixed Lasso strength, more than 128 groups
    selecting, and partial varying sets selecting beyond 64 groups."""
    if l1_reg in (False, 0):
        return 0, 0, []
    explicit = _explicit_l1(l1_reg)

    sizes = [M for M in range(2, G + 1) if hist[M] > 0 and (explicit is not None or _auto_selects(M, nsamples))]
    if not sizes:
        return 0, 0, []
    if max(sizes) > 128:
        raise NotImplementedError(
            f"l1_reg={l1_reg!r} selects features among {max(sizes)} varying groups; the CUDA engine's LARS path covers at "
            "most 128 groups -- pass l1_reg=False for the plain constrained WLS (or 'num_features(k)' on a narrower "
            "grouping)")
    partial = [M for M in sizes if M != G]
    if partial and G > 64:
        raise NotImplementedError(
            f"l1_reg={l1_reg!r} selects features for instances with M in {partial[:8]} varying groups of {G} (a partial "
            "varying set): beyond 64 groups the CUDA engine selects for instances whose groups all vary only -- pass "
            "l1_reg=False")
    mode, k = explicit if explicit is not None else (1, 0)
    return mode, k, sizes


def _dtype_code(t):
    """``DKS_EXTERNAL_FLOAT32`` / ``_FLOAT64`` of a float32 / float64 tensor."""
    import torch
    return _cabi.EXTERNAL_FLOAT64 if t.dtype == torch.float64 else _cabi.EXTERNAL_FLOAT32


class GpuKernelExplainer:
    """CUDA KernelSHAP explainer with the interface of ``shap.KernelExplainer`` / ``KernelExplainerWrapper``.

    Parameters
    ----------
    model
        What the reference passes as ``predictor``: a bound ``predict_proba`` / ``decision_function`` of a linear
        model or of a ``Pipeline`` of per-column preprocessing ending in one (explained in raw feature space), or a
        ``LinearModelSpec`` (see ``predictors.extract_linear_spec``); a tree model (``trees.extract_tree_spec``:
        ``IsolationForest`` and ``AdaBoostClassifier`` included), bare or behind such a ``Pipeline``
        (``trees.extract_tree_pipeline_spec``: the device replays the steps bit for bit); a kernel machine; a
        scikit-learn MLP (``mlp.extract_mlp_spec``); a k-nearest-neighbour model (``neighbors.extract_knn_spec``); each of
        the last three bare, behind affine scalers (folded into the model) or behind such a ``Pipeline``
        (``trees.extract_encoded_pipeline_spec``, replayed like a tree's); a soft ``VotingClassifier`` or a
        ``VotingRegressor`` mixing those families with linear members, bare or behind such a ``Pipeline``
        (``ensembles.extract_ensemble_spec``); a ``StackingClassifier`` (``predict_proba``, ``decision_function``) or a
        ``StackingRegressor`` over those families with a linear final estimator, bare or behind such a ``Pipeline``
        (``stacking.extract_stacking_spec``).  A raw value the pipeline would refuse (NaN, or an unseen category under
        ``handle_unknown='error'``) raises ``ValueError``.  Or a ``torch.nn.Module`` in eval mode on one CUDA device,
        float32 or float64, mapping [B, D] to [B] or [B, C <= 8] (``torch_models.TorchModelSpec``): the engine builds the
        masked rows on the device, the module runs on them and the engine reduces its outputs and solves (up to 64
        groups, no column encoding, no ``explain_device``).
    data
        Background data: array, DataFrame or ``DenseData`` (groups and weights honoured).
    link
        ``'identity'`` or ``'logit'``.
    seed
        As in ``KernelExplainerWrapper.__init__`` (kernel_shap.py:225-228): seeds the global legacy NumPy stream the
        sampled part of the coalition plans is drawn from.
    device
        CUDA device ordinal (default: ``LOCAL_RANK`` under torchrun, else 0; a module's own device).
    model_batch_rows
        A module only: masked rows per module call (default 2^20), rounded down to whole coalitions of the background,
        at least one.  The module's activation memory grows with it.
    """

    def __init__(self, model, data, link="identity", seed=None, device=None, kernel="auto", plan_mode="shared",
                 model_batch_rows=None, **kwargs):
        if kwargs:
            raise TypeError(f"unexpected keyword arguments {sorted(kwargs)}")
        if plan_mode not in ("shared", "per_instance"):
            raise ValueError("plan_mode must be 'shared' or 'per_instance'")
        if seed is not None:
            np.random.seed(seed)           # the reference's constructor side effect (kernel_shap.py:225-228)
        self.seed = None if seed is None else int(seed)
        self.plan_mode = plan_mode
        self.plan_seed = 0 if seed is None else int(seed) & 0xFFFFFFFFFFFFFFFF
        self.lib = _cabi.load()
        self.link = convert_to_link(link)
        self.model_callable = model
        torch_models.refuse_module_in_pipeline(model)
        linear_target = model
        if torch_models.is_torch_module(model):
            # a module: recognised and checked here, run on the background below
            if kernel not in ("auto", "simt"):
                raise NotImplementedError(f"kernel={kernel!r}: a torch module runs on the module route (kernel 'auto' or "
                                          "'simt')")
            ens, pipe_spec = None, None
        else:
            # a stacking or soft-voting ensemble of the families below (bare: its spec; behind per-column preprocessing:
            # with the encoding); an all-linear stacking regressor folds into one linear model
            ens = extract_stacking_spec(model)
            if isinstance(ens, LinearModelSpec):
                linear_target, ens = ens, None
            elif ens is None:
                ens = extract_ensemble_spec(model)
            pipe_spec = ens if isinstance(ens, tuple) else None
            if ens is None:
                pipe_spec = extract_tree_pipeline_spec(model)
                if pipe_spec is None:
                    pipe_spec = extract_encoded_pipeline_spec(model)
        # a model behind per-column preprocessing: explained in raw feature space, the device replaying the steps; the
        # extractors below pass its spec through
        target, self.encoding = pipe_spec if pipe_spec is not None else (linear_target if ens is None else ens, None)
        # the model families with their own kernels: the first extractor that reads the model wins; the family's kernels
        # cover at most max_groups groups.  Built per construction, so the module's extractors are looked up when it runs.
        families = ((lambda t: TorchModelSpec(t) if torch_models.is_torch_module(t) else None, torch_models.MAX_GROUPS,
                     "torch modules"),
                    (lambda t: t if isinstance(t, EnsembleSpec) else None, ENSEMBLE_MAX_GROUPS, "soft-voting ensembles"),
                    (lambda t: t if isinstance(t, StackingSpec) else None, STACKING_MAX_GROUPS, "stacking ensembles"),
                    (extract_tree_spec, TREE_MAX_GROUPS, "tree ensembles"),
                    (extract_kernel_machine_spec, KMACH_MAX_GROUPS, "kernel machines"),
                    (extract_mlp_spec, MLP_MAX_GROUPS, "MLPs"),
                    (extract_knn_spec, KNN_MAX_GROUPS, "nearest-neighbour models"))
        for extract, max_groups, family in families:
            own = extract(target)
            if own is not None:
                break
        self.spec = own if own is not None else extract_linear_spec(linear_target)
        if (self.spec.activation == "exp" or getattr(self.spec, "head", None) == "exp") and str(self.link) == "logit":
            raise NotImplementedError("the exp head (log-link GLM regressors) supports link='identity' only: the logit "
                                      "link log(ey / (1 - ey)) is undefined wherever a predicted mean exceeds 1")
        if getattr(self.spec, "head", None) == "iforest" and str(self.link) == "logit":
            raise NotImplementedError("the anomaly head (IsolationForest) supports link='identity' only: its scores are "
                                      "negative and not probabilities, so they have no logit")
        self.data = convert_to_data(data)
        if self.data.transposed:
            raise NotImplementedError("transposed DenseData (group sizes matching axis 0) is not supported")
        bg = np.ascontiguousarray(np.asarray(self.data.data, dtype=np.float64))
        if bg.ndim != 2:
            raise TypeError("background data must be two-dimensional")
        self.N, self.P = bg.shape
        self._bg_outputs = None
        if isinstance(own, TorchModelSpec):
            if self.data.groups_size > max_groups:
                raise NotImplementedError(f"{self.data.groups_size} groups: {family} are explained up to {max_groups} "
                                          "groups")
            if device is not None and int(device) != own.device:
                raise ValueError(f"device={device}: the module is on cuda:{own.device}")
            device = own.device
            self._bg_outputs = own.bind_background(bg)
            self.model_batch_rows = torch_models.model_batch_rows(model_batch_rows, self.N)
        if self.spec.n_features != self.P:
            raise ValueError(f"model expects {self.spec.n_features} columns, background has {self.P}")
        if self.N > 100:
            logger.warning("Using %d background data samples could cause slower run times. Consider using "
                           "shap.sample(data, K) or shap.kmeans(data, K) to summarize the background as K samples.",
                           self.N)
        if device is None:
            import os
            device = int(os.environ.get("LOCAL_RANK", "0"))
        self.device = int(device)

        self._ctx = C.c_void_p()
        _cabi.check(self.lib.dks_create(C.byref(self._ctx), self.device))
        self._stream = None
        if isinstance(own, TorchModelSpec):
            self._bind_torch_stream()           # the background outputs are read on torch's stream
        weights = np.ascontiguousarray(self.data.weights, dtype=np.float64)
        _cabi.check(self.lib.dks_set_background(self._ctx, _cabi.ptr(bg), self.N, self.P, _cabi.ptr(weights)))
        offsets = np.zeros(self.data.groups_size + 1, dtype=np.int32)
        offsets[1:] = np.cumsum([len(g) for g in self.data.groups])
        cols = np.ascontiguousarray(np.concatenate([np.asarray(g, dtype=np.int32) for g in self.data.groups]), dtype=np.int32)
        _cabi.check(self.lib.dks_set_groups(self._ctx, _cabi.ptr(offsets), _cabi.ptr(cols), self.data.groups_size))
        maps = self.spec.maps
        if own is not None and self.data.groups_size > max_groups:
            raise NotImplementedError(f"{self.data.groups_size} groups: {family} are explained up to {max_groups} groups")
        W = None if own is not None else \
            self.spec.W if maps is None else np.zeros((self.spec.R, self.P))
        self._set_encoding(self._ctx)   # before the model: its columns are the encoded ones
        if isinstance(own, EnsembleSpec):
            self._set_ensemble(own, bg, weights)
        elif isinstance(own, StackingSpec):
            self._set_stacking(own, bg, weights)
        elif isinstance(own, TorchModelSpec):
            _cabi.check(self.lib.dks_set_external_model(self._ctx, own.n_outputs, int(own.scalar_out), own.dtype_code))
            y = self._bg_outputs
            _cabi.check(self.lib.dks_set_external_background(self._ctx, C.c_void_p(y.data_ptr()), _dtype_code(y)))
            self._bg_outputs = None
        elif own is not None:
            self._set_own_model(self._ctx, own)
        elif self.spec.activation == "mixture":
            member = {"binary_logistic": _cabi.ACT_BINARY_LOGISTIC, "softmax": _cabi.ACT_SOFTMAX,
                      "ovr": _cabi.ACT_OVR}[self.spec.member]
            _cabi.check(self.lib.dks_set_mixture(self._ctx, self.spec.K, member, self.spec.R // self.spec.K, _cabi.ptr(W),
                                                 _cabi.ptr(self.spec.b), _cabi.ptr(self.spec.pi), int(self.spec.scalar_out)))
        else:
            _cabi.check(self.lib.dks_set_model(self._ctx, _cabi.ptr(W), _cabi.ptr(self.spec.b), self.spec.R,
                                               self.spec.act_code, self.spec.kappa, int(self.spec.scalar_out)))
        if maps is not None:
            _cabi.check(self.lib.dks_set_column_maps(self._ctx, maps.D, maps.R, _cabi.ptr(maps.hdr), _cabi.ptr(maps.keys),
                                                     len(maps.keys), _cabi.ptr(maps.vals), len(maps.vals)))
        link_code = _cabi.LINK_LOGIT if str(self.link) == "logit" else _cabi.LINK_IDENTITY
        _cabi.check(self.lib.dks_set_link(self._ctx, link_code))
        self.set_kernel(kernel)
        _cabi.check(self.lib.dks_set_plan_mode(self._ctx, 1 if plan_mode == "per_instance" else 0, self.plan_seed))
        _cabi.check(self.lib.dks_fit(self._ctx))

        self.D = self.spec.n_outputs
        fnull = np.zeros(self.D)
        expected = np.zeros(self.D)
        _cabi.check(self.lib.dks_get_fnull(self._ctx, _cabi.ptr(fnull), _cabi.ptr(expected)))
        self.vector_out = not self.spec.scalar_out
        self.fnull = fnull
        self.expected_value = expected if self.vector_out else float(expected[0])
        self._nsamples_req = None
        self._plan_cache = {}
        self._l1_uploaded = {}
        self._l1_state = (0, 0, 0, 0)
        self._l1_general_all_select = False
        self._link_fx_parts = []
        self._last_rows = 0
        if self.encoding is not None:
            self._check_encoding(bg)
        if not isinstance(own, TorchModelSpec):     # a module's outputs are the module's: nothing was extracted
            self._check_model_against_callable(bg, own if isinstance(own, (KnnSpec, EnsembleSpec, StackingSpec)) else None)

    def _bind_torch_stream(self):
        """A module: the engine enqueues on torch's current stream of the module's device, so the masked rows, the module
        and the reduction run in order without host synchronisation."""
        import torch
        stream = torch.cuda.current_stream(torch.device("cuda", self.device)).cuda_stream
        if stream != self._stream:
            self.set_stream(stream)
            self._stream = stream

    def _set_encoding(self, ctx):
        e = self.encoding
        if e is not None:
            _cabi.check(self.lib.dks_set_column_encoding(ctx, e.E, _cabi.ptr(e.hdr), _cabi.ptr(e.ops), _cabi.ptr(e.opvals),
                                                         len(e.ops), _cabi.ptr(e.tab), len(e.tab)))

    def _set_own_model(self, ctx, own):
        """The family setter of the C ABI for a tree, kernel-machine, MLP or neighbour spec."""
        if isinstance(own, KnnSpec):
            k = own
            _cabi.check(self.lib.dks_set_knn_model(
                ctx, k.n_fit, _cabi.ptr(k.fitX), _cabi.ptr(k.colw), _cabi.ptr(k.colo), k.k, k.metric_code, k.p,
                k.weights_code, k.R, _cabi.ptr(k.y), k.head_code, int(k.scalar_out)))
        elif isinstance(own, MlpSpec):
            widths, Wm, bm = own.flat()
            _cabi.check(self.lib.dks_set_mlp(ctx, own.n_hidden, _cabi.ptr(widths), _cabi.ptr(Wm), _cabi.ptr(bm),
                                             own.act_code_hidden, own.head_code, int(own.scalar_out)))
        elif isinstance(own, KernelMachineSpec):
            k = own
            _cabi.check(self.lib.dks_set_kernel_machine(
                ctx, k.K, _cabi.ptr(k.sv_off), _cabi.ptr(k.sv), _cabi.ptr(k.dual), k.R, _cabi.ptr(k.intercept),
                _cabi.ptr(k.colw), _cabi.ptr(k.colo), _cabi.ptr(k.gamma), k.kernel_code, k.degree, k.coef0, k.head_code,
                _cabi.ptr(k.cal_a), _cabi.ptr(k.cal_b), _cabi.ptr(k.pi), int(k.scalar_out)))
        else:
            t = own
            _cabi.check(self.lib.dks_set_tree_model(
                ctx, t.n_nodes, _cabi.ptr(t.feature), _cabi.ptr(t.threshold), _cabi.ptr(t.left), _cabi.ptr(t.right),
                _cabi.ptr(t.missing_left), _cabi.ptr(t.value), t.R, t.n_trees, _cabi.ptr(t.roots), _cabi.ptr(t.base),
                t.head_code, t.cmp, int(t.scalar_out)))
            if t.head == "iforest":
                _cabi.check(self.lib.dks_set_tree_offset(ctx, t.offset))

    def _member_contexts(self, spec, bg, weights, members):
        """Appends to ``members`` one context per member of a soft-voting or stacking ensemble (its background and column
        encoding give the setter the model's width)."""
        for _, member in spec.members:
            m = C.c_void_p()
            _cabi.check(self.lib.dks_create(C.byref(m), self.device))
            members.append(m)
            _cabi.check(self.lib.dks_set_background(m, _cabi.ptr(bg), self.N, self.P, _cabi.ptr(weights)))
            self._set_encoding(m)
            self._set_own_model(m, member)

    def _set_ensemble(self, spec, bg, weights):
        """One context per member, handed to ``dks_set_ensemble``, which owns them from then on."""
        members = []
        try:
            self._member_contexts(spec, bg, weights, members)
            ptrs = (C.c_void_p * len(members))(*[m.value for m in members])
            pi = np.ascontiguousarray(spec.weights, dtype=np.float64)
            _cabi.check(self.lib.dks_set_ensemble(self._ctx, len(members), ptrs, _cabi.ptr(pi), spec.n_outputs,
                                                  int(spec.scalar_out)))
        except Exception:
            for m in members:               # not handed over: still ours
                self.lib.dks_destroy(m)
            raise

    def _set_stacking(self, spec, bg, weights):
        """One context per member, as for a soft-voting ensemble, handed to ``dks_set_stacking`` with the final
        estimator and ``MAX_STACKING_BYTES_PER_CALL`` as the workspace budget of a call."""
        members = []
        try:
            self._member_contexts(spec, bg, weights, members)
            ptrs = (C.c_void_p * len(members))(*[m.value for m in members])
            first, count = spec.col_first, spec.col_count
            _cabi.check(self.lib.dks_set_stacking(self._ctx, len(members), ptrs, _cabi.ptr(first), _cabi.ptr(count),
                                                  _cabi.ptr(spec.W), _cabi.ptr(spec.b), spec.W.shape[0], spec.head_code,
                                                  _cabi.ptr(spec.W_pass), spec.n_outputs, int(spec.scalar_out),
                                                  int(MAX_STACKING_BYTES_PER_CALL)))
        except Exception:
            for m in members:               # not handed over: still ours
                self.lib.dks_destroy(m)
            raise

    # ------------------------------------------------------------------------------------------------------
    def encode(self, X):
        """The encoded rows ``pipe[:-1].transform(X)`` [n, E] as the device computes them (``dks_encode_host``), for a
        model behind a column encoding."""
        if self.encoding is None:
            raise TypeError("the model has no column encoding (not a model behind a Pipeline of per-column steps)")
        X = np.ascontiguousarray(np.atleast_2d(np.asarray(X, dtype=np.float64)))
        out = np.zeros((X.shape[0], self.encoding.E))
        _cabi.check(self.lib.dks_encode_host(self._ctx, _cabi.ptr(X), X.shape[0], _cabi.ptr(out)))
        return out

    def _check_encoding(self, bg):
        """The device's encoding of the background must be what the pipeline's own steps give, bit for bit."""
        import warnings
        want = bg
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for step in self.encoding.steps:
                want = step.transform(want)
        if hasattr(want, "toarray"):
            want = want.toarray()
        want = np.asarray(want, dtype=np.float64)
        got = self.encode(bg)
        if want.shape != got.shape or not np.array_equal(got, want, equal_nan=True):
            bad = "shape mismatch" if want.shape != got.shape else \
                f"{int((~((got == want) | (np.isnan(got) & np.isnan(want)))).sum())} entries differ"
            raise ValueError("the column encoding compiled from the pipeline does not reproduce "
                             f"pipeline[:-1].transform(background) bit for bit ({bad}): refusing to explain a different "
                             "function")

    def _check_model_against_callable(self, bg, knn_spec=None):
        """The extracted model must reproduce the user's callable on the background rows.  A neighbour model (or a
        soft-voting ensemble with neighbour members: ``knn_spec`` is then the ``EnsembleSpec``) is compared on the rows
        whose k-th and (k + 1)-th nearest training rows are not equidistant in any neighbour model; a row with such a
        boundary tie is compared with the spec's own NumPy evaluation instead (which of equidistant rows is a neighbour is
        the engine's rule, not scikit-learn's), and at least one row must be compared with the callable."""
        if not callable(self.model_callable):
            return
        want = np.asarray(self.model_callable(bg), dtype=np.float64).reshape(self.N, -1)
        got = self.predict(bg)
        knns = [s for _, s in knn_spec.members if isinstance(s, KnnSpec)] \
            if isinstance(knn_spec, (EnsembleSpec, StackingSpec)) else \
            [knn_spec] if knn_spec is not None else []
        if knns and want.shape == got.shape:
            if self.encoding is not None:
                bg = self.encode(bg)    # the spec reads the encoded columns
            tied = np.zeros(self.N, dtype=bool)
            for k in knns:
                tied |= k.boundary_ties(bg)
            if tied.all():
                raise ValueError("every background row has a tie between its k-th and (k + 1)-th nearest training rows: "
                                 "the neighbour model extracted from `predictor` cannot be checked against "
                                 "predictor(background); refusing to explain a function that was not checked")
            if tied.any():
                logger.warning("%d of %d background rows have equidistant k-th and (k + 1)-th nearest training rows: "
                               "they are checked against the engine's rule (the lower training index wins), not "
                               "against `predictor`", int(tied.sum()), self.N)
                want = want.copy()
                want[tied] = np.asarray(knn_spec(bg[tied]), dtype=np.float64).reshape(int(tied.sum()), -1)
        if want.shape != got.shape or not np.allclose(got, want, rtol=1e-7, atol=1e-9, equal_nan=True):
            raise ValueError("the linear model extracted from `predictor` does not reproduce predictor(background): "
                             "refusing to explain a different function (max abs diff "
                             f"{np.max(np.abs(got - want)) if want.shape == got.shape else 'shape mismatch'})")

    def predict(self, X):
        """Model outputs [n, C] computed on the GPU in float64 (a module: its own outputs, in float64)."""
        if isinstance(self.spec, TorchModelSpec):
            return self.spec.predict(np.atleast_2d(np.asarray(X, dtype=np.float64)))
        X = np.ascontiguousarray(np.atleast_2d(np.asarray(X, dtype=np.float64)))
        out = np.zeros((X.shape[0], self.D))
        _cabi.check(self.lib.dks_predict_host(self._ctx, _cabi.ptr(X), X.shape[0], _cabi.ptr(out)))
        return out

    def set_kernel(self, kernel):
        code = {"auto": _cabi.KERNEL_AUTO, "simt": _cabi.KERNEL_SIMT, "tcgen05": _cabi.KERNEL_TCGEN05,
                "shared": _cabi.KERNEL_SHARED}[kernel]
        _cabi.check(self.lib.dks_set_kernel(self._ctx, code))
        self.kernel = kernel

    def set_option(self, name, value):
        """Tuning knob of the C library (``dks_set_option``): 'fused', 'fused_warps', 'fused_batch', 'fused_table',
        'push_in_kernel', 'graph', 'graph_timing'."""
        _cabi.check(self.lib.dks_set_option(self._ctx, str(name).encode(), int(value)))

    # ------------------------------------------------------------------------------------------------------
    def _set_nsamples(self, nsamples):
        req = 0 if nsamples in ("auto", None) else int(nsamples)
        if req != self._nsamples_req:
            _cabi.check(self.lib.dks_set_nsamples(self._ctx, req))
            self._nsamples_req = req

    def _l1_guard(self, l1_reg, nsamples):
        """Whether the call needs the M histogram to decide which instances run upstream's l1 feature selection
        (``l1_selecting_sizes``); a fixed Lasso strength is refused here, before any work."""
        if l1_reg in (False, 0):
            return False
        return _explicit_l1(l1_reg) is not None or any(_auto_selects(M, nsamples)
                                                       for M in range(2, self.data.groups_size + 1))

    def _apply_l1(self, l1_reg, nsamples, hist):
        """Tells the library which M select (``l1_selecting_sizes``) and uploads the l1 tables of their shared plans,
        cached per (M, S).  The selection runs on the shared plans only, never solved without it: what the library does
        not cover raises."""
        G = self.data.groups_size
        mode, k, sizes = (0, 0, []) if l1_reg in (False, 0) else l1_selecting_sizes(l1_reg, nsamples, G, hist)
        if sizes and self.plan_mode != "shared":
            raise NotImplementedError("l1 feature selection runs with plan_mode='shared' only")
        for M in sizes:
            S, _ = resolve_nsamples(M, nsamples)
            if self._l1_uploaded.get(M) != S:
                self._ensure_shared_plans(hist, nsamples)
                t = l1_tables(self.shared_plan(M, nsamples))
                sqab = np.ascontiguousarray(t["sqa"] + t["sqb"])
                _cabi.check(self.lib.dks_set_l1_tables(
                    self._ctx, M, _cabi.ptr(t["gram_raw"]), _cabi.ptr(t["gram_norm"]), _cabi.ptr(t["colsum"]),
                    _cabi.ptr(t["scale"]), _cabi.ptr(t["bz"]), _cabi.ptr(t["gram_w"]), _cabi.ptr(t["b"]), _cabi.ptr(sqab),
                    t["sum_b"], t["sum_sqb"], t["n_aug"]))
                self._l1_uploaded[M] = S
        sel_lo = sum(1 << (M - 1) for M in sizes if M <= 64)
        sel_hi = sum(1 << (M - 65) for M in sizes if M > 64)
        # the general list (instances with M < G) runs the selection for some; does it hold any that do not select?
        self._l1_general_all_select = bool(sizes) and not any(hist[M] > 0 for M in range(G) if M not in sizes)
        if (mode, k, sel_lo, sel_hi) != self._l1_state:
            _cabi.check(self.lib.dks_set_l1(self._ctx, mode, k, sel_lo, sel_hi))
            self._l1_state = (mode, k, sel_lo, sel_hi)

    def shared_plan(self, M, nsamples="auto"):
        """The coalition plan every instance with ``M`` varying groups shares under ``plan_mode='shared'`` (also the
        source of the enumerated prefix of device-drawn plans).  With a ``seed`` the sampled part comes from a private
        ``RandomState`` keyed by (seed, M, rows): the same plan on every worker, thread and rank whatever the order in
        which they meet the M values.  Without a seed it is drawn from the global legacy stream at first use, like the
        reference's unseeded explainer."""
        S, _ = resolve_nsamples(M, nsamples)
        cached = self._plan_cache.get((M, S))
        if cached is not None:
            return cached
        rng = None
        if self.seed is not None:
            rng = np.random.RandomState((self.seed * 1000003 + 7919 * M + S) & 0xFFFFFFFF)
        plan = build_plan(M, nsamples, rng=rng)
        self._plan_cache[(M, S)] = plan         # what was uploaded is what this accessor reports
        return plan

    def _ensure_shared_plans(self, hist, nsamples):
        refuse_partial_sets_beyond_64_groups(self.data.groups_size, hist)
        for M in range(2, self.data.groups_size + 1):
            if hist[M] == 0:
                continue
            present = C.c_int(0)
            _cabi.check(self.lib.dks_has_shared_plan(self._ctx, M, C.byref(present)))
            if present.value:
                continue
            plan = self.shared_plan(M, nsamples)
            _cabi.check(self.lib.dks_set_shared_plan(self._ctx, M, plan.S, _cabi.ptr(plan.zbits), _cabi.ptr(plan.weights)))
            if M > 128:
                # sixteen-word rows: the (M-1) x (M-1) normal matrix is factored here, once per plan, in float64
                pt, dvec = projection(plan)
                _cabi.check(self.lib.dks_set_plan_projection(self._ctx, M, _cabi.ptr(pt), _cabi.ptr(dvec)))
            nfixed, n_full, n_paired, cdf, weight_left = sampling_info(plan)
            if not device_sampling_supported(M, len(cdf)):
                if self.plan_mode == "per_instance":
                    raise NotImplementedError(f"per-instance device plans support at most 128 groups and "
                                              f"{MAX_SAMPLED_SIZES} sampled subset sizes (M={M})")
                continue
            if M > 64 and self.plan_mode != "per_instance":
                continue                        # two-word rows are drawn per instance only
            _cabi.check(self.lib.dks_set_plan_sampling(self._ctx, M, nfixed, n_full, n_paired, len(cdf),
                                                       _cabi.ptr(cdf) if len(cdf) else None, weight_left))

    def m_histogram(self):
        hist = np.zeros(self.data.groups_size + 1, dtype=np.int32)
        _cabi.check(self.lib.dks_get_m_histogram(self._ctx, _cabi.ptr(hist)))
        return hist

    def varying(self, X):
        """(M [n], bit-mask [n]) of ``KernelExplainer.varying_groups`` for every row of X (GPU)."""
        X = np.ascontiguousarray(np.atleast_2d(np.asarray(X, dtype=np.float64)))
        _cabi.check(self.lib.dks_prepare_host(self._ctx, _cabi.ptr(X), X.shape[0]))
        M = np.zeros(X.shape[0], dtype=np.int32)
        mask = np.zeros(X.shape[0], dtype=np.uint64)
        _cabi.check(self.lib.dks_get_varying(self._ctx, _cabi.ptr(M), _cabi.ptr(mask)))
        return M, mask

    # ------------------------------------------------------------------------------------------------------
    def shap_values(self, X, **kwargs):
        """``KernelExplainer.shap_values``: list of C arrays [n, groups] (vector output) or one array.

        kwargs: ``nsamples`` ('auto' | int), ``l1_reg`` ('auto' | False | 0), ``silent`` (ignored), and
        ``plans`` = per-instance coalition plans ``[(Z [S_i, M_i] | zbits [S_i], w [S_i]) | None, ...]`` evaluated
        instead of the engine's own shared plans (this is how tests give the oracle and the GPU identical inputs)."""
        nsamples = kwargs.pop("nsamples", "auto")
        l1_reg = kwargs.pop("l1_reg", "auto")
        plans = kwargs.pop("plans", None)
        row_offset = int(kwargs.pop("row_offset", 0))
        kwargs.pop("silent", None)
        if kwargs:
            raise TypeError(f"unexpected keyword arguments {sorted(kwargs)}")
        try:
            import pandas as pd
            if isinstance(X, (pd.DataFrame, pd.Series)):
                X = X.values
        except ImportError:  # pragma: no cover
            pass
        try:
            from scipy import sparse
            if sparse.issparse(X):
                X = X.toarray()
        except ImportError:  # pragma: no cover
            pass
        X = np.asarray(X, dtype=np.float64)
        single = X.ndim == 1
        if single:
            X = X.reshape(1, -1)
        assert X.ndim == 2, "Instance must have 1 or 2 dimensions!"
        if X.shape[1] != self.P:
            raise ValueError(f"X has {X.shape[1]} columns, background has {self.P}")
        X = np.ascontiguousarray(X)
        n, G = X.shape[0], self.data.groups_size
        if n == 0:                              # nothing to explain: empty arrays of the right shape (the C ABI wants n > 0)
            self._last_rows = 0
            empty = np.zeros((self.D, 0, G))
            return [empty[c] for c in range(self.D)] if self.vector_out else empty[0]
        self._set_nsamples(nsamples)
        need_hist = self._l1_guard(l1_reg, nsamples)

        rows = self._rows_per_call()
        if n > rows:                  # large inputs go through in row chunks (results are independent per row)
            parts, fx_parts = [], []
            for lo in range(0, n, rows):
                hi = min(n, lo + rows)
                sub = dict(nsamples=nsamples, l1_reg=l1_reg, row_offset=row_offset + lo)
                if plans is not None:
                    sub["plans"] = plans[lo:hi]
                part = self.shap_values(X[lo:hi], **sub)
                fx_parts.append(self.link_predictions().reshape(hi - lo, -1))
                parts.append(part if isinstance(part, list) else [part])
            merged = [np.concatenate([pt[c] for pt in parts], axis=0) for c in range(len(parts[0]))]
            self._link_fx_parts = fx_parts
            self._last_rows = n
            return merged if self.vector_out else merged[0]

        phi = np.empty((self.D, n, G))      # the device writes every entry (zeros for groups that do not vary)
        self._link_fx_parts = []
        if self.plan_mode == "per_instance":
            # the device draws each row's plan from (seed, global row index): tell it where this block starts
            _cabi.check(self.lib.dks_set_row_offset(self._ctx, row_offset))
        if isinstance(self.spec, TorchModelSpec):
            self._explain_module(X, phi, nsamples, l1_reg, plans, need_hist)
        elif plans is not None:
            if G > 64:
                raise NotImplementedError("caller-supplied per-instance plans need at most 64 groups (multi-word coalition "
                                          "rows exist on the shared-plan path only)")
            zb, w, stride = self._pack_external_plans(plans, n, nsamples)
            if need_hist:
                _cabi.check(self.lib.dks_prepare_host(self._ctx, _cabi.ptr(X), n))
                if l1_selecting_sizes(l1_reg, nsamples, G, self.m_histogram())[2]:
                    raise NotImplementedError("l1 feature selection runs on the engine's shared plans, not on "
                                              "caller-supplied per-instance plans -- pass l1_reg=False")
            self._apply_l1(False, nsamples, None)
            _cabi.check(self.lib.dks_explain_host(self._ctx, _cabi.ptr(X), n, _cabi.ptr(phi), _cabi.ptr(zb), _cabi.ptr(w),
                                                  stride))
        else:
            if need_hist:
                _cabi.check(self.lib.dks_prepare_host(self._ctx, _cabi.ptr(X), n))
                hist = self.m_histogram()
                self._ensure_shared_plans(hist, nsamples)
                self._apply_l1(l1_reg, nsamples, hist)
            else:
                self._apply_l1(False, nsamples, None)
            rc = self.lib.dks_explain_host(self._ctx, _cabi.ptr(X), n, _cabi.ptr(phi), None, None, 0)
            if rc == _cabi.DKS_ERR_PLAN_MISSING:
                # first call (or a new M): build the missing plans from the M histogram and run again
                self._ensure_shared_plans(self.m_histogram(), nsamples)
                rc = self.lib.dks_explain_host(self._ctx, _cabi.ptr(X), n, _cabi.ptr(phi), None, None, 0)
            _cabi.check(rc)

        self._last_rows = n
        if not self.vector_out:
            return phi[0, 0] if single else phi[0]
        if single:
            return [phi[c, 0] for c in range(self.D)]
        return [phi[c] for c in range(self.D)]

    def _explain_module(self, X, phi, nsamples, l1_reg, plans, need_hist):
        """One block of rows through a module: stage 1 on the module's outputs, the plans (and the l1 decision), then
        mask -> module -> reduce per block of ``model_batch_rows`` masked rows into one reused input tensor, then the
        solve into ``phi``."""
        import torch
        n, G, spec = X.shape[0], self.data.groups_size, self.spec
        dev = torch.device("cuda", self.device)
        with torch.cuda.device(dev), torch.inference_mode():
            self._bind_torch_stream()
            X_dev = torch.from_numpy(X).to(dev)             # read by every mask launch until finish returns
            fx = spec.outputs(X_dev.to(spec.dtype))
            _cabi.check(self.lib.dks_external_prepare(self._ctx, C.c_void_p(X_dev.data_ptr()), n,
                                                      C.c_void_p(fx.data_ptr()), _dtype_code(fx)))
            zb = w = None
            stride = 0
            if plans is not None:
                zb, w, stride = self._pack_external_plans(plans, n, nsamples)
                if need_hist and l1_selecting_sizes(l1_reg, nsamples, G, self.m_histogram())[2]:
                    raise NotImplementedError("l1 feature selection runs on the engine's shared plans, not on "
                                              "caller-supplied per-instance plans -- pass l1_reg=False")
                self._apply_l1(False, nsamples, None)
            elif need_hist:
                hist = self.m_histogram()
                self._ensure_shared_plans(hist, nsamples)
                self._apply_l1(l1_reg, nsamples, hist)
            else:
                self._apply_l1(False, nsamples, None)
            total = C.c_int64(0)
            rc = self.lib.dks_external_begin(self._ctx, _cabi.ptr(zb), _cabi.ptr(w), stride, C.byref(total))
            if rc == _cabi.DKS_ERR_PLAN_MISSING:
                # first call (or a new M): build the missing plans from the M histogram and lay the call out again
                self._ensure_shared_plans(self.m_histogram(), nsamples)
                rc = self.lib.dks_external_begin(self._ctx, _cabi.ptr(zb), _cabi.ptr(w), stride, C.byref(total))
            _cabi.check(rc)
            blocks = torch_models.plan_blocks(total.value, self.N, self.model_batch_rows)
            rows_in = torch.empty((blocks[0][1] if blocks else 0, self.P), dtype=spec.dtype, device=dev)
            for row0, rows in blocks:
                x = rows_in[:rows]
                _cabi.check(self.lib.dks_external_mask(self._ctx, row0, rows, C.c_void_p(x.data_ptr())))
                y = spec.outputs(x)
                _cabi.check(self.lib.dks_external_reduce(self._ctx, row0, rows, C.c_void_p(y.data_ptr()),
                                                         _dtype_code(y)))
            _cabi.check(self.lib.dks_external_finish(self._ctx, _cabi.ptr(phi)))

    def _refuse_module(self, what):
        if isinstance(self.spec, TorchModelSpec):
            raise NotImplementedError(f"{what}: a torch module runs between the engine's launches, so it cannot be "
                                      "explained from device rows in one enqueued sequence or replayed as a CUDA graph; "
                                      "use shap_values")

    def _rows_per_call(self):
        """Rows per C-ABI call (``rows_per_call``); a column encoding also bounds the encoded rows of a call by
        ``MAX_ENCODED_BYTES_PER_CALL`` (results are per row and device plans keyed by the global row: the block size
        does not change phi)."""
        rows = rows_per_call(self.spec.act_code, self.D, self.plan_mode, self.data.groups_size, self.spec.R)
        if self.encoding is not None:
            rows = min(rows, max(1, MAX_ENCODED_BYTES_PER_CALL // (8 * self.encoding.E)))
        if isinstance(self.spec, (EnsembleSpec, StackingSpec, TorchModelSpec)):
            # the members' weighted background means (or the module's): C outputs x S rows per instance, S at most that
            # of all G groups
            S, _ = resolve_nsamples(self.data.groups_size, self._nsamples_req or "auto")
            rows = min(rows, max(1, MAX_ENSEMBLE_BYTES_PER_CALL // (8 * self.D * (S + 2))))
        return rows

    def link_predictions(self):
        """``link(f(x))`` of the rows of the last ``shap_values`` call, ``[n, C]`` (``[n]`` for scalar-output models):
        stage 1 of the explain call computes it on the device, so ``KernelShap.build_explanation`` does not have to run
        the predictor over ``X`` again for ``raw_prediction`` (kernel_shap.py:949)."""
        if self._link_fx_parts:                 # the call went through in row chunks
            out = np.concatenate(self._link_fx_parts, axis=0)
        elif self._last_rows == 0:
            return None
        else:
            out = np.zeros((self._last_rows, self.D))
            rc = self.lib.dks_get_link_fx(self._ctx, _cabi.ptr(out), self._last_rows)
            if rc == _cabi.DKS_ERR_INVALID:     # another call (varying(), explain_device()) ran stage 1 since
                return None
            _cabi.check(rc)
        return out if self.vector_out else out[:, 0]

    def summarise(self, n, segments=None, want_sums=False):
        """``KernelShap.build_explanation`` post-processing on the device, off the phi of the last host-path
        ``shap_values`` call over ``n`` rows (kernel_shap.py:36-109, :112-207, :952-956): mean |phi| per output and
        aggregated (``mean_abs`` [C + 1, Gp]), their descending order (``order``), the arg-max class of the raw prediction
        (``argmax`` [n]) and, with ``segments`` (offsets of consecutive groups to add up: ``sum_categories``), the summed
        shap values (``phi_sum`` [C, n, Gp]).  Returns None when the last call is not resident (row chunks, other calls)."""
        if n != self._last_rows or self._link_fx_parts:
            return None
        G = self.data.groups_size
        seg = None if segments is None else np.ascontiguousarray(segments, dtype=np.int32)
        Gp = G if seg is None else len(seg) - 1
        mean_abs = np.zeros((self.D + 1, Gp))
        order = np.zeros((self.D + 1, Gp), dtype=np.int32)
        argmax = np.zeros(n, dtype=np.int32)
        phi_sum = np.zeros((self.D, n, Gp)) if (want_sums and seg is not None) else None
        rc = self.lib.dks_summarise_host(self._ctx, n, _cabi.ptr(seg), Gp, _cabi.ptr(phi_sum), _cabi.ptr(mean_abs),
                                         _cabi.ptr(order), _cabi.ptr(argmax))
        if rc == _cabi.DKS_ERR_INVALID:
            return None
        _cabi.check(rc)
        return {"mean_abs": mean_abs, "order": order, "argmax": argmax, "phi_sum": phi_sum}

    def instance_plans(self):
        """Plans the device drew in the last ``plan_mode='per_instance'`` call: ``(zbits uint64[n, stride],
        w float64[n, stride])`` -- rows past an instance's S are zero; beyond 64 groups the rows have two words and
        ``zbits`` is ``uint64[n, stride, 2]`` (little-endian: bit k of the row is bit k % 64 of word k // 64).  For audits
        and tests."""
        n, stride, words = C.c_int(0), C.c_int(0), C.c_int(0)
        _cabi.check(self.lib.dks_get_instance_plans_w(self._ctx, None, None, C.byref(n), C.byref(stride), C.byref(words)))
        shape = (n.value, stride.value) if words.value <= 1 else (n.value, stride.value, words.value)
        zb = np.zeros(shape, dtype=np.uint64)
        w = np.zeros((n.value, stride.value), dtype=np.float64)
        if n.value:
            _cabi.check(self.lib.dks_get_instance_plans_w(self._ctx, _cabi.ptr(zb), _cabi.ptr(w), C.byref(n),
                                                          C.byref(stride), C.byref(words)))
        return zb, w

    def _pack_external_plans(self, plans, n, nsamples):
        if len(plans) != n:
            raise ValueError(f"got {len(plans)} plans for {n} instances")
        stride = max([len(p[1]) for p in plans if p is not None and p[1] is not None] + [2])
        zb = np.zeros((n, stride), dtype=np.uint64)
        w = np.zeros((n, stride), dtype=np.float64)
        for i, p in enumerate(plans):
            if p is None or p[1] is None:
                continue
            Z, wi = p[-2], np.asarray(p[-1], dtype=np.float64)
            Z = np.asarray(Z)
            bits = pack_dense_plan(Z) if Z.ndim == 2 else Z.astype(np.uint64)
            zb[i, :len(bits)] = bits
            w[i, :len(wi)] = wi
        return zb, w, stride

    # ---- device-resident API (torch tensors appear only as raw pointers) ---------------------------------------
    def set_stream(self, cuda_stream_ptr):
        """Enqueue the engine's work on the given ``cudaStream_t`` (e.g. ``torch.cuda.current_stream().cuda_stream``)."""
        _cabi.check(self.lib.dks_set_stream(self._ctx, C.c_void_p(int(cuda_stream_ptr))))

    def explain_device(self, X_dev_ptr, n, phi_dev_ptr, nsamples="auto"):
        """Asynchronously explain ``n`` rows resident in device memory (float64 [n, D] at ``X_dev_ptr``) into the device
        buffer ``phi_dev_ptr`` (float64 [C, n, G]) using the shared plans already on the device.  Call ``check_status()``
        after synchronising to learn about missing plans / numerical failures."""
        self._refuse_module("explain_device")
        self._set_nsamples(nsamples)
        self._apply_l1(False, nsamples, None)             # the device-resident call is the plain constrained WLS
        _cabi.check(self.lib.dks_run_dev(self._ctx, C.c_void_p(int(X_dev_ptr)), int(n), C.c_void_p(int(phi_dev_ptr))))

    def explain_block_to_device(self, X, nsamples="auto", l1_reg="auto", row_offset=0, silent=None):
        """Explain host rows ``X`` and leave the shap values ON THE DEVICE: returns a float64 CUDA tensor ``[C, n, G]``
        (torch owns the buffers; the engine sees raw pointers).  Used by the SPMD path of ``DistributedExplainer`` so that
        the all-gather runs on what the solve wrote, without a host round trip.  Zero rows give an empty tensor."""
        self._refuse_module("explain_block_to_device")
        import torch
        X = np.ascontiguousarray(np.atleast_2d(np.asarray(X, dtype=np.float64)))
        n, G = X.shape[0], self.data.groups_size
        dev = torch.device("cuda", self.device)
        phi = torch.empty((self.D, n, G), dtype=torch.float64, device=dev)
        if n == 0:
            return phi
        if X.shape[1] != self.P:
            raise ValueError(f"X has {X.shape[1]} columns, background has {self.P}")
        self._set_nsamples(nsamples)
        need_hist = self._l1_guard(l1_reg, nsamples)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            if getattr(self, "_block_stream", None) != stream.cuda_stream:
                self.set_stream(stream.cuda_stream)
                self._block_stream = stream.cuda_stream
            X_dev = torch.from_numpy(X).to(dev, non_blocking=True)
            if self.plan_mode == "per_instance":
                _cabi.check(self.lib.dks_set_row_offset(self._ctx, int(row_offset)))
            if need_hist:
                _cabi.check(self.lib.dks_prepare_dev(self._ctx, C.c_void_p(X_dev.data_ptr()), n))
                hist = self.m_histogram()
                self._ensure_shared_plans(hist, nsamples)
                self._apply_l1(l1_reg, nsamples, hist)
            else:
                self._apply_l1(False, nsamples, None)
            for attempt in range(2):
                _cabi.check(self.lib.dks_run_dev(self._ctx, C.c_void_p(X_dev.data_ptr()), n, C.c_void_p(phi.data_ptr())))
                detail = C.c_int(0)
                rc = self.lib.dks_last_status(self._ctx, C.byref(detail))            # synchronises the stream
                if rc == _cabi.DKS_ERR_PLAN_MISSING and attempt == 0:
                    self._ensure_shared_plans(self.m_histogram(), nsamples)       # first call / new M: build and rerun
                    continue
                _cabi.check(rc)
                break
        self._last_rows = 0                     # link_predictions() refers to host-path calls only
        return phi

    def set_peers(self, world, rank, gathered_ptrs, slab_doubles):
        """Multi-GPU push all-gather: ``gathered_ptrs[r]`` = device address (mapped in this process) of rank r's gathered
        ``[world, C, n, G]`` buffer; after every ``explain_device`` this rank's phi is stored into slab ``rank`` of every
        peer's buffer by the engine's own kernel.  ``world <= 1`` switches it off."""
        if world <= 1:
            _cabi.check(self.lib.dks_set_peers(self._ctx, 0, 0, None, 0))
            return
        ptrs = np.asarray([int(p) for p in gathered_ptrs], dtype=np.uint64)
        _cabi.check(self.lib.dks_set_peers(self._ctx, int(world), int(rank), _cabi.ptr(ptrs), int(slab_doubles)))

    def set_peer_flags(self, flag_ptrs):
        """Multi-GPU: ``flag_ptrs[r]`` = device address (mapped here) of rank r's zero-initialised ``uint64[world]`` flag
        array.  Every ``explain_device`` then ends with the engine's own cross-GPU signal / wait, so the gathered buffer is
        complete when the stream reaches the next operation.  ``None`` switches it off."""
        if flag_ptrs is None:
            _cabi.check(self.lib.dks_set_peer_flags(self._ctx, None))
            return
        ptrs = np.asarray([int(p) for p in flag_ptrs], dtype=np.uint64)
        _cabi.check(self.lib.dks_set_peer_flags(self._ctx, _cabi.ptr(ptrs)))

    def graph_launches(self):
        """How many ``explain_device`` calls were replayed as one CUDA-graph launch."""
        cnt = C.c_int64(0)
        _cabi.check(self.lib.dks_graph_launches(self._ctx, C.byref(cnt)))
        return cnt.value

    def check_status(self):
        """Synchronise the engine's stream and raise if the last explain reported a problem."""
        detail = C.c_int(0)
        _cabi.check(self.lib.dks_last_status(self._ctx, C.byref(detail)))

    # ---- KernelExplainerWrapper members (kernel_shap.py:231-261) ---------------------------------------------
    def get_explanation(self, X, **kwargs):
        """Accepts an array, or a ``(batch_index, batch)`` tuple when called from a distributed context."""
        if isinstance(X, tuple):
            batch_idx, batch = X
            return batch_idx, self.shap_values(batch, **kwargs)
        return self.shap_values(X, **kwargs)

    def return_attribute(self, name):
        return self.__getattribute__(name)

    # ---- introspection used by bench.py / tests -----------------------------------------------------------------
    def kernel_launches(self):
        v = C.c_int64(0)
        _cabi.check(self.lib.dks_kernel_launches(self._ctx, C.byref(v)))
        return int(v.value)

    def last_timings_ms(self):
        out = np.zeros(3, dtype=np.float32)
        _cabi.check(self.lib.dks_last_timings(self._ctx, _cabi.ptr(out)))
        return {"prepare": float(out[0]), "coalitions": float(out[1]), "total": float(out[2])}

    _PATH_NAMES = {
        "shared": ("none", "fused", "smem", None, "softmax", "affine", "ovr", "exp", "mixture"),   # 3: not used
        "solve": ("none", "fused", "pmat", "wls_shared", "wide", "l1"),
        "general": ("none", "tc", "simt", "flagged", "simt_wide", "trees", "kmach", "mlp", "knn", "ensemble", "torch", "stacking"),
    }

    def last_path(self):
        """Which kernels the last explain call launched (``dks_last_path``), recorded when the call was enqueued (a
        replayed CUDA graph reports the call it captured): ``shared`` (shared-plan coalition kernel: 'none' | 'fused' |
        'smem' | 'softmax' | 'ovr', or 'affine' for the identity head and 'exp' for the exp head, whose y needs no
        coalition kernel), ``chunks`` (background chunks), ``warps`` / ``grid`` (warps per CTA and CTAs of that kernel),
        ``fused_B`` / ``fused_NI``, ``solve`` ('none' | 'fused' | 'pmat' | 'wls_shared' | 'wide' | 'l1'), ``pmat_kpad``,
        ``general`` (kernel of the remaining instances: 'none' | 'tc' | 'simt' | 'flagged', the last meaning they
        are reported as unsupported, not computed, 'simt_wide': per-instance plans of 65..128 groups, 'trees': the tree
        kernel, which takes every instance of a tree ensemble, 'kmach': the kernel-machine kernel, which takes every
        instance of a kernel machine, 'mlp': the MLP kernel, which takes every instance of a multi-layer perceptron, or
        'knn': the neighbour kernel, which takes every instance of a k-nearest-neighbour model, or 'ensemble': the
        members' kernels and the ensemble's tail, which take every instance of a soft-voting ensemble, or 'torch': the
        ensemble's tail on the background means of a module's outputs, every instance of a module, or 'stacking': per
        background chunk the members' kernels and the final estimator's reduction, then the ensemble's tail, every
        instance of a stacking ensemble),
        ``cta_warps`` (warps per CTA the fused kernel runs: ``warps``
        row-group slices at one warp each, or fewer slices shared by several warps each) and ``bg_weights`` ('uniform' |
        'weighted': which instantiation of the shared-plan kernels ran; background weights that are not all equal take
        the weighted one), ``fused_table`` (1: the fused kernel read y from the plan's link table, passes outside its
        domain excepted; 0: the exact loop over the background throughout) and ``general_l1`` (1: the general list's
        instances whose M selects ran the l1 selection -- moments on the CUDA-core kernel, then the LARS kernel; ``general``
        then names the kernel of the others, or 'simt' when every instance of the general list selected)."""
        out = np.zeros(13, dtype=np.int32)
        _cabi.check(self.lib.dks_last_path(self._ctx, _cabi.ptr(out), len(out)))
        names = self._PATH_NAMES
        general = names["general"][out[8]]
        if out[12] and self._l1_general_all_select and general != "torch":
            general = "simt"
        return {"shared": names["shared"][out[0]], "chunks": int(out[1]), "warps": int(out[2]), "grid": int(out[3]),
                "fused_B": int(out[4]), "fused_NI": int(out[5]), "solve": names["solve"][out[6]],
                "pmat_kpad": int(out[7]), "general": general,
                "cta_warps": int(out[9]), "bg_weights": ("uniform", "weighted")[out[10]], "fused_table": int(out[11]),
                "general_l1": int(out[12])}

    def general_l1_timings_ms(self):
        """Device time of the last explain's l1 selection on the general list (``last_path()["general_l1"]``), from the
        engine's CUDA events: ``general`` (the CUDA-core kernel forming the moments) and ``lars`` (the LARS kernel)."""
        out = np.zeros(2, dtype=np.float32)
        _cabi.check(self.lib.dks_last_general_l1_timings(self._ctx, _cabi.ptr(out)))
        return {"general": float(out[0]), "lars": float(out[1])}

    def fused_table_info(self, M):
        """The fused kernel's link table of the plan over M groups: ``bytes`` (0: no table, the exact loop runs) and
        ``fallback_passes``, the passes of this engine's fused launches so far that left a table's domain and took the
        exact loop."""
        nbytes, fb = C.c_int64(0), C.c_int64(0)
        _cabi.check(self.lib.dks_fused_table_info(self._ctx, int(M), C.byref(nbytes), C.byref(fb)))
        return {"bytes": int(nbytes.value), "fallback_passes": int(fb.value)}

    def debug_scores(self, X, instance, nsamples="auto"):
        """Raw accumulator tile of the tensor-core kernel for one instance: float32 [S_cap, Npad] of scaled masked scores
        ``-kappa*log2(e) * score(s, j)`` (tests only)."""
        _cabi.check(self.lib.dks_debug_score_dump(self._ctx, int(instance)))
        try:
            self.shap_values(X, nsamples=nsamples, l1_reg=False)
            buf = np.zeros(1 << 22, dtype=np.float32)
            rows, cols = C.c_int(0), C.c_int(0)
            _cabi.check(self.lib.dks_debug_get_scores(self._ctx, _cabi.ptr(buf), buf.size, C.byref(rows), C.byref(cols)))
        finally:
            _cabi.check(self.lib.dks_debug_score_dump(self._ctx, -1))
        return buf[:rows.value * cols.value].reshape(rows.value, cols.value).copy()

    def debug_timeline(self, X, nsamples="auto"):
        """clock64 timeline [6, 256] of CTA 0 of the tensor-core kernel (see ``dks_debug_get_timeline``); tests/tuning only."""
        self.shap_values(X, nsamples=nsamples, l1_reg=False)          # plans uploaded, steady state
        _cabi.check(self.lib.dks_debug_score_dump(self._ctx, 0))
        try:
            self.shap_values(X, nsamples=nsamples, l1_reg=False)
            buf = np.zeros((6, 256), dtype=np.float32)
            _cabi.check(self.lib.dks_debug_get_timeline(self._ctx, _cabi.ptr(buf)))
        finally:
            _cabi.check(self.lib.dks_debug_score_dump(self._ctx, -1))
        return buf

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self.lib.dks_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:  # pragma: no cover
            pass
