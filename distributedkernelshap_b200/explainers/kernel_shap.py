"""``KernelShap`` with the reference's public API over the CUDA engine (reference: explainers/kernel_shap.py).

Kept identical to the reference: constructor / ``fit`` / ``explain`` / ``build_explanation`` signatures
(kernel_shap.py:266-273, :697-704, :810-815, :900-904), the input checks and the flags they set (:369-501), the
background -> ``DenseData`` conversion (:544-671), metadata bookkeeping (:673-695, :796-806), the ``Explanation``
payload (:963-980), ``rank_by_importance`` (:36-109) and ``sum_categories`` (:112-207) semantics.

Replaced: the object stored in ``self._explainer``.  The reference puts a ``shap.KernelExplainer`` subclass there
(``KernelExplainerWrapper``, :217-261) or a ray ``DistributedExplainer`` of them (:777-785); here
``KernelExplainerWrapper`` is the CUDA-backed ``GpuKernelExplainer`` and ``DistributedExplainer`` shards rows over
GPUs.  Nothing in this module computes SHAP values on the CPU.
"""
import copy
import logging
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import pandas as pd
from scipy import sparse

from distributedkernelshap_b200 import data as shap_data
from distributedkernelshap_b200.data import Data, DenseData, DenseDataWithIndex, convert_to_link
from distributedkernelshap_b200.engine import GpuKernelExplainer
from distributedkernelshap_b200.explainers.distributed import DistributedExplainer
from distributedkernelshap_b200.torch_models import is_torch_module
from distributedkernelshap_b200.explainers.interface import (DEFAULT_DATA_KERNEL_SHAP, DEFAULT_META_KERNEL_SHAP,
                                                              Explainer, Explanation, FitMixin)

logger = logging.getLogger(__name__)

KERNEL_SHAP_PARAMS = [
    'link',
    'group_names',
    'groups',
    'weights',
    'summarise_background',
    'summarise_result',
    'kwargs',
]

KERNEL_SHAP_BACKGROUND_THRESHOLD = 300

DISTRIBUTED_OPTS = {
    'n_cpus': None,
    'batch_size': None,
    'actor_cpu_fraction': 1.0,
}


def rank_by_importance(shap_values: List[np.ndarray],
                       feature_names: Union[List[str], Tuple[str], None] = None) -> Dict:
    """Ranks features by mean absolute shap value, per model output and aggregated over outputs.

    Returns ``{'0': {'ranked_effect': ..., 'names': ...}, ..., 'aggregated': {...}}`` with effects and names sorted
    from most to least important (same structure as the reference, kernel_shap.py:54-69)."""
    if shap_values[0].ndim == 1:
        shap_values = [np.atleast_2d(arr) for arr in shap_values]
    n_feats = shap_values[0].shape[1]

    default_names = ['feature_{}'.format(i) for i in range(n_feats)]
    if not feature_names:
        feature_names = default_names
    elif len(feature_names) != n_feats:
        logger.warning(
            "The feature names provided do not match the number of shap values estimated. "
            "Received {} feature names but estimated {} shap values!".format(len(feature_names), n_feats))
        feature_names = default_names

    def _ranked(magnitudes):
        order = np.argsort(magnitudes)[::-1]
        return {'ranked_effect': magnitudes[order], 'names': [feature_names[i] for i in order]}

    per_output = [np.abs(values).mean(axis=0) for values in shap_values]
    importances = {str(idx): _ranked(mag) for idx, mag in enumerate(per_output)}
    importances['aggregated'] = _ranked(np.sum(per_output, axis=0))
    return importances


def category_segments(width: int, start_idx: Sequence[int], enc_feat_dim: Sequence[int]) -> np.ndarray:
    """Offsets ``[0, ..., width]`` of the column segments ``sum_categories`` adds up (one per categorical variable, one per
    remaining column): the form the device-side summary takes."""
    block_len = dict(zip(start_idx, enc_feat_dim))
    offsets, col = [], 0
    while col < width:
        offsets.append(col)
        col += block_len.get(col, 1)
    offsets.append(width)
    return np.asarray(offsets, dtype=np.int32)


def importances_from_device(summary: Dict, feature_names) -> Dict:
    """``rank_by_importance`` output from the device-side summary (mean |phi| [C + 1, G'] and descending order)."""
    mean_abs, order = summary['mean_abs'], summary['order']
    n_feats = mean_abs.shape[1]
    if not feature_names or len(feature_names) != n_feats:
        if feature_names:
            logger.warning(
                "The feature names provided do not match the number of shap values estimated. "
                "Received {} feature names but estimated {} shap values!".format(len(feature_names), n_feats))
        feature_names = ['feature_{}'.format(i) for i in range(n_feats)]
    out = {}
    for r in range(mean_abs.shape[0]):
        key = str(r) if r < mean_abs.shape[0] - 1 else 'aggregated'
        out[key] = {'ranked_effect': mean_abs[r][order[r]], 'names': [feature_names[i] for i in order[r]]}
    return out


def sum_categories(values: np.ndarray, start_idx: Sequence[int], enc_feat_dim: Sequence[int]):
    """Sums, for every ``start_idx[i]``, the ``enc_feat_dim[i]`` consecutive columns starting there (the encoded levels
    of one categorical variable); other columns are kept.  Rank-3 inputs (interaction values) are reduced along both
    trailing axes."""
    if start_idx is None or enc_feat_dim is None:
        raise ValueError("Both the start indices or the encoding dimension need to be specified!")
    if len(enc_feat_dim) != len(start_idx):
        raise ValueError("The lengths of the sequences of start indices and encodings must be equal!")
    if sum(enc_feat_dim) > values.shape[-1]:
        raise ValueError("The sum of the encoded features dimensions exceeds data dimension!")
    if values.ndim not in (2, 3):
        raise ValueError(
            f"Shap value summarisation can only be applied to tensors of shap values (dim=2) or shap "
            f"interaction values (dim=3). The tensor to be summarised had dimension {values.shape}!")

    width = values.shape[-1]
    block_len = dict(zip(start_idx, enc_feat_dim))
    segment_starts, col = [], 0
    while col < width:
        segment_starts.append(col)
        col += block_len.get(col, 1)

    if values.ndim == 3:
        reduced = np.add.reduceat(values, segment_starts, axis=2)
        return np.add.reduceat(reduced, segment_starts, axis=1)
    return np.add.reduceat(values, segment_starts, axis=1)


class KernelExplainerWrapper(GpuKernelExplainer):
    """Name the reference uses for the per-worker explainer (kernel_shap.py:217-261).  Here it is the CUDA engine:
    same constructor shape ``(predictor, background_data, link=..., seed=...)``, ``get_explanation`` accepting an
    array or a ``(batch_index, batch)`` tuple, and ``return_attribute``."""


class KernelShap(Explainer, FitMixin):

    def __init__(self,
                 predictor: Callable,
                 link: str = 'identity',
                 feature_names: Union[List[str], Tuple[str], None] = None,
                 categorical_names: Optional[Dict[int, List[str]]] = None,
                 task: str = 'classification',
                 seed: int = None,
                 distributed_opts: Optional[Dict] = None,
                 plan_mode: str = 'shared',
                 model_batch_rows: Optional[int] = None):
        """KernelSHAP explainer with grouping of encoded categorical variables; see the reference docstring
        (kernel_shap.py:274-337) for parameter semantics -- they are unchanged.

        ``distributed_opts``: ``n_cpus`` now counts worker GPUs (one CUDA context each) instead of ray CPU actors,
        ``batch_size`` still sets the mini-batch of rows sent to a worker at a time.  Under ``torchrun`` every rank is
        one worker and the shap values are all-gathered over NCCL.

        ``plan_mode`` (not in the reference): ``'shared'`` evaluates one coalition plan per number of varying groups for
        all instances (drawn on the host from the seeded NumPy stream); ``'per_instance'`` draws a fresh plan for every
        instance on the GPU, as shap does on the CPU, from a counter-based stream keyed by (seed, row index).

        ``predictor`` may also be a ``torch.nn.Module`` on a CUDA device (see ``GpuKernelExplainer``); ``model_batch_rows``
        (not in the reference) then caps the masked rows per module call.  A module is explained on one GPU: it cannot
        be combined with ``distributed_opts``."""
        super().__init__(meta=copy.deepcopy(DEFAULT_META_KERNEL_SHAP))

        self.link = link
        self.predictor = predictor
        self.feature_names = feature_names if feature_names else []
        self.categorical_names = categorical_names if categorical_names else {}
        self.task = task
        self.seed = seed
        self.plan_mode = plan_mode
        self._update_metadata({"task": self.task})

        self.use_groups = False            # user passed groups / group names
        self.create_group_names = False    # groups without usable names -> 'group_i'
        self.transposed = False            # group sizes match axis 0 of the background instead of axis 1
        self.ignore_weights = False        # weights unusable -> dropped
        self.summarise_result = False      # sum shap values over encoded levels after the fact
        self.summarise_background = False  # background was subsampled / clustered
        self._fitted = False
        self.model_batch_rows = model_batch_rows
        if distributed_opts and is_torch_module(predictor):
            raise NotImplementedError("distributed_opts with a torch.nn.Module: the pool replicates the explainer on "
                                      "every GPU, and moving a module between devices is not supported; explain it on "
                                      "its own device without distributed_opts")
        self.distributed_opts = copy.deepcopy(DISTRIBUTED_OPTS)
        if distributed_opts:
            self.distributed_opts.update(distributed_opts)
        self.distributed_opts['algorithm'] = 'kernel_shap'
        self.distribute = True if self.distributed_opts['n_cpus'] else False

    # ------------------------------------------------------------------------------------------------------
    # input validation (kernel_shap.py:369-501): only warns and sets flags, never raises
    # ------------------------------------------------------------------------------------------------------
    def _check_inputs(self, background_data, group_names, groups, weights) -> None:
        if isinstance(background_data, Data):
            # a prepared data object is trusted unless it was produced by the summarisation step
            if not self.summarise_background:
                self.use_groups = False
                return
            background_data = background_data.data

        if isinstance(background_data, np.ndarray) and background_data.ndim == 1:
            background_data = np.atleast_2d(background_data)

        n_records = background_data.shape[0]
        if n_records > KERNEL_SHAP_BACKGROUND_THRESHOLD:
            logger.warning(
                "Large datasets can cause slow runtimes for shap. The background dataset provided has {} records. "
                "Consider passing a subset or allowing the algorithm to automatically summarize the data by setting "
                "the summarise_background=True or setting summarise_background to 'auto' which will default to {} "
                "samples!".format(n_records, KERNEL_SHAP_BACKGROUND_THRESHOLD))

        if group_names and not groups:
            logger.info("Specified group_names but no corresponding sequence 'groups' with indices for each group was "
                        "specified. All groups will have len=1.")
            if len(group_names) not in background_data.shape:
                logger.warning(
                    "Specified {} group names but data dimension is {}. When grouping indices are not specifies the "
                    "number of group names should equal one of the data dimensions! Igoring grouping inputs!".format(
                        len(group_names), background_data.shape))
                self.use_groups = False

        if groups and not group_names:
            logger.warning("No group names specified but groups specified! Automatically assigning 'group_' name for "
                           "every index group specified!")
            if self.feature_names and len(self.feature_names) == len(groups):
                group_names = self.feature_names
            else:
                if self.feature_names:
                    logger.warning(
                        "Number of feature names specified did not match the number of groups. Specified {} groups "
                        "and {} features names. Creating default names for specified groups".format(
                            len(groups), len(self.feature_names)))
                self.create_group_names = True

        if groups:
            self._check_groups(background_data, groups, group_names)
        if weights is not None:
            self._check_weights(background_data, weights)

    def _check_groups(self, background_data, groups, group_names) -> None:
        if not isinstance(groups[0], (tuple, list)):
            logger.warning(
                "groups should be specified as List[Union[Tuple[int], List[int]]] where each sublist represents a "
                "group and int represent group instance. Specified group elements have type {}. Ignoring grouping "
                "inputs!".format(type(groups[0])))
            self.use_groups = False

        expected_dim = sum(len(g) for g in groups)
        actual_dim = background_data.shape[0] if background_data.ndim == 1 else background_data.shape[1]
        if expected_dim != actual_dim:
            if background_data.shape[0] == expected_dim:
                logger.warning("The sum of the group indices list did not match the data dimension along axis=1 but "
                               "matched dimension along axis=0. Consider transposing the data!")
                self.transposed = True
            else:
                logger.warning(
                    "The sum of the group sizes specified did not match the number of features. Sum of group sizes: "
                    "{}. Number of features: {}. Ignoring grouping inputs!".format(expected_dim, actual_dim))
                self.use_groups = False

        if group_names and len(group_names) != len(groups):
            logger.warning(
                "The number of group names specified does not match the number of groups. Received {} groups and {} "
                "names! Ignoring grouping inputs!".format(len(groups), len(group_names)))
            self.use_groups = False

    def _check_weights(self, background_data, weights) -> None:
        if background_data.ndim == 1 or background_data.shape[0] == 1:
            logger.warning("Specified weights but the background data has only one record. Weights will be ignored!")
            self.ignore_weights = True
        else:
            data_dim, feat_dim = background_data.shape[0], background_data.shape[1]
            if len(weights) != data_dim and not (feat_dim == len(weights) and self.transposed):
                logger.warning(
                    "The number of weights specified did not match data dimension. Number of weights: {}. Number of "
                    "datapoints: {}. Weights will be ignored!".format(len(weights), data_dim))
                self.ignore_weights = True

        if self.summarise_background:  # the data has already been summarised at this point
            if background_data.ndim == 1:
                n_background_samples = 1
            else:
                n_background_samples = background_data.shape[1] if self.transposed else background_data.shape[0]
            if len(weights) != n_background_samples:
                logger.warning(
                    "The number of weights vector provided ({}) did not match the number of summary data points ({}). "
                    "The weights provided will be ignored!".format(len(weights), n_background_samples))
                self.ignore_weights = True

    # ------------------------------------------------------------------------------------------------------
    # background summarisation (kernel_shap.py:503-542); the reference delegates to shap.sample / shap.kmeans
    # ------------------------------------------------------------------------------------------------------
    def _summarise_background(self, background_data, n_background_samples: int):
        if isinstance(background_data, Data):
            logger.warning("Received option to summarise the data but the background_data object was an instance of "
                           "shap.common.Data. No summarisation will take place!")
            return background_data

        if background_data.ndim == 1:
            logger.warning(
                "Received option to summarise the data but the background_data object only had one record with {} "
                "features. No summarisation will take place!".format(len(background_data)))
            return background_data

        self.summarise_background = True

        # categorical / grouped / sparse data are subsampled; purely numeric data are clustered
        if self.use_groups or self.categorical_names or isinstance(background_data, sparse.spmatrix):
            return shap_data.sample(background_data, nsamples=n_background_samples)
        logger.info("When summarising with kmeans, the samples are weighted in proportion to their cluster occurrence "
                    "frequency. Please specify a different weighting of the samples through the by passing a weights "
                    "of len=n_background_samples to the constructor!")
        return shap_data.kmeans(background_data, n_background_samples)

    # ------------------------------------------------------------------------------------------------------
    # background -> data object (kernel_shap.py:544-671)
    # ------------------------------------------------------------------------------------------------------
    def _get_data(self, background_data, group_names, groups, weights, **kwargs):
        """Wraps the background in ``DenseData`` when grouping is on; otherwise hands the data through untouched."""
        if isinstance(background_data, Data):
            if weights is not None and self.summarise_background:
                if not self.ignore_weights:
                    background_data.weights = weights
                if self.use_groups:
                    background_data.groups = groups
                    background_data.group_names = group_names
                    background_data.group_size = len(groups)
            return background_data

        extra = (weights,) if weights is not None else ()

        if isinstance(background_data, np.ndarray):
            if self.use_groups:
                return DenseData(background_data, group_names, groups, *extra)
            return background_data

        if isinstance(background_data, sparse.spmatrix) or sparse.issparse(background_data):
            if self.use_groups:
                logger.warning("Grouping is not currently compatible with sparse matrix inputs. Converting background "
                               "data sparse array to dense matrix.")
                return DenseData(background_data.toarray(), group_names, groups, *extra)
            return background_data

        if isinstance(background_data, pd.DataFrame):
            if not self.use_groups:
                return background_data
            logger.info("Group names are specified by column headers, group_names will be ignored!")
            if kwargs.get("keep_index", False):
                return DenseDataWithIndex(background_data.values, list(background_data.columns),
                                          background_data.index.values, background_data.index.name, groups, *extra)
            return DenseData(background_data.values, list(background_data.columns), groups, *extra)

        if isinstance(background_data, pd.Series):
            if self.use_groups:
                return DenseData(background_data.values.reshape(1, len(background_data)), list(background_data.index),
                                 groups)
            return background_data

        raise TypeError("Type {} is not supported for background data!".format(type(background_data)))

    def _update_metadata(self, data_dict: dict, params: bool = False) -> None:
        """Stores ``data_dict`` in the metadata; with ``params`` only the keys listed in ``KERNEL_SHAP_PARAMS`` go into
        ``meta['params']``."""
        if params:
            for key, value in data_dict.items():
                if key in KERNEL_SHAP_PARAMS:
                    self.meta['params'].update([(key, value)])
        else:
            self.meta.update(data_dict)

    # ------------------------------------------------------------------------------------------------------
    def fit(self,  # type: ignore
            background_data,
            summarise_background: Union[bool, str] = False,
            n_background_samples: int = KERNEL_SHAP_BACKGROUND_THRESHOLD,
            group_names: Union[Tuple[str], List[str], None] = None,
            groups: Optional[List[Union[Tuple[int], List[int]]]] = None,
            weights: Union[Union[List[float], Tuple[float]], np.ndarray, None] = None,
            **kwargs) -> "KernelShap":
        """Initialises the explainer with a background dataset; parameters as in the reference (kernel_shap.py:705-742)."""
        np.random.seed(self.seed)

        self._fitted = True
        self.use_groups = groups is not None or group_names is not None

        if summarise_background:
            if isinstance(summarise_background, str):
                n_samples = background_data.data.shape[0] if isinstance(background_data, Data) \
                    else background_data.shape[0]
                n_background_samples = min(n_samples, KERNEL_SHAP_BACKGROUND_THRESHOLD)
            background_data = self._summarise_background(background_data, n_background_samples)

        self._check_inputs(background_data, group_names, groups, weights)
        if self.create_group_names:
            group_names = ['group_{}'.format(i) for i in range(len(groups))]
        if self.ignore_weights:
            weights = None
        if not self.use_groups:
            group_names, groups = None, None
        else:
            self.feature_names = group_names

        self.background_data = self._get_data(background_data, group_names, groups, weights, **kwargs)
        explainer_args = (self.predictor, self.background_data)
        # the seed travels with every replica (reference: only in a distributed context, kernel_shap.py:779; the engine keys
        # its private plan streams by it, so one GPU, a pool of GPUs and torchrun ranks all evaluate the same plans)
        explainer_kwargs = {'link': self.link, 'seed': self.seed}
        if self.plan_mode != 'shared':
            explainer_kwargs.update(plan_mode=self.plan_mode)
        if self.model_batch_rows is not None:
            explainer_kwargs.update(model_batch_rows=self.model_batch_rows)
        if self.distribute:
            self._explainer = DistributedExplainer(
                self.distributed_opts,
                KernelExplainerWrapper,
                explainer_args,
                explainer_kwargs,
            )
        else:
            self._explainer = KernelExplainerWrapper(*explainer_args, **explainer_kwargs)
        self.expected_value = self._explainer.expected_value
        if not self._explainer.vector_out:
            logger.warning("Predictor returned a scalar value. Ensure the output represents a probability or decision "
                           "score as opposed to a classification label!")

        self._update_metadata({
            'groups': groups,
            'group_names': group_names,
            'weights': weights,
            'kwargs': kwargs,
            'summarise_background': self.summarise_background,
            'grouped': self.use_groups,
            'transpose': self.transposed,
        }, params=True)

        return self

    def explain(self,
                X: Union[np.ndarray, pd.DataFrame, sparse.spmatrix],
                summarise_result: bool = False,
                cat_vars_start_idx: Sequence[int] = None,
                cat_vars_enc_dim: Sequence[int] = None,
                **kwargs) -> Explanation:
        """Explains the instances in ``X``.  ``kwargs`` (``nsamples``, ``l1_reg``, ``silent``) go to the engine untouched.

        Raises ``TypeError`` when called before ``fit`` or, in a distributed context, with a DataFrame / sparse ``X``."""
        if not self._fitted:
            raise TypeError("Called explain on an unfitted object! Please fit the explainer using the .fit method first!")

        if self.distribute and (isinstance(X, (sparse.spmatrix, pd.DataFrame)) or sparse.issparse(X)):
            raise TypeError("Incorrect type for `X` due to distributed context. Cast `X` to np.ndarray.")

        if self.use_groups and (isinstance(X, sparse.spmatrix) or sparse.issparse(X)):
            X = X.toarray()

        shap_values = self._explainer.get_explanation(X, **kwargs)
        self.expected_value = self._explainer.expected_value
        expected_value = self.expected_value
        if isinstance(shap_values, np.ndarray):  # scalar model output
            shap_values = [shap_values]
        if isinstance(expected_value, float):
            expected_value = [expected_value]

        # link(f(x)) was computed on the device by the explain call; the distributed explainer does not gather it
        getter = None if self.distribute else getattr(self._explainer, 'link_predictions', None)
        link_fx = getter() if getter is not None else None
        # ranking / category sums / arg-max of build_explanation: one small kernel pair off the phi still resident on the GPU
        device_summary = None
        summariser = None if self.distribute else getattr(self._explainer, 'summarise', None)
        if summariser is not None:
            segments = None
            if summarise_result and cat_vars_start_idx and cat_vars_enc_dim and not self.use_groups:
                segments = category_segments(shap_values[0].shape[-1], cat_vars_start_idx, cat_vars_enc_dim)
            device_summary = summariser(shap_values[0].shape[0] if shap_values[0].ndim == 2 else 1, segments=segments,
                                        want_sums=segments is not None)
        return self.build_explanation(
            X,
            shap_values,
            expected_value,
            link_predictions=link_fx,
            device_summary=device_summary,
            summarise_result=summarise_result,
            cat_vars_start_idx=cat_vars_start_idx,
            cat_vars_enc_dim=cat_vars_enc_dim,
        )

    def build_explanation(self, X, shap_values: List[np.ndarray], expected_value: List[float], **kwargs) -> Explanation:
        """Packs shap values, expected values, raw predictions and importances into an ``Explanation``."""
        cat_vars_start_idx = kwargs.get('cat_vars_start_idx', ())
        cat_vars_enc_dim = kwargs.get('cat_vars_enc_dim', ())
        summarise_result = kwargs.get('summarise_result', False)
        if summarise_result:
            self._check_result_summarisation(summarise_result, cat_vars_start_idx, cat_vars_enc_dim)
        device_summary = kwargs.get('device_summary')
        if self.summarise_result:
            if device_summary is not None and device_summary.get('phi_sum') is not None:
                shap_values = [device_summary['phi_sum'][c] for c in range(len(shap_values))]
            else:
                device_summary = None                  # computed on unsummed groups: not what is being reported
                shap_values = [sum_categories(arr, cat_vars_start_idx, cat_vars_enc_dim) for arr in shap_values]
        elif device_summary is not None and device_summary['mean_abs'].shape[1] != np.atleast_2d(shap_values[0]).shape[1]:
            device_summary = None

        # raw predictions on the scale the explainer works in (the reference wraps link.f in np.vectorize, an
        # interpreted per-element loop; both links are NumPy ufunc expressions, so they are applied to the array)
        raw_predictions = kwargs.get('link_predictions')
        if raw_predictions is None:
            # a module takes device tensors, not the NumPy rows a callable predictor takes: the explainer runs it
            predict = self._explainer.predict if is_torch_module(self.predictor) else self.predictor
            raw_predictions = convert_to_link(self.link).f(np.asarray(predict(X), dtype=np.float64))

        if device_summary is not None and len(shap_values) + 1 == device_summary['mean_abs'].shape[0]:
            argmax_pred = device_summary['argmax'] if self.task != 'regression' else []
            importances = importances_from_device(device_summary, self.feature_names)
        else:
            argmax_pred = np.argmax(np.atleast_2d(raw_predictions), axis=1) if self.task != 'regression' else []
            importances = rank_by_importance(shap_values, feature_names=self.feature_names)

        X = X.toarray() if (isinstance(X, sparse.spmatrix) or sparse.issparse(X)) else np.array(X)

        data = {key: (dict(value) if isinstance(value, dict) else copy.copy(value))      # fresh containers, two levels deep
                for key, value in DEFAULT_DATA_KERNEL_SHAP.items()}
        data['raw']['importances'] = {}
        data.update(
            shap_values=shap_values,
            expected_value=np.array(expected_value),
            link=self.link,
            categorical_names=self.categorical_names,
            feature_names=self.feature_names,
        )
        data['raw'].update(
            raw_prediction=raw_predictions,
            prediction=argmax_pred,
            instances=X,
            importances=importances,
        )
        self._update_metadata({"summarise_result": self.summarise_result}, params=True)

        return Explanation(meta=copy.deepcopy(self.meta), data=data)

    def _check_result_summarisation(self, summarise_result: bool, cat_vars_start_idx: Sequence[int],
                                    cat_vars_enc_dim: Sequence[int]) -> None:
        """Result summarisation needs both index sequences and is pointless when groups were used at fit time."""
        self.summarise_result = summarise_result
        if not summarise_result:
            return
        if not cat_vars_start_idx or not cat_vars_enc_dim:
            logger.warning("Results cannot be summarised as either the start indices for categorical variables or the "
                           "encoding dimensions were not passed!")
            self.summarise_result = False
        elif self.use_groups:
            logger.warning("Specified both groups as well as summarisation for categorical variables. By grouping, "
                           "only one shap value is estimated for each categorical variable. Summarisation is not "
                           "necessary!")
            self.summarise_result = False
