/*
 * dks.h -- C ABI of the H100-native KernelSHAP engine (libdks.so).
 *
 * The reference (alexcoca/DistributedKernelShap) has no FFI: its hot path is reached through a Python
 * duck-typed slot, `KernelShap._explainer` (explainers/kernel_shap.py:774-788), whose object must offer
 * `get_explanation(X, **kw)`, `.expected_value`, `.vector_out` (kernel_shap.py:789-790, :880-887).  The
 * object the reference puts there is `KernelExplainerWrapper` (kernel_shap.py:217-261), a subclass of
 * `shap.KernelExplainer` (shap==0.35.0, not vendored).  Each entry point below replaces one piece of
 * that object; the Python binding a maintainer adds is in INTEGRATION.md.
 *
 * Conventions: every function returns 0 on success or a DKS_ERR_* code; dks_last_error() returns the
 * message of the calling thread's last failure.  Plain pointers and sizes only -- no torch types.  A ctx
 * is bound to one CUDA device, owns only its workspace, and is not thread-safe.  `*_dev` pointers are
 * device memory owned by the caller (e.g. torch tensors); `*_host` pointers are host memory.  Work is
 * enqueued on the ctx stream (dks_set_stream) and is asynchronous unless the function says it
 * synchronises.  float64 at the boundary, like the reference.
 */
#ifndef DKS_H_
#define DKS_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DKS_VERSION 100

/* error codes */
#define DKS_OK 0
#define DKS_ERR_INVALID 1       /* bad argument / call order */
#define DKS_ERR_CUDA 2          /* a CUDA runtime call failed (message has the CUDA error string) */
#define DKS_ERR_UNSUPPORTED 3   /* valid request the engine does not implement (never a silent fallback) */
#define DKS_ERR_PLAN_MISSING 4  /* an instance needs a coalition plan for an M that was not provided */
#define DKS_ERR_NUMERIC 5       /* normal matrix not positive definite; exp head: a model output that is not finite */
#define DKS_ERR_DOMAIN 6        /* column maps: a raw value a map refuses (NaN or an unseen category under the policy
                                 * "error"); the detail is the instance (or background row) index */

/* model head applied to the linear scores z = W x + b   (replaces the opaque `predictor` callable,
 * benchmarks/ray_pool.py:34; sklearn LogisticRegression.predict_proba per scripts/fit_adult_model.py:27) */
#define DKS_ACT_IDENTITY 0      /* outputs = z (R outputs): regression / decision_function           */
#define DKS_ACT_BINARY_LOGISTIC 1 /* R = 1, outputs [1 - s, s], s = sigmoid(kappa * z): kappa = 1 is the
                                   * binary sigmoid, kappa = 2 the 2-class multinomial softmax([-z, z]) */
#define DKS_ACT_SOFTMAX 2       /* R = C >= 2 scores, outputs softmax(z)                              */
#define DKS_ACT_OVR 3           /* R = C in 3..8 scores, one-vs-rest: s_c = sigmoid(z_c), outputs s_c / sum_c' s_c'
                                 * (scikit-learn's _predict_proba_lr: liblinear / multi_class='ovr' LogisticRegression,
                                 * OneVsRestClassifier over binary linear models); kappa must be 1 */
#define DKS_ACT_EXP 4           /* R = 1 score, output exp(z): the log-link GLM regressors (scikit-learn's PoissonRegressor,
                                 * GammaRegressor, TweedieRegressor with a log link).  Link DKS_LINK_IDENTITY only (dks_fit
                                 * refuses the logit link: a predicted mean above 1 has no logit).  dks_fit refuses a
                                 * background whose prediction is not finite in float64; an instance whose f(x) or whose
                                 * ey(s) = sum_j w_j exp(z(s, j)) is not finite is reported as DKS_ERR_NUMERIC and nothing
                                 * non-finite is written into phi.  Shared plans with every group varying (G <= 128): y(s) =
                                 * exp(a(s) + l(s)) - fnull in float64, a(s) from the instance's nibble tables and l(s) =
                                 * ln sum_j w_j exp(d(s, j)) computed once per plan (DKS_SHARED_EXP); the CUDA-core kernels
                                 * sum 2^t over the background in fp32 and send rows outside their range rule to float64
                                 * (DESIGN.md §5.0.8); no tensor-core kernel */
#define DKS_ACT_MIX 5           /* mixture: outputs sum_k pi_k h(z_k) over K >= 2 members that share one member head h
                                 * (binary-logistic, outputs [1 - p, p]; softmax or one-vs-rest over 3..8 classes), z_k = W_k x
                                 * + b_k.  scikit-learn's CalibratedClassifierCV(method='sigmoid'), soft-voting and bagging
                                 * ensembles of linear classifiers.  Set by dks_set_mixture only (dks_set_model refuses it).
                                 * Shared plans with every group varying (G <= 128): one pass of the member head's
                                 * coalition kernel per member, each member's sums added times pi_k into one set of sums,
                                 * then the member head's solves and l1 selection (DKS_SHARED_MIX).  The rest (partial
                                 * varying sets, per-instance or caller-supplied plans, kernel 'simt'; up to 64 groups): a
                                 * CUDA-core kernel evaluating every member's head per element.  More than 128 groups, the
                                 * tensor-core kernel and per-instance plans of 65..128 groups are DKS_ERR_UNSUPPORTED
                                 * (DESIGN.md §5.0.10) */
#define DKS_ACT_TREES 6         /* tree ensemble: set by dks_set_tree_model only (dks_set_model refuses it) */

/* head of a tree ensemble on its raw scores r = base + sum_t leaf_t(x) (dks_set_tree_model) */
#define DKS_TREE_HEAD_IDENTITY 0 /* outputs r (R outputs): forests' mean class fractions or values, decision_function, predict */
#define DKS_TREE_HEAD_SIGMOID 1  /* R = 1, outputs [1 - expit(r), expit(r)]: binary gradient boosting predict_proba */
#define DKS_TREE_HEAD_SOFTMAX 2  /* R = K >= 2 raw scores, outputs softmax(r): multi-class gradient boosting */
#define DKS_TREE_HEAD_EXP 3      /* R = 1, output exp(r): histogram gradient boosting with a log-link loss; link identity only */
#define DKS_TREE_HEAD_IFOREST 4  /* R = 1, output -2^r - offset (dks_set_tree_offset): IsolationForest score_samples /
                                  * decision_function with -1 / (n_trees c(max_samples)) folded into the leaves; link
                                  * identity only */
/* split comparison: x goes left when x <= threshold */
#define DKS_TREE_CMP_F32 0       /* (double)(float)x <= threshold: scikit-learn's sklearn.tree casts X to float32 */
#define DKS_TREE_CMP_F64 1       /* x <= threshold in float64: the histogram gradient boosting estimators */
/* ops of a column encoding (dks_set_column_encoding): each maps the float64 value v of one encoded column, in program order,
 * rounding as scikit-learn's numpy arithmetic does (no fused multiply-add) */
#define DKS_ENC_OP_SUB 0         /* v - c0 (StandardScaler, RobustScaler centring) */
#define DKS_ENC_OP_DIV 1         /* v / c0 (StandardScaler, RobustScaler, MaxAbsScaler scaling) */
#define DKS_ENC_OP_MUL 2         /* v * c0 (MinMaxScaler) */
#define DKS_ENC_OP_ADD 3         /* v + c0 (MinMaxScaler) */
#define DKS_ENC_OP_CLIP 4        /* np.clip(v, c0, c1): NaN stays NaN (MinMaxScaler(clip=True)) */
#define DKS_ENC_OP_NANFILL 5     /* c0 where v is NaN (SimpleImputer) */
#define DKS_ENC_OP_ISNAN 6       /* 1 where v is NaN, else 0 (SimpleImputer's missing indicator) */
#define DKS_ENC_OP_PIECES 7      /* m sorted edges: output of bin numpy.searchsorted(edges, v, side='right') (KBinsDiscretizer) */
#define DKS_ENC_OP_TABLE 8       /* m sorted keys: output of the exactly equal key, else the unknown output (encoders) */
#define DKS_ENC_NAN_ERROR 2      /* op flag (PIECES, TABLE): a NaN is refused */
#define DKS_ENC_UNKNOWN_ERROR 4  /* op flag (TABLE): a value matching no key is refused */
#define DKS_ACT_KMACH 7        /* kernel machine: set by dks_set_kernel_machine only (dks_set_model refuses it) */

/* kernel of a kernel machine (dks_set_kernel_machine): K(x, v) = phi(t), t = sum_c h(x_c, v_c) with the member's column
 * weight w_c and origin o_c (its scalers folded in) */
#define DKS_KM_KERNEL_RBF 0       /* h = w_c (x_c - v_c)^2,         phi = exp(-gamma t) */
#define DKS_KM_KERNEL_LAPLACIAN 1 /* h = w_c |x_c - v_c|,           phi = exp(-gamma t) */
#define DKS_KM_KERNEL_POLY 2      /* h = w_c (x_c - o_c)(v_c - o_c), phi = (gamma t + coef0)^degree, integer degree >= 0 */
#define DKS_KM_KERNEL_SIGMOID 3   /* h = w_c (x_c - o_c)(v_c - o_c), phi = tanh(gamma t + coef0) */
#define DKS_KM_KERNEL_PROGRAM 4   /* up to DKS_KM_MAX_STATS statistics and an expression over them (dks_set_kernel_program):
                                   * scikit-learn's kernel algebra (GaussianProcessRegressor, KernelRidge with a Kernel) */
/* statistic of the program kernel: t_l = sum_c h(x_c, v_c) with the statistic's own column weights w and origins o */
#define DKS_KM_STAT_SQDIST 0      /* h = w_c (x_c - v_c)^2 */
#define DKS_KM_STAT_DOT 1         /* h = w_c (x_c - o_c)(v_c - o_c) */
/* instructions of the program kernel's postfix expression {op, arg, a, b}; leaves push, operators pop */
#define DKS_KM_OP_CONST 0         /* push a */
#define DKS_KM_OP_STAT 1          /* push t_arg */
#define DKS_KM_OP_EXP 2           /* push exp(-a t_arg) (RBF, Matern nu = inf: a = 1/2) */
#define DKS_KM_OP_MATERN05 3      /* push exp(-r), r = sqrt(max(t_arg, 0)) */
#define DKS_KM_OP_MATERN15 4      /* push (1 + k) exp(-k), k = sqrt(3) r */
#define DKS_KM_OP_MATERN25 5      /* push (1 + k + k^2 / 3) exp(-k), k = sqrt(5) r */
#define DKS_KM_OP_RQ 6            /* push (1 + t_arg)^a (RationalQuadratic: a = -alpha) */
#define DKS_KM_OP_EXPSINE 7       /* push exp(-2 (sin(pi r / a) / b)^2) (ExpSineSquared: a periodicity, b length scale) */
#define DKS_KM_OP_ADD 8           /* pop two, push their sum */
#define DKS_KM_OP_MUL 9           /* pop two, push their product */
#define DKS_KM_OP_POW 10          /* top = top^a */
#define DKS_KM_OP_ADDC 11         /* top = top + a */
#define DKS_KM_OP_MULC 12         /* top = top * a */
#define DKS_KM_MAX_STATS 4        /* statistics of the program kernel */
#define DKS_KM_MAX_OPS 32         /* instructions of the program kernel */
#define DKS_KM_MAX_STACK 4        /* operands the program kernel's expression holds at once */
/* head of a kernel machine on the member scores f_k = sum_v dual[v] K(x, v) + intercept_k */
#define DKS_KM_HEAD_IDENTITY 0    /* one member, R outputs f (SVC / NuSVC decision_function, SVR, NuSVR, KernelRidge) */
#define DKS_KM_HEAD_CALIBRATED 1  /* R = 1, outputs [1 - p1, p1], p1 = sum_k pi_k expit(-(a_k f_k + b_k)): sigmoid
                                   * CalibratedClassifierCV over a binary SVC / NuSVC */
#define DKS_KM_HEAD_OVO 2         /* multi-class SVC / NuSVC (dks_set_svc_multiclass): one-vs-one pair scores per member */
#define DKS_KM_MAX_R 8            /* outputs of the identity head */
#define DKS_KM_MAX_K 16           /* members of the calibrated head */
/* output mode of the one-vs-one head (dks_set_svc_multiclass) */
#define DKS_KM_OVO_DECISION 0     /* P = K (K - 1) / 2 pair values dec_k (decision_function_shape='ovo'), one member */
#define DKS_KM_OVO_PROBA 1        /* K probabilities: per member the ovr-vote decision function, sigmoid-calibrated per
                                   * class and normalised; members averaged with weights pi (CalibratedClassifierCV) */
#define DKS_KM_OVO_MAX_CLASSES 8  /* classes of the one-vs-one head (28 pairs) */
#define DKS_ACT_MLP 8          /* multi-layer perceptron: set by dks_set_mlp only (dks_set_model refuses it) */

/* hidden activation of a multi-layer perceptron (dks_set_mlp), scikit-learn's ACTIVATIONS */
#define DKS_MLP_ACT_IDENTITY 0    /* h = a */
#define DKS_MLP_ACT_LOGISTIC 1    /* h = 1 / (1 + exp(-a)) */
#define DKS_MLP_ACT_TANH 2        /* h = tanh(a) */
#define DKS_MLP_ACT_RELU 3        /* h = max(a, 0) */
/* output head of a multi-layer perceptron on the output layer's values z [R] */
#define DKS_MLP_HEAD_IDENTITY 0   /* outputs z (MLPRegressor.predict, R <= 8) */
#define DKS_MLP_HEAD_SIGMOID 1    /* R = 1, outputs [1 - expit(z), expit(z)] (binary MLPClassifier.predict_proba) */
#define DKS_MLP_HEAD_SOFTMAX 2    /* R = 2..8, outputs softmax(z) (multi-class MLPClassifier.predict_proba) */
#define DKS_MLP_MAX_HIDDEN 4      /* hidden layers */
#define DKS_MLP_MAX_WIDTH 256     /* units per hidden layer */
#define DKS_MLP_MAX_OUT 8         /* output units */
#define DKS_ACT_KNN 9          /* k-nearest neighbours: set by dks_set_knn_model only (dks_set_model refuses it) */

/* distance of a nearest-neighbour model (dks_set_knn_model): t = sum_c h(d_c) over the columns in order,
 * d_c = (colw_c x_c + colo_c) - v_c for training row v */
#define DKS_KNN_METRIC_EUCLIDEAN 0   /* h = d^2,   distance sqrt(t) */
#define DKS_KNN_METRIC_MANHATTAN 1   /* h = |d|,   distance t */
#define DKS_KNN_METRIC_MINKOWSKI 2   /* h = |d|^p, distance t^(1/p), finite p >= 1 */
#define DKS_KNN_METRIC_SQEUCLIDEAN 3 /* h = d^2,   distance t */
/* neighbour weights */
#define DKS_KNN_WEIGHTS_UNIFORM 0    /* 1 */
#define DKS_KNN_WEIGHTS_DISTANCE 1   /* 1 / distance; neighbours at distance 0 take 1 and the others 0 */
/* output head */
#define DKS_KNN_HEAD_CLASSIFY 0      /* R classes, outputs the per-class weight sums over their total (predict_proba) */
#define DKS_KNN_HEAD_REGRESS 1       /* R targets, outputs the weighted mean of the neighbours' targets (predict) */
#define DKS_KNN_MAX_K 32             /* neighbours */
#define DKS_KNN_MAX_R 8              /* classes or targets */
#define DKS_ACT_ENSEMBLE 10    /* soft-voting ensemble of the four families above: set by dks_set_ensemble only */
#define DKS_ENS_MAX_MEMBERS 16       /* members of a soft-voting ensemble */
#define DKS_ENS_MAX_OUT 8            /* its outputs */
#define DKS_ACT_EXTERNAL 11    /* a model the caller evaluates (a torch.nn.Module on the device): set by dks_set_external_model
                                * only, explained stepwise by dks_external_* */
#define DKS_EXTERNAL_FLOAT32 0       /* dtypes of the module's input rows and outputs */
#define DKS_EXTERNAL_FLOAT64 1
#define DKS_ACT_STACKING 12    /* stacking ensemble of the four families above: set by dks_set_stacking only */
#define DKS_STACK_MAX_F 128          /* meta columns the final estimator reads: DKS_ENS_MAX_MEMBERS x DKS_ENS_MAX_OUT */
/* head of a stacking ensemble's final estimator on its R scores r = W m + b (+ W_pass x) (dks_set_stacking) */
#define DKS_STACK_HEAD_IDENTITY 0    /* outputs r (C = R): decision_function, a linear regressor's predict */
#define DKS_STACK_HEAD_SIGMOID 1     /* R = 1, outputs [1 - expit(r), expit(r)] (C = 2): binary logistic predict_proba */
#define DKS_STACK_HEAD_SOFTMAX 2     /* R = C >= 2, outputs softmax(r): multinomial logistic predict_proba */
#define DKS_ACT_GAUSS 13       /* Gaussian generative model: set by dks_set_gaussian_model only */
/* head of a Gaussian generative model over its K component scores l_k (dks_set_gaussian_model) */
#define DKS_GAUSS_HEAD_SOFTMAX 0     /* K outputs softmax(l): QDA, GaussianNB, Gaussian mixtures predict_proba */
#define DKS_GAUSS_HEAD_LOGSUMEXP 1   /* one output log sum_k exp(l_k): Gaussian mixtures score_samples */
#define DKS_GAUSS_HEAD_IDENTITY 2    /* K outputs l: multi-class QDA decision_function, EllipticEnvelope (K = 1) */
#define DKS_GAUSS_HEAD_DIFF 3        /* K = 2, one output l_1 - l_0: binary QDA decision_function */
#define DKS_GAUSS_MAX_K 8            /* components or classes */

/* link (shap.common.convert_to_link; reference call sites kernel_shap.py:775, :949) */
#define DKS_LINK_IDENTITY 0
#define DKS_LINK_LOGIT 1

/* which fused kernel evaluates the coalitions */
#define DKS_KERNEL_AUTO 0
#define DKS_KERNEL_SIMT 1       /* CUDA-core kernel (all shapes) */
#define DKS_KERNEL_TCGEN05 2    /* tensor-core kernel: Z tile x background tile on wgmma (the name is historical) */
#define DKS_KERNEL_SHARED 3     /* shared-plan fast path for instances whose groups all vary (+ best general kernel
                                 * for the rest); DKS_KERNEL_AUTO picks it whenever it applies */

typedef struct dks_ctx dks_ctx;

int dks_version(void);
const char* dks_last_error(void);
/* number of CUDA devices visible to the process (0 when there is none; never an error) */
int dks_device_count(int* count);

/* ---- lifetime ------------------------------------------------------------------------------------
 * replaces KernelExplainerWrapper.__init__ (kernel_shap.py:225-229): one ctx per actor/GPU. */
int dks_create(dks_ctx** out, int device);
int dks_destroy(dks_ctx* ctx);
/* `stream` is a cudaStream_t (0 = legacy default stream).  The ctx creates its own stream by default. */
int dks_set_stream(dks_ctx* ctx, void* stream);
int dks_synchronize(dks_ctx* ctx);

/* ---- fit: shap.common.DenseData + KernelExplainer.__init__ (reached from kernel_shap.py:229) --------
 * background [N x D] row-major float64, optional weights [N] (NULL = uniform; normalised to sum 1). */
int dks_set_background(dks_ctx* ctx, const double* bg_host, int N, int D, const double* weights_host);
/* feature groups in CSR form: group g owns columns group_cols[group_offsets[g] .. group_offsets[g+1]).
 * Every column must belong to exactly one group (DenseData asserts the sizes add up to D). */
int dks_set_groups(dks_ctx* ctx, const int32_t* group_offsets, const int32_t* group_cols, int G);
/* linear scores z = W x + b with W [R x D] row-major, b [R]; head per DKS_ACT_*; kappa used by
 * DKS_ACT_BINARY_LOGISTIC (DKS_ACT_OVR requires kappa == 1 and R >= 3, DKS_ACT_EXP R == 1).  scalar_out != 0 marks a predictor returning a
 * 1-D array (vector_out False). */
int dks_set_model(dks_ctx* ctx, const double* W_host, const double* b_host, int R, int activation, double kappa,
                  int scalar_out);
/* mixture head (DKS_ACT_MIX) in place of dks_set_model: K >= 2 members with the member head member_act (DKS_ACT_BINARY_LOGISTIC
 * with R_m = 1 and kappa 1 -- fold kappa into W and b --, DKS_ACT_SOFTMAX or DKS_ACT_OVR with R_m = 3..8), K R_m <= 32 score
 * rows.  W_host [K R_m x D] and b_host [K R_m], member-major (row k R_m + q is row q of member k); pi_host [K] positive
 * finite weights, normalised to sum 1.  Outputs: 2 for binary members, R_m otherwise.  dks_set_column_maps may follow with
 * R = K R_m. */
int dks_set_mixture(dks_ctx* ctx, int K, int member_act, int R_m, const double* W_host, const double* b_host,
                    const double* pi_host, int scalar_out);
/* tree ensemble (DKS_ACT_TREES) in place of dks_set_model: n_trees trees whose nodes are concatenated into n_nodes entries.
 * Per node: feature (the split column, -1 at a leaf), threshold, left / right (global indices of the children, each larger
 * than the node's own; ignored at a leaf), missing_left (1: NaN goes left); value [n_nodes][R] row-major, read at leaves: the
 * leaf's contribution to the R raw scores (the learning rate or 1 / n_trees folded in).  roots [n_trees]; base [R].
 * r = base + sum over trees of the value of the leaf x reaches; outputs = head(r) per DKS_TREE_HEAD_*, compared per
 * DKS_TREE_CMP_*.  R <= 8 and at most 8 outputs.  Malformed arrays (a child not after its parent, a feature out of range, a
 * NaN threshold, a non-finite leaf value) are DKS_ERR_UNSUPPORTED.
 * The models read this way (DESIGN.md §5.0.11, §5.0.18): decision trees, random / extra-trees forests (identity head over
 * the mean class fractions or values), gradient boosting and histogram gradient boosting (identity, sigmoid, softmax or exp
 * head on the raw scores), SAMME AdaBoostClassifier over sklearn.tree classifiers (each leaf holds its tree's weighted class
 * vote, 1 / sum of the weights and, for predict_proba, 1 / (K - 1) folded in: identity, sigmoid or softmax head) and
 * IsolationForest (each leaf holds -(depth + c(n_node_samples) - 1) / (n_trees c(max_samples)): the anomaly head).
 * Every instance runs the tree kernels (DKS_GENERAL_TREES, DESIGN.md §5.0.11), up to 64 groups: shared plans (full and partial
 * varying sets), per-instance device plans and caller-supplied plans, kernel 'auto' or 'simt' (tcgen05 / shared are
 * DKS_ERR_UNSUPPORTED), l1 selection through the general list's LARS route.  Float64 throughout; a link(ey) or link(f(x)) that
 * is not finite (the logit of a probability of exactly 0 or 1) is DKS_ERR_NUMERIC, nothing non-finite is written into phi.
 * A forest whose per-instance buffers do not fit shared memory is DKS_ERR_UNSUPPORTED.  With a column encoding set
 * (dks_set_column_encoding) the split features index the E encoded columns, not the D raw ones. */
int dks_set_tree_model(dks_ctx* ctx, int n_nodes, const int32_t* feature, const double* threshold, const int32_t* left,
                       const int32_t* right, const uint8_t* missing_left, const double* value, int R, int n_trees,
                       const int32_t* roots, const double* base, int head, int cmp, int scalar_out);
/* the offset the anomaly head (DKS_TREE_HEAD_IFOREST) subtracts: IsolationForest.offset_ for decision_function, 0 for
 * score_samples.  Call after dks_set_tree_model, which sets it to 0, and before dks_fit.  A context whose model is not a tree
 * ensemble with the anomaly head is DKS_ERR_INVALID; a non-finite offset is DKS_ERR_UNSUPPORTED. */
int dks_set_tree_offset(dks_ctx* ctx, double offset);
/* kernel machine (DKS_ACT_KMACH) in place of dks_set_model: K members, member k owning support vectors sv_off[k] ..
 * sv_off[k + 1] (sv_off [K + 1], non-decreasing from 0, n_sv = sv_off[K] >= 1).  sv [n_sv][D] row-major in raw feature space,
 * dual [n_sv][R], intercept [K][R]; per member colw [K][D] (> 0 at every column), colo [K][D] and gamma [K] (>= 0);
 * kernel DKS_KM_KERNEL_*, degree (POLY: an integer >= 0) and coef0 shared by the members.  Member score
 * f_k = sum_v dual[v] phi(sum_c h(x_c, sv[v][c])) + intercept_k; outputs per DKS_KM_HEAD_*: IDENTITY needs K = 1 and gives
 * R <= 8 outputs; CALIBRATED needs R = 1 and reads cal_a, cal_b and pi [K] (pi > 0, normalised to sum 1), K <= 16.
 * Non-finite values, bad offsets and unknown kernel or head codes are DKS_ERR_UNSUPPORTED.
 * Every instance runs the kernel-machine kernel (DKS_GENERAL_KMACH, DESIGN.md §5.0.12), up to 64 groups: shared plans (full
 * and partial varying sets), per-instance device plans and caller-supplied plans, kernel 'auto' or 'simt' (tcgen05 / shared
 * are DKS_ERR_UNSUPPORTED), l1 selection through the general list's LARS route.  Float64 throughout.  NaN in a background
 * row (dks_fit) or an instance (dks_predict_host, the explain calls) is DKS_ERR_DOMAIN with the row; a link(ey) or
 * link(f(x)) that is not finite is DKS_ERR_NUMERIC and nothing non-finite is written into phi.  Shapes whose per-instance
 * buffers do not fit shared memory are DKS_ERR_UNSUPPORTED.  dks_set_column_maps is refused.  With a column encoding set
 * (dks_set_column_encoding) D is its E encoded columns.  kernel DKS_KM_KERNEL_PROGRAM needs K = 1, the identity head and
 * dks_set_kernel_program before dks_fit (which is DKS_ERR_INVALID without it); gamma, degree, coef0, colw and colo are then
 * unused (colw must still be positive). */
int dks_set_kernel_machine(dks_ctx* ctx, int K, const int32_t* sv_off, const double* sv, const double* dual, int R,
                           const double* intercept, const double* colw, const double* colo, const double* gamma, int kernel,
                           double degree, double coef0, int head, const double* cal_a, const double* cal_b,
                           const double* pi, int scalar_out);
/* the program kernel (DESIGN.md §5.0.21) of a kernel machine set with DKS_KM_KERNEL_PROGRAM: K(x, v) is a postfix expression
 * of n_ops (1..DKS_KM_MAX_OPS) instructions ops / args / a / b (DKS_KM_OP_*) over L (1..DKS_KM_MAX_STATS) statistics
 * t_l = sum_c h_l(x_c, v_c) of kind kinds[l] (DKS_KM_STAT_*) with column weights colw [L][D] (> 0) and origins colo [L][D].
 * Leaves read statistic args[i] < L; the expression must leave exactly one value and hold at most DKS_KM_MAX_STACK at once.
 * Unknown codes, out-of-range operands, a stack that under- or overflows, non-finite or zero-divisor constants are
 * DKS_ERR_UNSUPPORTED; a context without a DKS_KM_KERNEL_PROGRAM kernel machine is DKS_ERR_INVALID.  Call before dks_fit.
 * The explain kernel holds the tables of every statistic for 32 / L support vectors per tile, in the shared memory the
 * other kernels use for 32: one masked row costs L ceil(M / 4) table reads and one expression per support vector. */
int dks_set_kernel_program(dks_ctx* ctx, int L, const int32_t* kinds, const double* colw, const double* colo, int n_ops,
                           const int32_t* ops, const int32_t* args, const double* a, const double* b);
/* multi-class SVC / NuSVC (DKS_ACT_KMACH, head DKS_KM_HEAD_OVO, DESIGN.md §5.0.22) in place of dks_set_model: K members
 * (1..DKS_KM_MAX_K calibration folds, or one SVM) over `classes` (3..DKS_KM_OVO_MAX_CLASSES) classes.  Member m owns support
 * vectors sv_off[m] .. sv_off[m + 1] (sv_off [K + 1], non-decreasing from 0, n_sv = sv_off[K] >= 1), stored in class blocks:
 * class c of member m owns cls_off[m (classes + 1) + c] .. cls_off[m (classes + 1) + c + 1] (absolute rows, from sv_off[m]
 * to sv_off[m + 1], non-decreasing; a class may own none).  sv [n_sv][D] in raw feature space, dual [n_sv][classes - 1]
 * (scikit-learn's dual_coef_ transposed), intercept [K][P] with P = classes (classes - 1) / 2; colw [K][D] (> 0), colo [K][D],
 * gamma [K] (>= 0), kernel DKS_KM_KERNEL_RBF / _POLY / _SIGMOID, degree and coef0 as for dks_set_kernel_machine.  Pair
 * k = (i, j), i < j, in the order i, then j:
 *   dec_k = sum_{v in class i} dual[v][j - 1] K(x, v) + sum_{v in class j} dual[v][i] K(x, v) + intercept[m][k].
 * mode DKS_KM_OVO_DECISION: one member, P <= 8 outputs dec (decision_function_shape='ovo').  mode DKS_KM_OVO_PROBA:
 * `classes` outputs sum_m pi_m p_m (pi > 0, normalised to sum 1), p_m,c = e_c / sum e, e_c = expit(-(a f_c + b)) with
 * a = cal_a[m][c], b = cal_b[m][c] [K][classes] and f the ovr-vote decision function votes_c + conf_c / (3 (|conf_c| + 1))
 * (dec_k >= 0 votes for i, else for j; conf_i += dec_k, conf_j -= dec_k); a zero sum gives 1 / classes, and values in
 * (1, 1 + 1e-5] become 1.  The device sums support vectors in its own fixed order, so a dec_k within rounding of 0 may vote
 * otherwise than libsvm.  Non-finite values, bad offsets, unknown kernel or mode codes and out-of-range counts are
 * DKS_ERR_UNSUPPORTED.  Everything else -- plans, groups, l1, NaN refusals, column encodings, ensembles -- is as for
 * dks_set_kernel_machine; shapes whose per-instance buffers do not fit shared memory are DKS_ERR_UNSUPPORTED. */
int dks_set_svc_multiclass(dks_ctx* ctx, int K, int classes, const int32_t* sv_off, const int32_t* cls_off, const double* sv,
                           const double* dual, const double* intercept, const double* colw, const double* colo,
                           const double* gamma, int kernel, double degree, double coef0, int mode, const double* cal_a,
                           const double* cal_b, const double* pi, int scalar_out);
/* multi-layer perceptron (DKS_ACT_MLP) in place of dks_set_model: n_hidden (1..DKS_MLP_MAX_HIDDEN) hidden layers.
 * widths [n_hidden + 2] = {D, H_1 .. H_n_hidden, R}: hidden widths 1..DKS_MLP_MAX_WIDTH, R outputs 1..DKS_MLP_MAX_OUT.
 * W_host: the layers' weights concatenated, layer l [widths[l]][widths[l + 1]] row-major (scikit-learn's coefs_[l]; layer 0
 * reads raw feature space, per-column scalers folded in); b_host: the biases concatenated, layer l [widths[l + 1]].
 * a_l = act(a_{l-1} W_l + b_l) for the hidden layers (activation DKS_MLP_ACT_*), z = a_n W + b for the output layer, outputs
 * per DKS_MLP_HEAD_*.  Non-finite weights, bad widths and unknown codes are DKS_ERR_UNSUPPORTED.
 * Every instance runs the MLP kernel (DKS_GENERAL_MLP, DESIGN.md §5.0.14), up to 64 groups: shared plans (full and partial
 * varying sets), per-instance device plans and caller-supplied plans, kernel 'auto' or 'simt' (tcgen05 / shared are
 * DKS_ERR_UNSUPPORTED), l1 selection through the general list's LARS route.  Float64 throughout, every product on the FP64
 * tensor cores.  NaN or an infinity in a background row (dks_fit) or an instance (dks_predict_host, the explain calls) is
 * DKS_ERR_DOMAIN with the row; a link(ey) or link(f(x)) that is not finite is DKS_ERR_NUMERIC and nothing non-finite is
 * written into phi.  Shapes whose per-instance buffers do not fit shared memory are DKS_ERR_UNSUPPORTED.
 * dks_set_column_maps is refused.  With a column encoding set (dks_set_column_encoding) widths[0] is its E encoded columns. */
int dks_set_mlp(dks_ctx* ctx, int n_hidden, const int32_t* widths, const double* W_host, const double* b_host, int activation,
                int head, int scalar_out);
/* k-nearest-neighbour model (DKS_ACT_KNN) in place of dks_set_model: n_fit >= k training rows fitX [n_fit][D] row-major in
 * the space the model was fitted in; a row x is read as x'_c = colw_c x_c + colo_c (colw [D] non-zero, colo [D]: per-column
 * scalers folded in).  k neighbours (1..DKS_KNN_MAX_K), metric DKS_KNN_METRIC_* (p: the Minkowski exponent, read for
 * DKS_KNN_METRIC_MINKOWSKI), weights DKS_KNN_WEIGHTS_*.  head DKS_KNN_HEAD_CLASSIFY: R = 2..8 classes and
 * labels_or_targets [n_fit] holds each row's class index 0..R-1; DKS_KNN_HEAD_REGRESS: R = 1..8 targets, labels_or_targets
 * [n_fit][R].  The neighbours are the first k training rows ranked by (t, row index): of equidistant rows the lower index
 * wins.  A row equal to a training row column for column (x'_c == v_c exactly) is at distance exactly 0 whatever the
 * rounding of t; other distances are clamped at 0.  Non-finite arrays, bad sizes and unknown codes are
 * DKS_ERR_UNSUPPORTED.
 * Every instance runs the neighbour kernel (DKS_GENERAL_KNN, DESIGN.md §5.0.15), up to 64 groups: shared plans (full and
 * partial varying sets), per-instance device plans and caller-supplied plans, kernel 'auto' or 'simt' (tcgen05 / shared are
 * DKS_ERR_UNSUPPORTED), l1 selection through the general list's LARS route; every output is solved on its own.  Float64
 * throughout.  NaN or an infinity in a background row (dks_fit) or an instance (dks_predict_host, the explain calls) is
 * DKS_ERR_DOMAIN with the row; a link(ey) or link(f(x)) that is not finite (the logit of a probability of exactly 0 or 1) is
 * DKS_ERR_NUMERIC and nothing non-finite is written into phi.  Shapes whose per-instance buffers do not fit shared memory
 * are DKS_ERR_UNSUPPORTED.  dks_set_column_maps is refused.  With a column encoding set (dks_set_column_encoding) D is its E
 * encoded columns. */
int dks_set_knn_model(dks_ctx* ctx, int n_fit, const double* fitX, const double* colw, const double* colo, int k, int metric,
                      double p, int weights, int R, const double* labels_or_targets, int head, int scalar_out);
/* Gaussian generative model (DKS_ACT_GAUSS) in place of dks_set_model: K (1..DKS_GAUSS_MAX_K) component scores
 *   l_k(x) = c_k - gamma_k ||L_k^T (x - mu_k)||^2
 * over D columns (the model's width: the E encoded columns behind a column encoding), then the head DKS_GAUSS_HEAD_*.
 * mu [K][D]; L_k is D x r_k (r_k >= 1), its columns stored as rows: row r_off[k] + t of L [r_off[K]][D] is column t of L_k
 * (r_off [K + 1] increasing from 0); gamma [K] positive, c [K]; everything finite.  QDA, GaussianNB, GaussianMixture,
 * BayesianGaussianMixture and EllipticEnvelope read this way (DESIGN.md §5.0.23), per-column scalers folded into mu and L.
 * Malformed input is DKS_ERR_UNSUPPORTED.
 * Every instance runs the Gaussian kernel (DKS_GENERAL_GAUSS), up to 64 groups: shared plans (full and partial varying
 * sets), per-instance device plans and caller-supplied plans, kernel 'auto' or 'simt' (tcgen05 / shared are
 * DKS_ERR_UNSUPPORTED), l1 selection through the general list's LARS route; every output is solved on its own.  Float64
 * throughout.  NaN or an infinity in a background row (dks_fit) or an instance (dks_predict_host, the explain calls) is
 * DKS_ERR_DOMAIN with the row; a link(ey) or link(f(x)) that is not finite is DKS_ERR_NUMERIC and nothing non-finite is
 * written into phi.  The explain kernel holds K (G^2 + 1) doubles of tables in shared memory: shapes that do not fit are
 * DKS_ERR_UNSUPPORTED.  dks_set_column_maps is refused; a Gaussian model is not an ensemble member. */
int dks_set_gaussian_model(dks_ctx* ctx, int K, int D, const int32_t* r_off, const double* mu, const double* L,
                           const double* gamma, const double* c, int head, int scalar_out);
/* soft-voting ensemble (DKS_ACT_ENSEMBLE) in place of dks_set_model: outputs f = sum_k pi_k f_k over K (1..DKS_ENS_MAX_MEMBERS)
 * members, pi = weights / sum(weights) (finite, >= 0, positive sum), members in order.  members [K] are distinct contexts on
 * the same device, each made by dks_create and one dks_set_tree_model / dks_set_kernel_machine / dks_set_mlp /
 * dks_set_knn_model (with the dks_set_background and dks_set_column_encoding that setter needs to know the model's width),
 * every one giving C (1..DKS_ENS_MAX_OUT) outputs.  The ensemble takes ownership: dks_destroy of the ensemble frees them,
 * and every call on a member afterwards is DKS_ERR_INVALID.  dks_fit fits every member on the ensemble's background,
 * weights, groups and column encoding; fnull = sum_k pi_k fnull_k.  All member launches go on the ensemble's stream.
 * Every instance runs the members' explain kernels back to back (DKS_GENERAL_ENSEMBLE, DESIGN.md §5.0.17), each adding
 * pi_k times its background means of every output into one workspace [n][C][S_cap], then explain_ensemble_tail_kernel takes
 * the link and the solve, every output solved on its own: K + 1 launches per call (stage 1: K predict launches and one
 * that forms f(x)).  Up to 64 groups, every plan source, kernel 'auto' or 'simt' (tcgen05 / shared are
 * DKS_ERR_UNSUPPORTED), l1 selection through the general list's LARS route.  A raw value any member refuses is
 * DKS_ERR_DOMAIN with the row (NaN in an ensemble of trees only is explained); a link(ey) or link(f(x)) that is not finite
 * is DKS_ERR_NUMERIC and nothing non-finite is written into phi. */
int dks_set_ensemble(dks_ctx* ctx, int K, dks_ctx* const* members, const double* weights, int C, int scalar_out);
/* stacking ensemble (DKS_ACT_STACKING) in place of dks_set_model: outputs f(x) = head(W m(x) + b + W_pass x) of the final
 * estimator (DKS_STACK_HEAD_*: R = C scores, or R = 1 and C = 2 under the sigmoid) over the meta columns m(x) [F]: outputs
 * col_first[k] .. col_first[k] + col_count[k] - 1 of each of the K (1..DKS_ENS_MAX_MEMBERS) members in order, F = sum
 * col_count <= DKS_STACK_MAX_F.  W [R][F], b [R] and W_pass [R][D] (passthrough over the columns the members read -- the
 * encoded ones behind a column encoding -- or NULL) must be finite.  Members, ownership, stream, status word and dks_fit of
 * the members follow dks_set_ensemble; fnull = sum_j w_j f(bg_j) in background order.  Every instance runs, per chunk
 * j0 <= j < j1 of the background, the members' explain kernels (each storing its kept outputs of every masked row (s, j)
 * into a workspace [n][F][j1 - j0][S_cap]) and stacking_reduce_kernel (the final estimator per row, ey(s) += w_j f), then
 * explain_ensemble_tail_kernel (DKS_GENERAL_STACKING, DESIGN.md §5.0.20).  The chunks are the fewest whose workspace fits
 * workspace_bytes (at least one background row each): chunks (K + 1) + 1 launches per call, phi bit-identical whatever the
 * chunking.  Up to 64 groups, every plan source, kernel 'auto' or 'simt', l1 selection through the general list's LARS
 * route; raw values and non-finite results are reported as for dks_set_ensemble.  Malformed input (non-finite weights,
 * column ranges outside a member's outputs, F or R out of range, R not matching the head) is DKS_ERR_UNSUPPORTED. */
int dks_set_stacking(dks_ctx* ctx, int K, dks_ctx* const* members, const int32_t* col_first, const int32_t* col_count,
                     const double* W, const double* b, int R, int head, const double* W_pass, int C, int scalar_out,
                     int64_t workspace_bytes);
/* a model the engine cannot evaluate (DKS_ACT_EXTERNAL) in place of dks_set_model: C (1..DKS_ENS_MAX_OUT) outputs that the
 * caller computes on the device from rows of `dtype` (DKS_EXTERNAL_FLOAT32 / _FLOAT64) -- a torch.nn.Module (DESIGN.md
 * §5.0.19).  Before dks_fit, dks_set_external_background hands over the module's outputs on the N background rows, y_dev
 * [N][C] of y_dtype in device memory, read on the context's stream before the call returns; fnull is their weighted mean.
 * The engine never calls the module, so dks_predict_host, dks_prepare_*, dks_explain_* and dks_run_dev are
 * DKS_ERR_UNSUPPORTED; a column encoding or column maps are refused.  An explain call is stepwise, all on the context's
 * stream (dks_set_stream: the caller's, so that its module runs in order with the engine's kernels):
 *   dks_external_prepare: stage 1 over the rows X_dev [n][D] (float64, device; kept by the caller until _finish returns)
 *     with the module's outputs fx_dev [n][C] on them (read before the call returns): varying groups, the M histogram,
 *     link(f(x)).  dks_get_m_histogram then decides the plans and the l1 selection as for any model.
 *   dks_external_begin: the route (shared, caller-supplied or device-drawn plans; l1 selection) and the coalition offsets;
 *     synchronises once and returns in *rows_total the masked rows of the call, sum over instances with M >= 2 of S_i N.
 *     DKS_ERR_PLAN_MISSING when a shared plan is missing (upload it and call again).
 *   dks_external_mask: masked rows row0 .. row0 + rows - 1 into out_dev [rows][D] of the module's dtype: row (i, s, j) =
 *     z_s(group(d)) ? x_i[d] : bg_j[d], rows numbered instances in index order, then coalition s of the instance's plan, then
 *     background row j; row0 and rows are whole coalitions (multiples of N).
 *   dks_external_reduce: the module's outputs y_dev [rows][C] (y_dtype) on those rows into the background means
 *     ey[i][c][s] = sum_j w_j y(i, s, j)_c, summed over j in a fixed order whatever the split into calls.
 *   dks_external_finish: link + constrained WLS (with l1 selection: moments, LARS, restricted solve) of every instance,
 *     phi_host [C][n][G] as dks_explain_host writes it (dks_summarise_host and dks_get_link_fx then apply); synchronises.
 * After dks_external_begin, another stage 1, a dks_fit, a plan or l1 table upload, a change of nsamples, plan mode, row
 * offset, kernel or stream makes _mask, _reduce and _finish DKS_ERR_INVALID until the call is prepared and begun again.
 * Under DKS_LINK_LOGIT every output is taken as a probability of its own: y = log(ey_c / (1 - ey_c)) - link(fnull_c), as
 * for f(x) and fnull, whether or not the outputs sum to one.
 * Up to 64 groups, kernel 'auto' or 'simt'; a non-finite link(ey), link(f(x)) or link(fnull) is DKS_ERR_NUMERIC. */
int dks_set_external_model(dks_ctx* ctx, int C, int scalar_out, int dtype);
int dks_set_external_background(dks_ctx* ctx, const void* y_dev, int y_dtype);
int dks_external_prepare(dks_ctx* ctx, const double* X_dev, int n, const void* fx_dev, int fx_dtype);
int dks_external_begin(dks_ctx* ctx, const uint64_t* ext_zbits_host, const double* ext_w_host, int ext_stride,
                       int64_t* rows_total);
int dks_external_mask(dks_ctx* ctx, int64_t row0, int64_t rows, void* out_dev);
int dks_external_reduce(dks_ctx* ctx, int64_t row0, int64_t rows, const void* y_dev, int y_dtype);
int dks_external_finish(dks_ctx* ctx, double* phi_host);
/* column maps (call after dks_set_model, before dks_fit): the scores become z_r = b_r + sum_col f_{r,col}(x_col), a linear
 * model behind per-column preprocessing (a scikit-learn Pipeline of scalers, encoders, binning and imputation) read in raw
 * feature space; W is then not read.  Per column, hdr_host[4 col ..] = {flags, m, key offset, value offset}:
 *   piecewise affine (flags & 1 == 0): m pieces, m - 1 strictly increasing breakpoints t at keys_host[key offset ..]; piece
 *     k = number of breakpoints <= x (numpy searchsorted side='right'), f_r(x) = a[k][r] x + c[k][r]; values [m][2][R] (the a
 *     row then the c row of each piece) then the NaN row [R];
 *   categorical (flags & 1): m strictly increasing keys; an exact match gives that key's row, no match the unknown row;
 *     values [m][R], the unknown row [R], then the NaN row [R].
 * flags & 2: NaN is refused; flags & 4 (categorical): an unknown value is refused.  A refused value is reported as
 * DKS_ERR_DOMAIN (by dks_fit for a background row, by dks_predict_host and the explain calls for an instance); it is never
 * evaluated.  Varying groups are still decided on the raw columns.  Malformed tables (shape, offsets, unsorted or
 * non-finite keys, non-finite values) return DKS_ERR_UNSUPPORTED.  hdr_host == NULL clears the maps; dks_set_model does too. */
int dks_set_column_maps(dks_ctx* ctx, int D, int R, const int32_t* hdr_host, const double* keys_host, int n_keys,
                        const double* vals_host, int n_vals);
/* column encoding of a tree ensemble, kernel machine, MLP or neighbour model (call after dks_set_background /
 * dks_set_groups, before dks_set_tree_model, dks_set_kernel_machine, dks_set_mlp or dks_set_knn_model, which then check the
 * model's width against E): the model reads E encoded columns, each an exact program over one raw column -- a scikit-learn
 * Pipeline of per-column steps replayed bit for bit (DESIGN.md §5.0.13, §5.0.16).  hdr_host [E][3] = {raw source column,
 * first op, op count}; ops_host [n_ops][4] = {code DKS_ENC_OP_*, flags DKS_ENC_*_ERROR, m, table offset}; opvals_host
 * [n_ops][2] = {c0, c1}; tab_host [n_tab]: per PIECES / TABLE op at its offset, the m strictly increasing finite edges /
 * keys, the m + 1 outputs (bins; or keys then the unknown output), then the NaN output.  Varying groups stay on the raw
 * columns: encoded column e belongs to the group of its source, and the model's kernels read the encoded rows, the
 * encoded background and (kernel machines, MLPs, neighbour models) a group CSR over the encoded columns.  The encode kernel
 * (one thread per row and encoded column) runs first in dks_fit, stage 1 and dks_predict_host; for kernel machines, MLPs
 * and neighbour models it also refuses a raw +-inf that an encoded column reads.  A refused value is DKS_ERR_DOMAIN (by
 * dks_fit for a background row, by dks_predict_host and the explain calls for an instance).  Malformed input (a source
 * out of range, an unknown op or flag, unsorted or non-finite keys or edges, non-finite constants, offsets out of range)
 * is DKS_ERR_UNSUPPORTED; so is any other model (dks_set_model and dks_set_mixture clear the encoding).  hdr_host == NULL
 * clears it. */
int dks_set_column_encoding(dks_ctx* ctx, int E, const int32_t* hdr_host, const int32_t* ops_host, const double* opvals_host,
                            int n_ops, const double* tab_host, int n_tab);
/* the encoded rows [n x E] of host rows X_host [n x D], computed by the device's encode kernel (needs dks_fit with an
 * encoding set); a refused value is DKS_ERR_DOMAIN with the row. */
int dks_encode_host(dks_ctx* ctx, const double* X_host, int n, double* out_host);
int dks_set_link(dks_ctx* ctx, int link);
/* runs the fit kernels (grouped background scores, fnull = sum_j w_j f(bg_j), link(fnull)); synchronises. */
int dks_fit(dks_ctx* ctx);
int dks_num_outputs(dks_ctx* ctx, int* C);
/* fnull[C] and expected_value[C] = link(fnull)  (KernelExplainer.fnull / .expected_value) */
int dks_get_fnull(dks_ctx* ctx, double* fnull_host, double* expected_value_host);
/* model outputs f(X) [n x C] for host rows (used to check the extracted model against the callable). */
int dks_predict_host(dks_ctx* ctx, const double* X_host, int n, double* out_host);

/* ---- coalition plans: the enumeration/sampling part of KernelExplainer.explain ----------------------
 * nsamples request shared by all instances: 0 = 'auto' (2M + 2048); capped per instance at 2^M - 2 (M<=30). */
int dks_set_nsamples(dks_ctx* ctx, int nsamples);
/* S an instance with M varying groups evaluates under the current request (upstream rule). */
int dks_effective_nsamples(dks_ctx* ctx, int M, int* S);
/* one plan shared by every instance with M varying groups: zbits [S][W] little-endian 64-bit words, W = 1 for M <= 64,
 * 2 for 64 < M <= 128 and 16 for 128 < M <= 1024 (bit k = k-th varying group present; multi-word rows are evaluated by the
 * shared-plan path only), w [S] kernel weights, in upstream row order.  Copies to the device and, up to 128 groups,
 * factors the normal matrix there. */
int dks_set_shared_plan(dks_ctx* ctx, int M, int S, const uint64_t* zbits_host, const double* w_host);
/* plans of more than 128 groups: the solve of KernelExplainer.solve (reached from kernel_shap.py:250/253; ungrouped wide
 * arrays: kernel_shap.py:581-621) in projection form, beta = P y - delta d with P = inv(E^T W E) E^T W and d = P z_L, factored
 * by the host in float64 (np.linalg.inv like upstream).  pt_host = P^T [S][M-1] row-major, dvec_host = d [M-1].  Call after
 * dks_set_shared_plan of the same M; the plan is reported present (dks_has_shared_plan) only with its projection. */
int dks_set_plan_projection(dks_ctx* ctx, int M, const double* pt_host, const double* dvec_host);
int dks_clear_plans(dks_ctx* ctx);
int dks_has_shared_plan(dks_ctx* ctx, int M, int* present);

/* ---- l1 feature selection: the l1_reg branch of KernelExplainer.solve (kwargs path kernel_shap.py:836-845, :880) --------
 * mode 0 = off (plain constrained WLS), 1 = LassoLarsIC 'aic' (what l1_reg='auto' means when under 20% of the coalition
 * space is sampled), 2 = 'bic', 3 = 'num_features(k)' (lars_path with max_iter = k); scikit-learn 0.23.2 semantics (the
 * reference's pin).  Upstream decides per instance whether to select (under 'auto' from its own M); the caller makes that
 * decision per M and passes the 128-bit set of the M that select: bit M - 1 of (sel_lo, sel_hi), M = 2..128.  Instances
 * whose M is not in the set take the plain constrained WLS.  Those whose groups all vary select on the shared-plan path;
 * those with a partial varying set (at most 64 groups, kernel auto or shared) on the CUDA-core kernel, which forms their
 * moments of y, and the same LARS kernel, on the shared plan of their own M.  A selecting instance no kernel covers is
 * reported as DKS_ERR_UNSUPPORTED, never solved without the selection.  dks_set_l1_tables uploads what plan.py:l1_tables
 * computes for the shared plan of M <= 128 groups (after dks_set_shared_plan), for every M in the set: Gram matrices of the
 * augmented system [M x M], column sums / norms / b-weighted column sums [M], the w-weighted Gram of the plain rows [M x M],
 * per-row b_s and sqrt(a_s) + sqrt(b_s) [S], and three scalars. */
int dks_set_l1(dks_ctx* ctx, int mode, int k, uint64_t sel_lo, uint64_t sel_hi);
int dks_set_l1_tables(dks_ctx* ctx, int M, const double* gram_raw, const double* gram_norm, const double* colsum,
                      const double* scale, const double* bz, const double* gram_w, const double* b_rows,
                      const double* sqab_rows, double sum_b, double sum_sqb, int n_aug);

/* ---- per-instance plans drawn on the device -----------------------------------------------------------
 * shap.KernelExplainer.explain draws a fresh plan for every instance (the sampling loop that follows the subset
 * enumeration; reached from kernel_shap.py:250/253).  Mode 1 does that on the GPU: the enumerated prefix comes from the
 * shared plan of the instance's M, the sampled rows from Philox4x32-10 keyed by `seed` with counter (draw, global row),
 * with upstream's duplicate / complement / truncation / rescaling rules.  Plans depend on the global row index only
 * (dks_set_row_offset gives the index of row 0 of the next call), never on batching or the number of GPUs.
 * Up to 64 groups every instance draws a one-word plan; from 65 to 128 groups (two-word rows) the instances whose groups
 * all vary do, with the binary-logistic, identity or exp head and kernel auto or simt (DKS_GENERAL_SIMT_WIDE).  A partial varying
 * set, another head, kernel tcgen05 / shared, l1 selection or more than 128 groups is reported as DKS_ERR_UNSUPPORTED there.
 * dks_set_plan_sampling uploads what the sampler needs for one M <= 128 (plan.py: sampling_info); cdf has ncdf <= 64
 * entries (M <= 128 has at most 63 sampled sizes). */
int dks_set_plan_sampling(dks_ctx* ctx, int M, int nfixed, int n_full, int n_paired, int ncdf, const double* cdf_host,
                          double weight_left);
int dks_set_plan_mode(dks_ctx* ctx, int mode /* 0 shared per M, 1 per instance */, uint64_t seed);
int dks_set_row_offset(dks_ctx* ctx, int64_t offset);
/* plans of the last mode-1 explain call ([n][stride] each; pass NULL buffers to query n and stride); tests / audit.
 * One-word rows only: when the last plans have two-word rows (65..128 groups) copying them is DKS_ERR_INVALID. */
int dks_get_instance_plans(dks_ctx* ctx, uint64_t* zbits_host, double* w_host, int* n_out, int* stride_out);
/* the same for any row width: zbits [n][stride][words], w [n][stride]; *words_out = 1 (up to 64 groups) or 2. */
int dks_get_instance_plans_w(dks_ctx* ctx, uint64_t* zbits_host, double* w_host, int* n_out, int* stride_out,
                             int* words_out);

/* ---- explain: KernelExplainer.shap_values (reached from kernel_shap.py:250/253) ---------------------
 * Stage 1 (dks_prepare_*): per instance, grouped contributions W_g x_g, f(x), link(f(x)) - link(fnull),
 * varying_groups() bit-mask and M.  X is [n x D] row-major float64. */
int dks_prepare_host(dks_ctx* ctx, const double* X_host, int n);
int dks_prepare_dev(dks_ctx* ctx, const double* X_dev, int n);
/* after prepare: hist[m] = number of instances with M == m, m in [0, G]; synchronises. */
int dks_get_m_histogram(dks_ctx* ctx, int32_t* hist_host);
/* after prepare / explain: link(f(x)) per instance and output, [n][C] -- what KernelShap.build_explanation stores as
 * `raw_prediction` (kernel_shap.py:949 runs the predictor over X a second time for it); synchronises. */
int dks_get_link_fx(dks_ctx* ctx, double* out_host, int n /* rows the caller's buffer holds: must match */);
/* after prepare: per-instance M and varying bit-mask (debug / tests); synchronises. */
int dks_get_varying(dks_ctx* ctx, int32_t* M_host, uint64_t* mask_host);

/* Stage 2: evaluate coalitions + solve.  phi is [C x n x G] float64 (one [n x G] slab per model output,
 * the list-of-arrays layout KernelExplainer.shap_values returns).
 * Plans: ext_zbits/ext_w == NULL -> shared plans (dks_set_shared_plan) looked up by each instance's M;
 * otherwise per-instance plans [n x ext_stride] (row i holds the S_i = dks_effective_nsamples(M_i) rows of
 * instance i), device pointers for _dev and host pointers for _host. */
int dks_explain_dev(dks_ctx* ctx, double* phi_dev, const uint64_t* ext_zbits_dev, const double* ext_w_dev,
                    int ext_stride);
/* prepare + explain for rows resident in device memory with the engine's own plans, as ONE CUDA-graph launch once the
 * same call (same buffers, n, nsamples, kernel, plans) has been seen twice: the second call captures the sequence (memset,
 * stage 1, coalition kernels, solve), later ones replay it.  DKS_GRAPH=0 in the environment keeps plain launches.
 * Asynchronous like dks_explain_dev; dks_last_timings keeps working (external event-record nodes). */
int dks_run_dev(dks_ctx* ctx, const double* X_dev, int n, double* phi_dev);
int dks_graph_launches(dks_ctx* ctx, int64_t* count);
/* Multi-GPU, one process per GPU: gathered_ptrs_host[r] is the device address, valid in THIS process (peer mapping, e.g.
 * torch symmetric memory), of rank r's gathered buffer [world][slab_doubles].  After every dks_run_dev the engine stores
 * its phi into slab `rank` of every peer's buffer with its own kernel over NVLink peer memory -- the all-gather of the
 * reference's result collection (distributed.py:156-179) without NCCL; the caller completes it with a cross-GPU barrier.
 * Pass phi_dev = own buffer + rank * slab_doubles to have the solve write the local slab in place.  world <= 1 clears. */
int dks_set_peers(dks_ctx* ctx, int world, int rank, const uint64_t* gathered_ptrs_host, int64_t slab_doubles);
/* Optional completion of that all-gather inside the engine: flag_ptrs_host[r] is the device address (mapped in THIS process) of
 * rank r's flag array, uint64[world], zero-initialised (peer-mapped like the gathered buffers).  With flags set, every
 * dks_run_dev ends with the engine's own cross-GPU signal/wait (one thread per peer, system-scope release/acquire): when the
 * call's stream work is done, every peer's block has arrived in this rank's gathered buffer -- no library barrier needed.
 * Call after dks_set_peers; NULL switches it off. */
int dks_set_peer_flags(dks_ctx* ctx, const uint64_t* flag_ptrs_host);
/* convenience: prepare + explain from/to host memory; H2D, kernels, D2H; synchronises.  This is the call a
 * non-torch host (ctypes / cgo) makes and the one bench.py's end-to-end number goes through. */
int dks_explain_host(dks_ctx* ctx, const double* X_host, int n, double* phi_host, const uint64_t* ext_zbits_host,
                     const double* ext_w_host, int ext_stride);
/* Page-locked host memory for result arrays (optional).  When the phi_host handed to dks_explain_host lies in page-locked
 * memory (allocated here, or registered by the caller) the shap values arrive by ONE asynchronous DMA; pageable memory goes
 * through the library's pinned staging buffer and a host memcpy. */
int dks_host_alloc(void** out, uint64_t bytes);
int dks_host_free(void* p);
/* status of the LAST explain call on this context (the asynchronous calls leave it on the device; this fetches it and
 * synchronises): 0 ok, DKS_ERR_PLAN_MISSING, DKS_ERR_NUMERIC, DKS_ERR_UNSUPPORTED;
 * *detail = the offending M / instance index. */
int dks_last_status(dks_ctx* ctx, int* detail);

/* ---- post-processing of KernelShap.build_explanation off the resident phi (kernel_shap.py:36-109 rank_by_importance, :112-207
 * sum_categories, :952-956 argmax) for the rows of the LAST dks_explain_host call: segment sums over consecutive groups
 * (seg_offsets_host [Gp + 1], NULL = one segment per group, Gp = G), mean |phi| per output and aggregated over outputs
 * ([C + 1][Gp]), their descending order, argmax of the raw prediction.  Output pointers may be NULL.  Synchronises. */
int dks_summarise_host(dks_ctx* ctx, int n, const int32_t* seg_offsets_host, int Gp, double* phi_sum_host,
                       double* mean_abs_host, int32_t* order_host, int32_t* argmax_host);

/* ---- knobs / introspection ---------------------------------------------------------------------- */
int dks_set_kernel(dks_ctx* ctx, int kernel);       /* DKS_KERNEL_* */
/* tuning knobs, all optional (defaults are the measured best): "fused" 0/1 -- link + projection solve inside the shared-plan
 * coalition kernel (default 1; 0 = separate (sum p1, sum p0) buffer + solve kernel); "fused_warps" caps the warps per CTA (default: as many as fit, at most 20); "fused_batch" instances
 * parked per warp before the turn-around; "fused_table" 0/1 -- the fused kernel reads y from the plan's link table
 * (default 1; 0 = the exact loop over the background for every pass);
 * "push_in_kernel" 0/1 -- multi-GPU: the fused route's finish kernel stores the phi rows of its instances into the peers'
 * buffers as it writes them, and the push kernel after the solve moves only the other instances' rows (default 0: the
 * push kernel moves every row); "graph" 0/1 (CUDA-graph
 * replay of dks_run_dev); "graph_timing" 0/1 -- keep the timing event records inside the graph (default 0: a replayed graph
 * carries no timing nodes and dks_last_timings reports an error after it). */
int dks_set_option(dks_ctx* ctx, const char* name, int value);
int dks_kernel_launches(dks_ctx* ctx, int64_t* count); /* kernels launched by this ctx so far */
/* device and pinned-host allocations the library holds for itself now, across every context of the process (memory from
 * dks_host_alloc belongs to the caller and is not counted): a context that is destroyed gives back all it took */
int dks_live_allocations(int64_t* count);
/* The fused kernel's link table of the plan over M groups: its bytes (0 = the plan has none and the kernel runs the exact
 * loop), and the passes of this ctx's fused launches so far that left a table's domain and took the exact loop. */
int dks_fused_table_info(dks_ctx* ctx, int M, int64_t* table_bytes, int64_t* fallback_passes);
/* Which kernels the last explain call launched (dks_explain_* / dks_run_dev), recorded on the host while the launch
 * sequence is enqueued: a CUDA-graph replay keeps the record of the call it captured.  out[0 .. n) receives the first n
 * of the DKS_PATH_FIELDS entries indexed by DKS_PATH_*; n may be smaller (older callers) or larger (zero-filled). */
#define DKS_PATH_SHARED 0        /* shared-plan coalition kernel: DKS_SHARED_* */
#define DKS_PATH_CHUNKS 1        /* background chunks (launches) of the unfused coalition kernel; 1 for the fused one */
#define DKS_PATH_WARPS 2         /* warps per CTA the coalition kernel uses (the fewest over the chunks) */
#define DKS_PATH_GRID 3          /* CTAs of the coalition kernel (the largest over the chunks) */
#define DKS_PATH_FUSED_B 4       /* fused kernel: instances parked per warp before the turn-around */
#define DKS_PATH_FUSED_NI 5      /* fused kernel: instances per pass over a warp's rows (1) */
#define DKS_PATH_SOLVE 6         /* DKS_SOLVE_* */
#define DKS_PATH_PMAT_KPAD 7     /* projection solve (DKS_SOLVE_PMAT): coefficient rows of P, padded */
#define DKS_PATH_GENERAL 8       /* DKS_GENERAL_*: the kernel of the instances the shared-plan path does not take */
#define DKS_PATH_FUSED_CTA_WARPS 9 /* fused kernel: warps per CTA it runs.  DKS_PATH_WARPS is the row-group slices a CTA
                                    * holds with one warp per slice (what decides fused or not); when fewer slices cover the
                                    * plan, several warps share each slice and this is larger */
#define DKS_PATH_BG_WEIGHTS 10   /* shared-plan kernels: 0 = uniform-background instantiations, 1 = the weighted ones
                                  * (background weights not all equal) */
#define DKS_PATH_FUSED_TABLE 11  /* fused kernel: 1 = y read from the plan's per-row link table (passes outside its domain
                                  * take the exact loop), 0 = exact loop only ("fused_table" 0, or the plan has no table) */
#define DKS_PATH_GENERAL_L1 12   /* 1: the general list's instances whose M selects ran the l1 selection (moments on the
                                  * CUDA-core kernel, then the LARS kernel); DKS_PATH_GENERAL names the rest's kernel */
#define DKS_PATH_FIELDS 13
#define DKS_SHARED_NONE 0
#define DKS_SHARED_FUSED 1       /* explain_shared_fused_kernel: link + projection solve inside */
#define DKS_SHARED_SMEM 2        /* explain_shared_smem_kernel (Dm rows in shared memory) */
/* 3 is not used: a retired kernel's code, kept free so that the other codes keep their meaning */
#define DKS_SHARED_SOFTMAX 4     /* explain_softmax_kernel: per-class sums of the softmax head (C = R classes) */
#define DKS_SHARED_AFFINE 5      /* identity head: y read from per-class tables, no coalition kernel */
#define DKS_SHARED_OVR 6         /* explain_ovr_kernel: per-class sums of the one-vs-rest head (C = R classes) */
#define DKS_SHARED_EXP 7         /* exp head: y from the instance's tables and the plan's l(s), no coalition kernel */
#define DKS_SHARED_MIX 8         /* mixture head: one pass of the member head's coalition kernel per member (binary members:
                                  * explain_shared_smem_kernel, softmax / one-vs-rest members: the class-sum kernels), each
                                  * added times pi_k into one set of sums; DKS_PATH_CHUNKS counts member x chunk launches */
#define DKS_SOLVE_NONE 0
#define DKS_SOLVE_FUSED 1
#define DKS_SOLVE_PMAT 2         /* wls_pmat_kernel */
#define DKS_SOLVE_WLS_SHARED 3   /* wls_shared_kernel */
#define DKS_SOLVE_WIDE 4         /* more than 128 groups: float64 projection product (dks_wide.cuh) */
#define DKS_SOLVE_L1 5           /* l1 feature selection + restricted WLS */
#define DKS_GENERAL_NONE 0
#define DKS_GENERAL_TC 1         /* explain_wgmma_kernel */
#define DKS_GENERAL_SIMT 2       /* explain_simt_kernel */
#define DKS_GENERAL_FLAGGED 3    /* not computed: instances left for it are reported as DKS_ERR_UNSUPPORTED */
#define DKS_GENERAL_SIMT_WIDE 4  /* explain_wide_instance_kernel: per-instance plans of 65..128 groups (two-word rows) */
#define DKS_GENERAL_TREES 5      /* explain_tree_kernel: every instance of a tree ensemble (dks_set_tree_model) */
#define DKS_GENERAL_KMACH 6      /* explain_kmach_kernel: every instance of a kernel machine (dks_set_kernel_machine) */
#define DKS_GENERAL_MLP 7        /* explain_mlp_kernel: every instance of a multi-layer perceptron (dks_set_mlp) */
#define DKS_GENERAL_KNN 8        /* explain_knn_kernel: every instance of a nearest-neighbour model (dks_set_knn_model) */
#define DKS_GENERAL_ENSEMBLE 9   /* the members' explain kernels, then explain_ensemble_tail_kernel: every instance of a
                                  * soft-voting ensemble (dks_set_ensemble) */
#define DKS_GENERAL_EXTERNAL 10  /* explain_ensemble_tail_kernel on the means dks_external_reduce formed: every instance of a
                                  * module the caller runs (dks_set_external_model) */
#define DKS_GENERAL_STACKING 11  /* per background chunk the members' explain kernels and stacking_reduce_kernel, then
                                  * explain_ensemble_tail_kernel: every instance of a stacking ensemble (dks_set_stacking) */
#define DKS_GENERAL_GAUSS 12     /* explain_gauss_kernel: every instance of a Gaussian model (dks_set_gaussian_model) */
int dks_last_path(dks_ctx* ctx, int32_t* out, int n);
/* device-time of the last explain's stages in ms (CUDA events on the ctx stream): [0] prepare, [1] fused
 * coalition kernel, [2] total; synchronises. */
int dks_last_timings(dks_ctx* ctx, float* ms3);
/* device-time in ms of the last explain's general-list l1 selection (DKS_PATH_GENERAL_L1): [0] the CUDA-core kernel that
 * forms the moments, [1] the LARS kernel; an error when that call ran none (or was captured into a graph); synchronises. */
int dks_last_general_l1_timings(dks_ctx* ctx, float* ms2);

/* ---- debugging aid for the tensor-core kernel (tests only) ---------------------------------------------------
 * dks_debug_score_dump(ctx, i): the next explains also write the raw accumulator tile of instance i (scaled masked
 * scores T[s][j], float32 [rows x cols]); i < 0 switches it off.  dks_debug_get_scores copies the dump to the host
 * (synchronises); rows/cols report its shape. */
int dks_debug_score_dump(dks_ctx* ctx, int instance);
int dks_debug_get_scores(dks_ctx* ctx, float* out_host, int max_floats, int* rows, int* cols);
/* cycle timeline of CTA 0 recorded by the same debug run: float32 [6][256], event e of tile g at [e*256+g]
 * (0 A tile ready, 3 consumer starts waiting for it, 4 A tile seen by the consumer, 5 tile drained; 1 and 2 unused) */
int dks_debug_get_timeline(dks_ctx* ctx, float* out_host);

#ifdef __cplusplus
}
#endif
#endif /* DKS_H_ */
