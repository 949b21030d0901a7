// Shared declarations of the H100 KernelSHAP engine (host context + device parameter blocks).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <string>
#include <utility>
#include <vector>

#include "dks.h"

// ---- the memory the library holds for itself (host-only) --------------------------------------------------------------
// Every device and pinned-host allocation of the library goes through this one pair, which counts what is live across the
// process's contexts (dks_live_allocations).  The free is the synchronous one: its implicit device synchronisation is what
// makes freeing a buffer that a kernel in flight still reads safe.
namespace dks {
inline std::atomic<int64_t> g_live_allocations{0};

inline cudaError_t mem_alloc(void** p, size_t bytes, bool pinned) {
    const cudaError_t e = pinned ? cudaHostAlloc(p, bytes, cudaHostAllocDefault) : cudaMalloc(p, bytes);
    if (e == cudaSuccess) g_live_allocations++;
    return e;
}

inline void mem_free(void* p, bool pinned) {
    if (!p) return;
    if (pinned) cudaFreeHost(p);
    else cudaFree(p);
    g_live_allocations--;
}
}  // namespace dks

// an array of device (or pinned host) memory and its element count, freed when it is reset, reallocated or destroyed
template <typename T, bool PINNED = false>
class DksBuf {
public:
    DksBuf() = default;
    DksBuf(DksBuf&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
    DksBuf(const DksBuf&) = delete;
    DksBuf& operator=(const DksBuf&) = delete;
    ~DksBuf() { reset(); }

    // frees what it holds, then holds `count` elements (at least one)
    cudaError_t alloc(size_t count) {
        reset();
        if (count == 0) count = 1;
        void* p;
        const cudaError_t e = dks::mem_alloc(&p, count * sizeof(T), PINNED);
        if (e == cudaSuccess) { p_ = static_cast<T*>(p); n_ = count; }
        return e;
    }
    void reset() { dks::mem_free(std::exchange(p_, nullptr), PINNED); n_ = 0; }
    T* release() { n_ = 0; return std::exchange(p_, nullptr); }     // the caller takes the memory over
    size_t size() const { return n_; }
    T* get() const { return p_; }
    operator T*() const { return p_; }

private:
    T* p_ = nullptr;
    size_t n_ = 0;
};
template <typename T> using DevBuf = DksBuf<T, false>;
template <typename T> using PinnedBuf = DksBuf<T, true>;

// device arrays whose pointers sit inside by-value kernel structs (TreeDev, PlanDev, ...): allocated through the pool that
// owns them and freed together by clear() or the pool's destructor
class DevPool {
public:
    DevPool() = default;
    DevPool(const DevPool&) = delete;
    ~DevPool() { clear(); }

    template <typename T>
    cudaError_t alloc(T** p, size_t count) {
        DevBuf<T> b;
        const cudaError_t e = b.alloc(count);
        *p = b;
        if (e == cudaSuccess) adopt(std::move(b));
        return e;
    }
    // the device copy of a host array, ordered on `stream`
    template <typename T>
    cudaError_t upload(const T** dst, const T* src, size_t count, cudaStream_t stream) {
        T* p;
        const cudaError_t e = alloc(&p, count);
        *dst = p;
        if (e != cudaSuccess || count == 0) return e;
        return cudaMemcpyAsync(p, src, sizeof(T) * count, cudaMemcpyHostToDevice, stream);
    }
    template <typename T>
    void adopt(DevBuf<T>&& b) { bufs_.push_back(b.release()); }
    void clear() {
        for (void* q : bufs_) dks::mem_free(q, false);
        bufs_.clear();
    }
    bool empty() const { return bufs_.empty(); }

private:
    std::vector<void*> bufs_;
};

#define DKS_MAX_GROUPS 1024 // coalition rows: one 64-bit word up to 64 groups; two words up to 128 and sixteen up to 1024 on
                            // the shared-plan path only
#define DKS_MAX_OUT 128     // model outputs a thread may hold in local arrays (R <= 8 score rows, C <= 8 outputs today)

// 64-bit words per coalition row of a plan over M groups: the kernels exist for rows of 1, 2 and 16 words
__host__ __device__ __forceinline__ int dks_plan_words(int M) { return M <= 64 ? 1 : (M <= 128 ? 2 : 16); }

namespace dks { namespace shared_path { struct LinkTabEntry; struct LinkTabRow; } }   // dks_fused.cuh

// ---- device-visible plan table entry: one shared coalition plan per number of varying groups M ----------
struct PlanDev {
    const uint64_t* z;   // [S][W] coalition bits in upstream row order (W = dks_plan_words(M))
    const double* w;     // [S] kernel weights
    const double* chol;  // [(M-1) x (M-1)] lower Cholesky factor of E^T W E (row-major), NULL if not factored
    const double* ainv;  // [(M-1) x (M-1)] inverse of E^T W E (row-major), NULL if not computed
    const float* dmT;    // [N][S_pad] 2^(scaled background part of the score - dme[s]) for the full varying set (shared fast path)
    const double* dme;   // [S_pad] row exponents: Dm rows are normalised so that their largest entry is ~1
    const float* pmat;   // [(M-1)][S_pad] P = inv(E^T W E) E^T W (float32): beta = P y - delta * dvec
    const double* dvec;  // [(M-1)] P z_L
    const double* pmat64;  // [S_pad][kpad] float64 P, one row per coalition (fused kernel), NULL if not built
    const double* dvec64;  // [kpad] P z_L with the float64 P
    const double* ptw;     // [S_pad][kpw] float64 P^T supplied by the host for plans of more than 128 groups (dks_wide.cuh)
    const double* dvecw;   // [kpw] P z_L
    const dks::shared_path::LinkTabEntry* ltab;      // per-row link table of the fused kernel, NULL if not built
    const dks::shared_path::LinkTabRow* ltab_rows;   // [S_pad]
    double ltab_inv_h;                               // 1 / its grid step
    long long ltab_bytes;                            // table and row headers
    int kpw;
    int kpad;
    int S;
    int S_pad;
    int W;               // 64-bit words per row
};

// ---- l1 feature selection: what plan.py:l1_tables computes for the shared plan of M groups (dks_set_l1_tables) -------
#define DKS_L1_MAX_GROUPS 128
namespace dks { namespace l1 {
struct Tables {              // device pointers
    const double* gram_raw;  // [M][M]
    const double* gram_norm; // [M][M]
    const double* colsum;    // [M]
    const double* scale;     // [M]
    const double* bz;        // [M]
    const double* gram_w;    // [M][M] sum_s w_s z_sk z_sl
    const double* b;         // [S] w_s |z_s|
    const double* sqab;      // [S] sqrt(a_s) + sqrt(b_s)
    double sum_b, sum_sqb;
    int n_aug, S;
};
} }

// What the device-side sampler needs to continue a plan past its enumerated prefix (per M; plan.py: sampling_info)
struct DksSamplingInfo {
    int nfixed;           // enumerated rows
    int n_full;           // fully enumerated subset sizes
    int n_paired;         // sizes whose complement has a different size
    int ncdf;             // sizes left to sample (0: the plan is fully enumerated)
    double weight_left;   // kernel mass of the sampled sizes
    double cdf[64];       // cumulative probabilities of the sampled sizes (last = 1); M <= 128 has at most 63
};

// nsamples resolution of KernelExplainer.explain: 'auto' (req <= 0) = 2M + 2^11; capped at 2^M - 2 for M <= 30
__host__ __device__ __forceinline__ int dks_effective_S(int M, int req) {
    long long s = req > 0 ? (long long)req : 2LL * M + 2048;
    if (M <= 30) {
        long long mx = (1LL << M) - 2;
        if (s > mx) s = mx;
    }
    return (int)s;
}

// ---- parameters of the fused coalition kernel ------------------------------------------------------------
struct ExplainParams {
    int n, N, G, R, C;
    int act, link;
    int S_req;
    int S_cap;            // capacity of the per-CTA y buffer (max S any instance can need)
    double scale;         // binary head: -kappa*log2(e); applied to grouped contributions
    const float* BWs;     // [R][G][N] scaled grouped background contributions (k-major: column j contiguous)
    const float* bases;   // [R][N]   scaled background scores
    const float* wbf;     // [N]      background weights (float)
    const double* wbg;    // [N]
    const double* Bbar;   // [G][R]   weighted mean grouped background contribution (identity head)
    const double* fnull;  // [C]
    const double* linkfnull;  // [C]
    const double* XW;     // [n][G][R] grouped instance contributions (unscaled)
    const uint64_t* vmask;  // [n]
    const int* Mcnt;      // [n]
    const double* dlink;  // [n][C] link(f(x)) - link(fnull)
    const PlanDev* plans; // [DKS_MAX_GROUPS + 1]
    const uint64_t* ext_z;  // per-instance plans or NULL
    const double* ext_w;
    int ext_stride;
    const double* ext_chol;   // per-instance Cholesky factor / inverse of E^T W E prepared with the plans ([n][ext_fstride],
    const double* ext_ainv;   // compact (M-1) x (M-1) row-major), or NULL: the explain kernel builds and factors it
    int ext_fstride;
    double* phi;          // [C][n][G]
    int* status;          // [2] {code, detail}
    const int* list;      // instances this launch handles (NULL = all n) ...
    const int* count;     // ... and how many (device memory)
};

// column maps (dks_set_column_maps, DESIGN.md §5.0.9): per raw column, a piecewise affine or categorical function giving
// that column's R score contributions -- a linear model behind per-column preprocessing, read in raw feature space
#define DKS_CM_CATEGORICAL 1
#define DKS_CM_NAN_ERROR 2
#define DKS_CM_UNKNOWN_ERROR 4
struct ColumnMapsDev {
    const int* hdr;       // [D][4] {flags, m, key offset, value offset}
    const double* keys;   // breakpoints (m - 1 per affine column) / keys (m per categorical column)
    const double* vals;   // affine [m][2][R] + NaN row [R]; categorical [m][R] + unknown row [R] + NaN row [R]
    int n_keys, n_vals;
};

// float64 background of the exp head's rows outside the range rule (a kernel parameter of its own: ExplainParams is
// embedded in other kernels' parameter blocks, whose layout stays as it is)
struct ExpBackground {
    const double* BW;     // [N][G] grouped background contributions
    const double* scores; // [N]    background scores
};

// mixture head (dks_set_mixture, DESIGN.md §5.0.10): outputs sum_k pi_k h(z_k), K members of R_m score rows each, stacked
// member-major (row k R_m + q), all with the member head h (binary-logistic with kappa folded into the scores, softmax or
// one-vs-rest); K R_m <= DKS_MIX_MAX_R
#define DKS_MIX_MAX_R 32
#define DKS_LOG2E 1.4426950408889634
struct MixHead {
    int K, Rm, mact;             // members, score rows per member, member head (DKS_ACT_*)
    float pif[DKS_MIX_MAX_R];    // pi_k in float (the CUDA-core kernel's fp32 sums)
    double pi[DKS_MIX_MAX_R];    // pi_k > 0, sum 1
};

// tree ensembles (dks_set_tree_model, DESIGN.md §5.0.11): every tree's nodes concatenated; raw scores r = base + sum over
// trees of the leaf value [R], then the head DKS_TREE_HEAD_*.  A split sends x left when x <= thr (DKS_TREE_CMP_F32: the value
// cast to float32 first, as sklearn.tree does), NaN where miss says.  Children have larger indices than their parent.
#define DKS_TREE_MAX_R 8
struct TreeDev {
    const int* feat;             // [nodes] split column, -1 at a leaf
    const double* thr;           // [nodes]
    const int* left;             // [nodes] global node indices
    const int* right;
    const unsigned char* miss;   // [nodes] 1: NaN goes left
    const double* val;           // [nodes][R] leaf values (learning rate / 1 over T folded in)
    const int* roots;            // [T]
    const double* base;          // [R]
    const int* colgrp;           // [D] group of each column
    const unsigned char* bgdir;  // [N][nodes] 1: background row j goes left at the node (internal nodes)
    unsigned char* xinfo;        // [CTAs][nodes] explain kernel scratch: (x goes left) << 7 | varying position (127: none)
    int nodes, T, R, head, cmp;
    double offset;               // subtracted by the anomaly head (DKS_TREE_HEAD_IFOREST), dks_set_tree_offset
};

// column encoding of a model with its own kernel (dks_set_column_encoding, DESIGN.md §5.0.13, §5.0.16): E encoded columns,
// each a program of DKS_ENC_OP_* over one raw column (dks_encode.cuh)
struct EncodingDev {
    const int* hdr;              // [E][3] {raw source column, first op, op count}
    const int* ops;              // [n_ops][4] {code, flags, m, table offset}
    const double* opv;           // [n_ops][2] constants
    const double* tab;           // lookups: keys [m], outputs [m + 1], NaN output
    int E;                       // 0: no encoding
};

// kernel machines (dks_set_kernel_machine, DESIGN.md §5.0.12): K members, member k owning support vectors sv_off[k] ..
// sv_off[k + 1]; f_k = sum_v dual[v] phi(t) + icpt, t = sum_c h(x_c, sv_c) per DKS_KM_KERNEL_*, then the head
// DKS_KM_HEAD_*.  Intercepts icpt[k R + q] (K R <= DKS_KM_MAX_K: one member of R <= 8 outputs, or K members of one).
struct KmDev {
    const double* sv;            // [n_sv][D] support vectors in raw feature space
    const double* dual;          // [n_sv][R]
    const double* colw;          // [K][D] column weights (the member's scalers folded in)
    const double* colo;          // [K][D] column origins (dot-product kernels)
    const double* Tbg;           // [N][n_sv] fit: t of background row j and support vector v
    int sv_off[DKS_KM_MAX_K + 1];
    double gamma[DKS_KM_MAX_K], icpt[DKS_KM_MAX_K], cal_a[DKS_KM_MAX_K], cal_b[DKS_KM_MAX_K], pi[DKS_KM_MAX_K];
    double degree, coef0;
    int K, R, n_sv, kernel, head;
};

// multi-layer perceptrons (dks_set_mlp, DESIGN.md §5.0.14): L = hidden + 1 weight layers, layer l mapping width[l] units to
// width[l + 1] (width[0] = D raw columns, width[L] = R outputs).  The explain kernel reads layers 1 .. L - 1 in the FP64 mma
// B-fragment order, zero-padded to pad[l] x pad[l + 1] (hidden widths to a multiple of 16, the output layer to 8): padding
// is zero weights, never zero activations.
struct MlpDev {
    const double* W;             // layer l: [width[l]][width[l + 1]] row-major at woff[l] (layer 0: the scalers folded in)
    const double* b;             // layer l: [width[l + 1]] at boff[l]
    const double* Wf;            // layers 1 .. L - 1: [pad[l] / 16][pad[l + 1] / 8][32 lanes][4] at wfoff[l]
    const double* bp;            // every layer's biases zero-padded to pad[l + 1], at bpoff[l]
    const double* Bbg;           // [N][width[1]] fit: b_0 + bg_j W_0
    int woff[DKS_MLP_MAX_HIDDEN + 1], boff[DKS_MLP_MAX_HIDDEN + 1], wfoff[DKS_MLP_MAX_HIDDEN + 1], bpoff[DKS_MLP_MAX_HIDDEN + 1];
    int width[DKS_MLP_MAX_HIDDEN + 2], pad[DKS_MLP_MAX_HIDDEN + 2];
    int L, act, head, R;
    int nbuf, hmax;              // activation buffers per warp (2 with two or more hidden layers) and the widest padded layer
};

// k-nearest neighbours (dks_set_knn_model, DESIGN.md §5.0.15): t(x, v) = sum_c h((colw_c x_c + colo_c) - v_c) per
// DKS_KNN_METRIC_*, the k smallest (t, index) over the training rows, then the vote or mean per DKS_KNN_HEAD_*
struct KnnDev {
    const double* fitX;          // [n_fit][D] training rows in the fitted space
    const double* colw;          // [D] x' = colw x + colo (the scalers folded in)
    const double* colo;          // [D]
    const double* y;             // classify: [n_fit] class index; regress: [n_fit][R]
    const int* colgrp;           // [D] group of every column
    const double* Tbg;           // [N][n_fit] fit: t of background row j and training row v
    const uint64_t* Ebg;         // [N][n_fit] fit: the groups on which background row j equals training row v exactly
    double p;                    // Minkowski exponent
    int n_fit, k, metric, weights, R, head;
};

// exp head, CUDA-core kernels (DESIGN.md §5.0.8): a coalition row is summed in fp32 when the largest weighted background
// exponent t'_j = log2 e d(s, j) + log2 w_j lies in [EXP_T_LO, EXP_T_HI]; other rows are evaluated in float64
#define DKS_EXP_T_LO -60.f
#define DKS_EXP_T_HI 100.f

// ---- what the host dispatcher knows about the head: filled once per dks_fit (describe_head, dks.cu) ----------------
enum HeadShared {               // what the shared-plan route of the full varying set evaluates
    HEAD_SHARED_BINARY,         // the binary-logistic head's Dm tables
    HEAD_SHARED_CLASS_SUMS,     // per-class sums of the softmax / one-vs-rest coalition kernels
    HEAD_SHARED_TABLES,         // y from the instance's nibble tables alone (identity; exp with the plan's l(s))
    HEAD_SHARED_MIX_BINARY,     // mixture of binary-logistic members: the binary head's kernel per member
    HEAD_SHARED_MIX_CLASS,      // mixture of softmax / one-vs-rest members: the class-sum kernel per member
};
// stacking ensemble (dks_set_stacking, DESIGN.md §5.0.20): the final estimator and the member columns it reads (by value;
// W, b and W_pass in device memory)
struct StackDev {
    const double* W;         // [R][F]
    const double* b;         // [R]
    const double* Wp;        // [R][D] passthrough weights over the columns the members read, or NULL
    int K, F, R, C, head, D;
    int ck[DKS_ENS_MAX_MEMBERS];        // outputs of member k
    int cfirst[DKS_ENS_MAX_MEMBERS];    // its first output kept
    int ccount[DKS_ENS_MAX_MEMBERS];    // outputs kept
};

struct HeadDesc {
    int shared = HEAD_SHARED_BINARY;
    bool ovr = false;           // the class sums (of the head or of its members) are one-vs-rest ones
    bool expo = false;          // exp head: the plan's l(s) and the exp instantiations of the CUDA-core kernels
    int shared_max_G = 0;       // the most groups the shared-plan route covers
    double scale = 1.0;         // applied to the grouped background contributions (fit) and the Dm tables
    double xt_scale = 1.0;      // of the nibble tables stage 1 writes
    bool xt_any = false;        // nibble tables for every G and plan mode (else up to 128 groups with shared plans)
    bool xt_bbar = false;       // nibble tables of XW - Bbar (identity head)
    int l1_nout = 1;            // outputs the l1 selection solves
    bool l1_binary = false;     // ... from the binary head's (sum p1, sum p0)
    int simt_R = 1, simt_C = 1; // score rows and outputs the CUDA-core kernel stages
    bool wide_pi = false;       // per-instance plans of 65..128 groups
    bool tc = false;            // tensor-core kernel
    int family = DKS_GENERAL_NONE;  // a model family whose every instance runs its own kernels: its DKS_GENERAL_* (tree
                                    // ensembles, kernel machines, MLPs, neighbour models, soft-voting ensembles of
                                    // those; own_kernel, dks.cu)
    bool mixture() const { return shared == HEAD_SHARED_MIX_BINARY || shared == HEAD_SHARED_MIX_CLASS; }
    bool own() const { return family != DKS_GENERAL_NONE; }
};

// Tables derived from the plan of the full varying set (M == G) that PlanDev does not hold: the class-sum heads' per-class
// Dm and row bounds (dks_multi.cuh), the exp head's l(s), the mixture members' tables.  Host-only; the buffers belong to
// plan_pool[M].
struct FullSetTables {
    int M;                              // the plan they were built for (0: none)
    const float* dm[DKS_MIX_MAX_R];     // per member ([0]: the head itself): binary Dm, or per-class Dm
    const double* dme[DKS_MIX_MAX_R];   // binary members: row exponents
    const float* lo[DKS_MIX_MAX_R];     // class sums: row bounds
    const double* ell;                  // exp head: l(s) = log2 sum_j w_j 2^(log2 e d(s, j)) [S_pad]
};

// number of instances a general kernel launch handles and the q-th of them
__device__ __forceinline__ int dks_inst_count(const ExplainParams& p) { return p.list ? *p.count : p.n; }
__device__ __forceinline__ int dks_inst_at(const ExplainParams& p, int q) { return p.list ? p.list[q] : q; }

// A context owns its device memory: DevBuf fields, fit_pool (what a dks_fit builds) and plan_pool[M] (the plan of M groups).
// A raw pointer field never owns: it points into one of those, or an ensemble member's status word into its ensemble's.
struct dks_ctx {
    ~dks_ctx() {
        if (gexec) cudaGraphExecDestroy(gexec);
        for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
        for (cudaEvent_t e : ev_l1) if (e) cudaEventDestroy(e);
        if (ev_fork) cudaEventDestroy(ev_fork);
        if (ev_join) cudaEventDestroy(ev_join);
        if (side_stream) cudaStreamDestroy(side_stream);
        if (own_stream && stream) cudaStreamDestroy(stream);
    }

    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int sm_count = 132;
    int max_smem_optin = 0;

    // problem definition
    int N = 0, D = 0, G = 0, R = 0, C = 0;
    int act = -1, link = DKS_LINK_IDENTITY, scalar_out = 0;
    double kappa = 1.0;
    bool fitted = false;
    int kernel_choice = DKS_KERNEL_AUTO;
    int nsamples_req = 0;
    bool uniform_w = true;      // background weights all equal
    DevBuf<float> dbg_T;        // debug dump of the tensor-core score tile of instance dbg_i ([dbg_rows][dbg_cols])
    int dbg_i = -1, dbg_rows = 0, dbg_cols = 0;
    DevBuf<float> dbg_time;     // [6][256] clock64 timeline of CTA 0 (debug kernel variant)

    // host copies
    MixHead mix = {};           // mixture head (act == DKS_ACT_MIX): members and weights
    DevBuf<MixHead> d_mix;      // its device copy (stage 1 and the fit kernels evaluate f(x) in float64 from it)
    DevBuf<double> d_mixBW;     // [K][N][G][R_m] the background contributions split per member (plan tables of each member)
    DevBuf<double> d_mixsc;     // [K][N][R_m] the background scores split per member
    DevBuf<float> d_mixscr;     // one member's sums before they are added, times pi_k, into the mixture's sums
    // tree ensemble (act == DKS_ACT_TREES): host copies of the node arrays, and their device copies built by dks_fit
    std::vector<int32_t> h_tfeat, h_tleft, h_tright, h_troots;
    std::vector<double> h_tthr, h_tval, h_tbase;
    std::vector<unsigned char> h_tmiss;
    TreeDev tree = {};
    DevBuf<unsigned char> txinfo;   // the explain kernel's node scratch tree.xinfo points at
    // the column encoding of a model with its own kernel (dks_set_column_encoding; empty h_ehdr: none), the device copy
    // dks_fit builds, the encoded background, the encoded group CSR and the encoded rows of the current call
    std::vector<int32_t> h_ehdr, h_eops;
    std::vector<double> h_eopv, h_etab;
    EncodingDev enc = {};
    double* d_bg_enc = nullptr;  // [N][E] (fit_pool)
    int32_t *d_egoff = nullptr, *d_egcols = nullptr;   // [G + 1], [E]: group g owns the encoded columns of its raw ones
    DevBuf<double> d_Xenc;       // [n][E]
    // what the family's own kernels of the current call read: the rows (d_Xenc, or the raw rows), their width, the
    // background and the group CSR over those columns
    const double* own_X = nullptr;
    int own_D = 0;
    const double* own_bg = nullptr;
    const int32_t *own_goff = nullptr, *own_gcols = nullptr;
    // kernel machine (act == DKS_ACT_KMACH): host copies of the arrays, and their device copies built by dks_fit
    std::vector<double> h_ksv, h_kdual, h_kcolw, h_kcolo;
    KmDev km = {};
    // multi-layer perceptron (act == DKS_ACT_MLP): host copies of the layers (natural, fragment-ordered, padded biases), and
    // their device copies built by dks_fit
    std::vector<double> h_mw, h_mb, h_mwf, h_mbp;
    MlpDev mlp = {};
    // k-nearest neighbours (act == DKS_ACT_KNN): host copies of the arrays, and their device copies built by dks_fit
    std::vector<double> h_nfitX, h_ncolw, h_ncolo, h_ny;
    KnnDev knn = {};
    // soft-voting ensemble (act == DKS_ACT_ENSEMBLE): the member contexts it owns, pi, its device copy (built by dks_fit), the
    // members' predictions of a call [K][n][C] and their weighted background means [n][C][S_cap]; a member points at its
    // ensemble, shares its stream and status word, and refuses every call of the C ABI
    std::vector<dks_ctx*> ens;
    std::vector<double> h_ens_pi;
    const double* d_ens_pi = nullptr;
    DevBuf<double> d_ens_out, d_ens_ey;
    dks_ctx* ens_parent = nullptr;
    // stacking ensemble (act == DKS_ACT_STACKING): its members in `ens` (owned as above); the final estimator's host copies
    // and its descriptor (stk.W / b / Wp built by dks_fit), the workspace budget of a call, the members' kept outputs of one
    // background chunk [n][F][j1 - j0][S_cap], the instances' passthrough table XWg [n][G][R] (stage 1), the background's
    // BWg [N][G][R] and BWtot [N][R] (dks_fit, fit_pool), and the chunks of the last call
    std::vector<double> h_stk_W, h_stk_b, h_stk_Wp;
    StackDev stk = {};
    int64_t stk_budget = 0;
    DevBuf<double> d_stk_ws, d_stk_XWg;
    const double* d_stk_BWg = nullptr;
    const double* d_stk_BWtot = nullptr;
    int stk_chunks = 0;
    // a module the caller runs (act == DKS_ACT_EXTERNAL, dks_set_external_model): the dtype of its input rows, its outputs on
    // the background in float64 (dks_set_external_background), the group of every column (d_ext_colgrp, fit_pool), the
    // outputs stage 1 reads while dks_external_prepare runs (the caller's memory), and the call dks_external_begin laid
    // out: its explain parameters, the plans it was given, the coalition offsets [n + 1] and their total (-1: none; also
    // the next stage 1 and dks_fit drop it), and ext_key below.  The background means ey go to d_ens_ey.
    int ext_in_f64 = 1;
    DevBuf<double> d_ext_bgy;
    const int32_t* d_ext_colgrp = nullptr;
    const void* ext_y = nullptr;
    int ext_y_f64 = 1;
    ExplainParams ext_p = {};
    const uint64_t* ext_call_z = nullptr;
    int ext_call_stride = 0;
    DevBuf<long long> d_ext_soff;
    long long ext_coalitions = -1;
    // every device array dks_fit builds that a by-value kernel struct points at (the pointers of tree, km, mlp, knn, enc, cm,
    // d_bg_enc, d_egoff, d_egcols, d_ens_pi), freed together by the next dks_fit or with the context.  No kernel reads one
    // after that: freeing clears fitted and prepared, and every launch needs them.
    DevPool fit_pool;
    std::vector<double> h_bg, h_wbg, h_W, h_b;
    std::vector<int32_t> h_cm_hdr;             // column maps (dks_set_column_maps); empty: the scores are W x + b
    std::vector<double> h_cm_keys, h_cm_vals;
    std::vector<int32_t> h_goff, h_gcols;

    // device, fit-time
    DevBuf<double> d_bg, d_wbg, d_W, d_b;
    ColumnMapsDev cm = {};                     // device copy of the column maps (cm.hdr == nullptr: none; fit_pool)
    DevBuf<int32_t> d_goff, d_gcols;
    DevBuf<double> d_colmin, d_colmax;
    DevBuf<int> d_colnan;
    DevBuf<double> d_BW, d_scores, d_Bbar, d_fnull, d_linkfnull;
    DevBuf<float> d_BWs, d_bases, d_wbf;
    DevBuf<float> d_wn;         // [N] N w_j in float: the background weights the weighted shared-plan kernels read
    HeadDesc head;
    std::vector<double> h_fnull, h_linkfnull;

    // plans
    PlanDev h_plans[DKS_MAX_GROUPS + 1];
    DevBuf<PlanDev> d_plans;
    DevPool plan_pool[DKS_MAX_GROUPS + 1];       // device buffers owned by the plan of each M (freed on replace)
    int max_plan_S = 0;
    // l1 feature selection (dks_set_l1 / dks_set_l1_tables): per-M tables on the device, and a device copy of the table
    // set (the general list's LARS reads each task's own M)
    dks::l1::Tables h_l1[DKS_MAX_GROUPS + 1] = {};
    DevBuf<dks::l1::Tables> d_l1;                // [DKS_L1_MAX_GROUPS + 1]
    int l1_mode = 0, l1_k = 0;
    uint64_t l1_sel[2] = {0, 0};                 // bit M - 1: instances with M varying groups select
    DevBuf<int> d_idx_sel;                       // [n] general-list instances whose M selects ...
    DevBuf<int> d_idx_plain;                     // [n] ... and the rest
    DevBuf<int> d_l1_counts;                     // [2] their counts
    cudaEvent_t ev_l1[3] = {nullptr, nullptr, nullptr};   // around the general list's moments kernel and LARS
    bool l1_timing_valid = false;
    FullSetTables full = {};     // tables of the plan of the full varying set, cleared with that plan
    DevBuf<double> d_mom;        // [n][outputs solved][2G + 4] per-instance moments of y
    DevBuf<double> d_yw;         // [n][S_pad] link-space y of the wide (more than 128 groups) solve
    DevBuf<double> d_betaw;      // [n][kpw] its coefficients before the delta term
    DevBuf<float> d_acache;      // [n][S_pad] A(i, s) of sixteen-word rows, shared by the launches of the background chunks
    // per-instance plans drawn on the device (plan_mode 1)
    int plan_mode = 0;
    uint64_t sampler_seed = 0;
    long long row_offset = 0;
    DksSamplingInfo h_sinfo[DKS_MAX_GROUPS + 1];
    DevBuf<DksSamplingInfo> d_sinfo;
    DevBuf<uint64_t> d_genz;     // [n][stride][gen_words]
    DevBuf<double> d_genw;       // [n][stride]
    DevBuf<double> d_genchol;
    DevBuf<double> d_genainv;
    int gen_words = 1;           // words per row d_genz is laid out for
    int gen_plan_words = 1;      // words per row of the last call's plans (dks_get_instance_plans_w)
    const double* h_afix[DKS_MAX_GROUPS + 1] = {};   // per M: normal matrix of the enumerated prefix (device pointers)
    DevBuf<const double*> d_afix;
    int gen_stride = 0, gen_n = 0;

    // per-call workspace
    int ws_n = 0, cur_n = 0;     // instances the workspace is laid out for (0: lay it out at the next call), and this call's
    bool prepared = false;
    DevBuf<double> d_X;          // staging for host inputs
    const double* cur_X = nullptr;
    DevBuf<double> d_XW;
    DevBuf<double> d_XT;         // [n][R][ceil(G/4)][16] nibble tables of the scaled grouped contributions (binary head:
                                 // R = 1; softmax: log2 e XW; identity head: XW - Bbar)
    DevBuf<float> d_msums;       // [n][C][S_pad] per-class sums of the softmax coalition kernel
    DevBuf<unsigned char> d_vflag;
    DevBuf<uint64_t> d_vmask;
    DevBuf<int> d_M;
    DevBuf<double> d_dlink;
    DevBuf<int> status;          // status[2], list counts[2], then the histogram of M [G + 1] (one allocation, one memset)
    int* d_status = nullptr;     // status, or an ensemble member's view of its ensemble's
    int* d_counts = nullptr;     // [0] instances on the shared fast path, [1] the others
    int* d_hist = nullptr;
    DevBuf<int> d_idx_full;      // [n] instances whose varying set is all G groups
    DevBuf<int> d_idx_other;     // [n] the rest
    DevBuf<float2> d_sums;       // [n][S_pad] (sum p1, sum p0) of the shared fast path
    DevBuf<long long> d_acc;     // [n][24] fixed-point partial beta of the fused kernel (zero between launches)
    DevBuf<double> d_phi;
    int phi_rows = 0;             // rows of the last dks_explain_host result held in d_phi
    PinnedBuf<double> h_phi_pin;  // pinned staging for results going to pageable host memory
    DevBuf<uint64_t> d_extz;
    DevBuf<double> d_extw;
    int h_status[2] = {0, 0};

    // CUDA graph of the device-resident explain sequence (dks_run_dev): captured on the second identical call
    struct GraphKey {
        const void* X; void* phi; int n, nsamples, kernel, plan_mode; long long row_offset; unsigned long long seed;
        unsigned epoch; cudaStream_t stream;
        bool operator==(const GraphKey& o) const {
            return X == o.X && phi == o.phi && n == o.n && nsamples == o.nsamples && kernel == o.kernel &&
                   plan_mode == o.plan_mode && row_offset == o.row_offset && seed == o.seed && epoch == o.epoch &&
                   stream == o.stream;
        }
    };
    bool graph_enabled = true;    // DKS_GRAPH=0 disables
    bool capturing = false;
    bool have_last_key = false;
    GraphKey last_key{}, graph_key{};
    GraphKey ext_key{};           // the rows, plans, options, epoch and stream dks_external_begin laid its call out for: the
                                  // steps after it refuse to run when anything of it changed since
    cudaGraphExec_t gexec = nullptr;
    unsigned epoch = 0;           // bumped by everything that changes what the sequence launches (fit, plans, ...)
    int64_t graph_launches = 0;
    int64_t graph_kernels = 0;    // kernels one replay of the captured graph launches

    // push all-gather over peer memory: after a device-resident explain, phi is stored into slab `peer_rank` of every
    // peer's gathered buffer (dks_set_peers)
    int peer_world = 0, peer_rank = 0;
    long long peer_slab = 0;                       // doubles per slab
    double* peer_base[16] = {};                    // device pointers to each rank's [world][slab] buffer
    unsigned long long* peer_flags[16] = {};       // rank r's flag array [world] (peer-mapped); [peer_rank] is this rank's own
    bool peer_flags_set = false;
    DevBuf<unsigned long long> d_step;             // device-side step counter of the flag exchange
    bool push_in_kernel = false;                   // 1: the fused route's finish kernel stores its phi rows into the peers'
                                                   // buffers itself (DESIGN.md §7)
    // tuning knobs (dks_set_option; defaults from the environment at dks_create: DKS_FUSED, DKS_FUSED_WARPS, ...)
    int opt_fused = 1, opt_fused_warps = 0, opt_fused_B = 0;
    int opt_fused_table = 1;                       // 0: the fused kernel ignores the plans' link tables (exact loop only)
    DevBuf<unsigned long long> d_ltab_fb;          // fused passes that fell back from the link table to the exact loop
    bool opt_graph_timing = false;   // keep the timing event records inside a captured graph (dks_last_timings after replays)
    bool timing_valid = false, last_was_graph = false;
    bool last_fused = false;                       // the last explain ran the fused shared-plan kernel
    int32_t last_path[DKS_PATH_FIELDS] = {};       // what the last explain launched (dks_last_path), recorded while enqueuing

    // the general kernel for the instances the shared-plan path does not take runs on a side stream, next to the fused kernel
    // (it is usually empty: a serialised empty launch cost 6 us per step)
    cudaStream_t side_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    int64_t launches = 0;
};
