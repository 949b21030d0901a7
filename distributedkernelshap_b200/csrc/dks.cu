// libdks.so -- host side of the C ABI declared in include/dks.h.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -shared -Xcompiler -fPIC (see build.py)
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <memory>

#include "dks_kernels.cuh"
#include "dks_tc.cuh"
#include "dks_shared.cuh"
#include "dks_fused.cuh"
#include "dks_l1.cuh"
#include "dks_mixture.cuh"
#include "dks_multi.cuh"
#include "dks_wide.cuh"
#include "dks_sampler.cuh"
#include "dks_instance_wide.cuh"
#include "dks_trees.cuh"
#include "dks_encode.cuh"
#include "dks_kmach.cuh"
#include "dks_mlp.cuh"
#include "dks_knn.cuh"
#include "dks_gauss.cuh"
#include "dks_ensemble.cuh"
#include "dks_external.cuh"
#include "dks_stacking.cuh"

namespace {

thread_local std::string g_last_error;

int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}

#define CUDA_TRY(expr)                                                                              \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess)                                                                      \
            return fail(DKS_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

#define REQUIRE(cond, ...)                                  \
    do {                                                    \
        if (!(cond)) return fail(DKS_ERR_INVALID, __VA_ARGS__); \
    } while (0)

inline int cdiv(long long a, int b) { return (int)((a + b - 1) / b); }

// drops the plan of one M (every M when M < 0) with everything derived from it -- its l1 tables, sampling info and
// full-set tables -- and brings the device copies the kernels read up to date
int drop_plans(dks_ctx* ctx, int M) {
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));       // nothing in flight may still read the buffers
    for (int m = 0; m <= DKS_MAX_GROUPS; ++m) {
        if (M >= 0 && m != M) continue;
        ctx->plan_pool[m].clear();
        ctx->h_plans[m] = PlanDev{};
        ctx->h_l1[m] = dks::l1::Tables{};
        ctx->h_afix[m] = nullptr;
        ctx->h_sinfo[m] = DksSamplingInfo{};
    }
    if (M < 0 || ctx->full.M == M) ctx->full = FullSetTables{};
    if (M < 0) ctx->max_plan_S = 0;
    ctx->epoch++;
    const cudaStream_t st = ctx->stream;
    CUDA_TRY(cudaMemcpyAsync(ctx->d_plans, ctx->h_plans, sizeof(ctx->h_plans), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_l1, ctx->h_l1, sizeof(dks::l1::Tables) * (DKS_L1_MAX_GROUPS + 1), cudaMemcpyHostToDevice,
                             st));
    if (ctx->d_sinfo) CUDA_TRY(cudaMemcpyAsync(ctx->d_sinfo, ctx->h_sinfo, sizeof(ctx->h_sinfo), cudaMemcpyHostToDevice, st));
    if (ctx->d_afix) CUDA_TRY(cudaMemcpyAsync(ctx->d_afix, ctx->h_afix, sizeof(ctx->h_afix), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return DKS_OK;
}

int bind(dks_ctx* ctx) {
    if (!ctx) return fail(DKS_ERR_INVALID, "null ctx");
    if (ctx->ens_parent)
        return fail(DKS_ERR_INVALID, "this context is a member of a soft-voting ensemble (dks_set_ensemble), which owns it");
    CUDA_TRY(cudaSetDevice(ctx->device));
    return DKS_OK;
}

#define BIND(ctx)                      \
    do {                               \
        int _rc = bind(ctx);           \
        if (_rc != DKS_OK) return _rc; \
    } while (0)

#define TRY(expr)                      \
    do {                               \
        int _rc = (expr);              \
        if (_rc != DKS_OK) return _rc; \
    } while (0)

int ensure_workspace(dks_ctx* ctx, int n) {
    if (n <= ctx->ws_n) return DKS_OK;
    const int G = ctx->G, R = ctx->R, C = ctx->C;
    CUDA_TRY(ctx->d_XW.alloc((size_t)n * G * R));
    CUDA_TRY(ctx->d_XT.alloc((size_t)n * R * ((G + 3) / 4) * 16));
    CUDA_TRY(ctx->d_vflag.alloc((size_t)n * G));
    CUDA_TRY(ctx->d_vmask.alloc((size_t)n));
    CUDA_TRY(ctx->d_M.alloc((size_t)n));
    CUDA_TRY(ctx->d_dlink.alloc((size_t)n * C));
    CUDA_TRY(ctx->d_idx_full.alloc((size_t)n));
    CUDA_TRY(ctx->d_idx_other.alloc((size_t)n));
    CUDA_TRY(ctx->d_idx_sel.alloc((size_t)n));
    CUDA_TRY(ctx->d_idx_plain.alloc((size_t)n));
    CUDA_TRY(ctx->d_acc.alloc((size_t)n * 16));
    CUDA_TRY(cudaMemsetAsync(ctx->d_acc, 0, sizeof(long long) * (size_t)n * 16, ctx->stream));   // the fused route's finish
                                                                                                  // kernel leaves it zeroed
    ctx->ws_n = n;
    ctx->epoch++;            // buffers moved: a captured graph holds the old addresses
    return DKS_OK;
}

// timing events: inside a stream capture they become external event-record nodes, so dks_last_timings keeps working
// for graph launches
cudaError_t record_ev(dks_ctx* ctx, int k) {
    if (ctx->capturing && !ctx->opt_graph_timing) {   // four event-record nodes cost a replayed graph several microseconds
        ctx->timing_valid = false;
        return cudaSuccess;
    }
    if (k == 0) ctx->timing_valid = true;
    return cudaEventRecordWithFlags(ctx->ev[k], ctx->stream, ctx->capturing ? cudaEventRecordExternal : cudaEventRecordDefault);
}

// persistent CTAs: as many per SM as shared memory holds (each also reserving `reserve` bytes), at most `max_per_sm`, and
// no more than there is work for
int persistent_grid(const dks_ctx* ctx, size_t smem, size_t reserve, int max_per_sm, long long work) {
    const int per_sm = std::min(std::max((int)((size_t)ctx->max_smem_optin / (smem + reserve)), 1), max_per_sm);
    return (int)std::min((long long)ctx->sm_count * per_sm, work);
}

// grows a per-call workspace buffer to at least `need` elements; a move changes the epoch (a captured graph holds the old
// address)
template <typename T>
int grow(dks_ctx* ctx, DevBuf<T>& buf, size_t need) {
    if (need <= buf.size()) return DKS_OK;
    CUDA_TRY(buf.alloc(need));
    ctx->epoch++;
    return DKS_OK;
}

// the head's capabilities, read by every dispatch decision (dks_fit: the head is fixed until the next fit)
HeadDesc describe_head(const dks_ctx* ctx) {
    HeadDesc h;
    switch (ctx->act) {
    case DKS_ACT_BINARY_LOGISTIC:
        h.shared = HEAD_SHARED_BINARY; h.shared_max_G = DKS_MAX_GROUPS; h.scale = -ctx->kappa * DKS_LOG2E;
        h.xt_any = true; h.l1_binary = true; h.wide_pi = true; h.tc = true;
        break;
    case DKS_ACT_SOFTMAX:
    case DKS_ACT_OVR:
        h.shared = HEAD_SHARED_CLASS_SUMS; h.ovr = ctx->act == DKS_ACT_OVR; h.scale = DKS_LOG2E;
        h.simt_R = ctx->R; h.simt_C = ctx->C;
        break;
    case DKS_ACT_IDENTITY:
        h.shared = HEAD_SHARED_TABLES; h.xt_bbar = true; h.wide_pi = true;
        break;
    case DKS_ACT_EXP:
        h.shared = HEAD_SHARED_TABLES; h.expo = true; h.scale = DKS_LOG2E; h.wide_pi = true;
        break;
    case DKS_ACT_MIX:
        // the tables are per member, member-major: -log2 e for binary members (the binary head's sign), log2 e else
        h.scale = DKS_LOG2E;
        if (ctx->mix.mact == DKS_ACT_BINARY_LOGISTIC) {
            h.shared = HEAD_SHARED_MIX_BINARY; h.l1_binary = true; h.xt_scale = -DKS_LOG2E;
        } else {
            h.shared = HEAD_SHARED_MIX_CLASS; h.ovr = ctx->mix.mact == DKS_ACT_OVR; h.xt_scale = DKS_LOG2E;
        }
        break;
    case DKS_ACT_TREES:
        // no shared-plan route: every instance runs the tree kernels; two outputs solve class 1 (class 0 its negation)
        h.family = DKS_GENERAL_TREES; h.l1_binary = ctx->C == 2;
        h.expo = ctx->tree.head == DKS_TREE_HEAD_EXP;
        break;
    case DKS_ACT_KMACH:
        // no shared-plan route: every instance runs the kernel-machine kernels; the calibrated head solves class 1 (class 0
        // its negation)
        h.family = DKS_GENERAL_KMACH; h.l1_binary = ctx->km.head == DKS_KM_HEAD_CALIBRATED;
        break;
    case DKS_ACT_MLP:
        // no shared-plan route: every instance runs the MLP kernels; the sigmoid head solves class 1 (class 0 its negation)
        h.family = DKS_GENERAL_MLP; h.l1_binary = ctx->mlp.head == DKS_MLP_HEAD_SIGMOID;
        break;
    case DKS_ACT_KNN:
        // no shared-plan route: every instance runs the neighbour kernels; every output is solved on its own (count / k
        // probabilities are not exact negations of each other in float64)
        h.family = DKS_GENERAL_KNN;
        break;
    case DKS_ACT_GAUSS:
        // no shared-plan route: every instance runs the Gaussian kernel; every output is solved on its own
        h.family = DKS_GENERAL_GAUSS;
        break;
    case DKS_ACT_ENSEMBLE:
        // no shared-plan route: every instance runs the members' kernels and the ensemble's tail; every output is solved on
        // its own
        h.family = DKS_GENERAL_ENSEMBLE;
        break;
    case DKS_ACT_STACKING:
        // no shared-plan route: every instance runs the members' kernels, the final estimator's reduction and the
        // ensemble's tail; every output is solved on its own
        h.family = DKS_GENERAL_STACKING;
        break;
    case DKS_ACT_EXTERNAL:
        // no shared-plan route: the caller's module evaluates the masked rows, every instance runs the ensemble's tail on
        // their background means; every output is solved on its own
        h.family = DKS_GENERAL_EXTERNAL;
        break;
    }
    if (h.shared != HEAD_SHARED_BINARY && !h.own()) h.shared_max_G = 128;
    if (!h.mixture()) h.xt_scale = h.scale;
    h.l1_nout = h.l1_binary ? 1 : ctx->C;
    return h;
}

// ---- the model families with their own kernels (tree ensembles, kernel machines, MLPs, neighbour models): what differs
// between them is here, keyed by HeadDesc::family.  Everything else treats them alike. --------------------------------

enum OwnRefuses {                       // the raw values a family's predict and explain kernels refuse (DKS_ERR_DOMAIN)
    REFUSES_NONE,                       // none: a tree sends NaN down the branch its node names
    REFUSES_NAN,
    REFUSES_NONFINITE,                  // NaN and the infinities
};

// a family (HeadDesc::family: its explain kernel's DKS_GENERAL_*) as the shared code sees it
struct OwnKernel {
    const char* family;      // "<family> run on the <kernel> only", "<family>: %d groups", "not for <family>"
    const char* kernel;
    const char* bound;       // "... nsamples, outputs or <bound> too many"
    const char* model;       // "<model>: the model reads %d columns", "<model>: link(fnull) of output %d ..."
    const char* maps_note;   // after "dks_set_column_maps: not for <family>"
    int refuses;             // OwnRefuses
    size_t (*smem)(const dks_ctx* ctx, int S_cap);   // the explain kernel's shared memory at S_cap coalition rows
};

// warps of explain_mlp_kernel that evaluate coalitions at S_cap rows: as many (up to 8) as shared memory holds, at least 1
int mlp_warps(const dks_ctx* ctx, int S_cap) {
    int nw = dks::mlp::WARPS;
    while (nw > 1 && dks::mlp::smem_bytes(S_cap, ctx->C, ctx->G, ctx->mlp, nw) > (size_t)ctx->max_smem_optin) --nw;
    return nw;
}

// coalitions per chunk of explain_knn_kernel at S_cap rows: as many neighbour lists as the opt-in shared memory holds next
// to the sums and the tables, at most S_cap and at least 1
int knn_chunk(const dks_ctx* ctx, int S_cap) {
    const size_t fixed = dks::knn::smem_bytes(S_cap, ctx->C, ctx->G, ctx->knn.k, 0);
    const size_t per = (sizeof(double) + sizeof(int)) * (size_t)ctx->knn.k;
    const long long room = (long long)ctx->max_smem_optin - (long long)fixed;
    return (int)std::max(1LL, std::min((long long)S_cap, room / (long long)per));
}

OwnKernel own_kernel(int family);

// shared memory of the widest launch of a soft-voting or stacking ensemble at S_cap rows: a member's explain kernel or the
// tail (stacking_reduce_kernel's is static and smaller)
size_t ensemble_smem(const dks_ctx* ctx, int S_cap) {
    size_t smem = dks::ens::tail_smem_bytes(S_cap, ctx->C);
    for (const dks_ctx* m : ctx->ens) smem = std::max(smem, own_kernel(m->head.family).smem(m, S_cap));
    return smem;
}

OwnKernel own_kernel(int family) {
    switch (family) {
    case DKS_GENERAL_TREES:
        return {"tree ensembles", "tree kernel", "trees", "tree ensemble", "", REFUSES_NONE,
                [](const dks_ctx* c, int S_cap) { return dks::trees::smem_bytes(S_cap, c->C, c->tree.R, c->tree.T); }};
    case DKS_GENERAL_KMACH:
        return {"kernel machines", "kernel-machine kernel", "groups", "kernel machine",
                " (their scalers fold into the support vectors and column weights)", REFUSES_NAN,
                [](const dks_ctx* c, int S_cap) {
                    if (c->km.head == DKS_KM_HEAD_OVO) return dks::kmach::ovo_smem_bytes(S_cap, c->C, c->km.R, c->G);
                    return dks::kmach::smem_bytes(S_cap, c->C, c->km.R, c->G, c->km.head == DKS_KM_HEAD_CALIBRATED); }};
    case DKS_GENERAL_MLP:
        return {"MLPs", "MLP kernel", "hidden units", "MLP", " (their scalers fold into the first layer)",
                REFUSES_NONFINITE,
                [](const dks_ctx* c, int S_cap) {
                    return dks::mlp::smem_bytes(S_cap, c->C, c->G, c->mlp, mlp_warps(c, S_cap)); }};
    case DKS_GENERAL_KNN:
        return {"nearest-neighbour models", "neighbour kernel", "neighbours", "nearest-neighbour model",
                " (their scalers fold into the column weights and origins)", REFUSES_NONFINITE,
                [](const dks_ctx* c, int S_cap) {
                    return dks::knn::smem_bytes(S_cap, c->C, c->G, c->knn.k, knn_chunk(c, S_cap)); }};
    case DKS_GENERAL_GAUSS:
        return {"Gaussian models", "Gaussian kernel", "components", "Gaussian model",
                " (their scalers fold into the means and projections)", REFUSES_NONFINITE,
                [](const dks_ctx* c, int S_cap) { return dks::gauss::smem_bytes(S_cap, c->C, c->G, c->gauss.K); }};
    case DKS_GENERAL_ENSEMBLE:          // refuses: what its members refuse (refusing_kernel)
        return {"soft-voting ensembles", "ensemble kernels", "groups", "soft-voting ensemble",
                " (put the preprocessing in front of the ensemble)", REFUSES_NONE, ensemble_smem};
    case DKS_GENERAL_STACKING:          // refuses: what its members refuse (refusing_kernel)
        return {"stacking ensembles", "stacking kernels", "groups", "stacking ensemble",
                " (put the preprocessing in front of the ensemble)", REFUSES_NONE, ensemble_smem};
    case DKS_GENERAL_EXTERNAL:          // refuses: nothing (the module sees every raw value)
        return {"modules", "module route", "nsamples", "module", " (put the preprocessing inside the module)", REFUSES_NONE,
                [](const dks_ctx* c, int S_cap) { return dks::ens::tail_smem_bytes(S_cap, c->C); }};
    }
    return {};                          // a linear head
}

// the family whose refusal of raw values applies: the ensemble member that refuses the most (the first of them), else the
// model's own
OwnKernel refusing_kernel(const dks_ctx* ctx) {
    OwnKernel ok = own_kernel(ctx->head.family);
    if (ctx->head.family != DKS_GENERAL_ENSEMBLE && ctx->head.family != DKS_GENERAL_STACKING) return ok;
    for (const dks_ctx* m : ctx->ens) {
        const OwnKernel mk = own_kernel(m->head.family);
        if (mk.refuses > ok.refuses) ok = mk;
    }
    return ok;
}

// runs a launch function of ensemble member m: its kernel launches count as the ensemble's, and a workspace it moved changes
// the ensemble's epoch (a captured graph holds the old address)
template <typename F>
int on_member(dks_ctx* ctx, dks_ctx* m, F&& launch) {
    const int64_t launches = m->launches;
    const unsigned epoch = m->epoch;
    const int rc = launch();
    ctx->launches += m->launches - launches;
    if (m->epoch != epoch) ctx->epoch++;
    return rc;
}

// the end of a family's dks_set_*: its head, and the linear part stage 1 evaluates while it decides the varying groups --
// one zero score row, no column maps
int set_own_model(dks_ctx* ctx, int act, int C, int scalar_out) {
    ctx->R = 1; ctx->C = C; ctx->act = act; ctx->kappa = 1.0; ctx->scalar_out = scalar_out;
    ctx->h_cm_hdr.clear(); ctx->h_cm_keys.clear(); ctx->h_cm_vals.clear();
    ctx->h_W.assign((size_t)ctx->D, 0.0);
    ctx->h_b.assign(1, 0.0);
    ctx->fitted = false;
    return DKS_OK;
}

bool all_finite(const double* a, size_t n) {
    for (size_t e = 0; e < n; ++e)
        if (!std::isfinite(a[e])) return false;
    return true;
}

// encoded columns of the column encoding set by dks_set_column_encoding (0: none)
int encoded_columns(const dks_ctx* ctx) { return (int)(ctx->h_ehdr.size() / 3); }
// columns a model with its own kernel reads: the encoded ones behind a column encoding, else the raw ones
int model_columns(const dks_ctx* ctx) { return encoded_columns(ctx) > 0 ? encoded_columns(ctx) : ctx->D; }

// the group of every column the model reads: each raw column's, or behind a column encoding each encoded column's raw
// source's
std::vector<int32_t> column_groups(const dks_ctx* ctx) {
    std::vector<int32_t> colgrp(ctx->D, 0);
    for (int g = 0; g < ctx->G; ++g)
        for (int c = ctx->h_goff[g]; c < ctx->h_goff[g + 1]; ++c) colgrp[ctx->h_gcols[c]] = g;
    const int E = encoded_columns(ctx);
    if (E == 0) return colgrp;
    std::vector<int32_t> enc(E);
    for (int e = 0; e < E; ++e) enc[e] = colgrp[ctx->h_ehdr[3 * e]];
    return enc;
}

// dks_fit: the columns the model reads against those the background gives (behind a column encoding: the encoded ones,
// whose sources must be raw columns of the background, which dks_set_background may have changed since)
int check_own_columns(const dks_ctx* ctx, const OwnKernel& ok) {
    const int E = encoded_columns(ctx), width = model_columns(ctx);
    for (int e = 0; e < E; ++e)
        if (ctx->h_ehdr[3 * e] >= ctx->D)
            return fail(DKS_ERR_UNSUPPORTED, "column encoding: encoded column %d reads raw column %d of %d", e,
                        ctx->h_ehdr[3 * e], ctx->D);
    int reads;
    switch (ctx->head.family) {
    case DKS_GENERAL_TREES:
        for (int32_t f : ctx->h_tfeat)
            if (f >= width)
                return fail(DKS_ERR_UNSUPPORTED, "tree ensemble: a split reads column %d of %d %s", f, width,
                            E > 0 ? "encoded columns" : "columns");
        return DKS_OK;
    case DKS_GENERAL_KMACH:
        if (ctx->km.kernel == DKS_KM_KERNEL_PROGRAM) {
            if (ctx->kprog.n == 0)
                return fail(DKS_ERR_INVALID, "kernel machine: the program kernel needs dks_set_kernel_program before dks_fit");
            reads = (int)(ctx->h_kpcolw.size() / ctx->kprog.L);
            break;
        }
        reads = (int)(ctx->h_kcolw.size() / ctx->km.K);
        break;
    case DKS_GENERAL_MLP: reads = ctx->mlp.width[0]; break;
    case DKS_GENERAL_GAUSS: reads = (int)(ctx->h_gmu.size() / ctx->gauss.K); break;
    case DKS_GENERAL_ENSEMBLE: return DKS_OK;         // each member checks its own (fit_members)
    case DKS_GENERAL_STACKING:                        // each member checks its own; the passthrough reads every column
        if (!ctx->h_stk_Wp.empty() && ctx->h_stk_Wp.size() != (size_t)ctx->stk.R * width)
            return fail(DKS_ERR_UNSUPPORTED, "%s: the passthrough reads %d columns, %s %d", ok.model,
                        (int)(ctx->h_stk_Wp.size() / ctx->stk.R), E > 0 ? "the column encoding gives" : "the background has",
                        width);
        return DKS_OK;
    case DKS_GENERAL_EXTERNAL:                        // the module reads the raw rows: the caller checked its width
        if (E > 0)
            return fail(DKS_ERR_UNSUPPORTED, "module: a column encoding is not supported (put the preprocessing inside the "
                        "module)");
        return DKS_OK;
    default: reads = (int)ctx->h_ncolw.size(); break;
    }
    if (reads != width)
        return fail(DKS_ERR_UNSUPPORTED, "%s: the model reads %d columns, %s %d", ok.model, reads,
                    E > 0 ? "the column encoding gives" : "the background has", width);
    return DKS_OK;
}

// dks_fit: the family's arrays on the device and its tables over the background bg [N][width] (encoded behind a column
// encoding) -- a tree's node arrays and every background row's direction at every node; a kernel machine's T[j][v] of
// every background row and support vector; an MLP's B[j] = b_0 + bg_j W_0; a neighbour model's T[j][v] and equality masks
// E[j][v] of every background row and training row
int own_fit_tables(dks_ctx* ctx, const double* bg, int width) {
    const int N = ctx->N;
    DevPool& pool = ctx->fit_pool;
    const cudaStream_t st = ctx->stream;
    switch (ctx->head.family) {
    case DKS_GENERAL_TREES: {
        TreeDev& t = ctx->tree;
        const size_t nodes = (size_t)t.nodes;
        const std::vector<int32_t> colgrp = column_groups(ctx);
        CUDA_TRY(pool.upload(&t.feat, ctx->h_tfeat.data(), nodes, st));
        CUDA_TRY(pool.upload(&t.thr, ctx->h_tthr.data(), nodes, st));
        CUDA_TRY(pool.upload(&t.left, ctx->h_tleft.data(), nodes, st));
        CUDA_TRY(pool.upload(&t.right, ctx->h_tright.data(), nodes, st));
        CUDA_TRY(pool.upload(&t.miss, ctx->h_tmiss.data(), nodes, st));
        CUDA_TRY(pool.upload(&t.val, ctx->h_tval.data(), nodes * t.R, st));
        CUDA_TRY(pool.upload(&t.roots, ctx->h_troots.data(), (size_t)t.T, st));
        CUDA_TRY(pool.upload(&t.base, ctx->h_tbase.data(), (size_t)t.R, st));
        CUDA_TRY(pool.upload(&t.colgrp, colgrp.data(), colgrp.size(), st));
        unsigned char* bgdir;
        CUDA_TRY(pool.alloc(&bgdir, (size_t)N * nodes));
        t.bgdir = bgdir;
        dks::trees::tree_bgdir_kernel<<<cdiv((long long)N * nodes, 256), 256, 0, st>>>(bg, N, width, t, bgdir);
        break;
    }
    case DKS_GENERAL_KMACH: {
        KmDev& k = ctx->km;
        const bool prog = k.kernel == DKS_KM_KERNEL_PROGRAM;
        CUDA_TRY(pool.upload(&k.sv, ctx->h_ksv.data(), ctx->h_ksv.size(), st));
        CUDA_TRY(pool.upload(&k.dual, ctx->h_kdual.data(), ctx->h_kdual.size(), st));
        const std::vector<double>& colw = prog ? ctx->h_kpcolw : ctx->h_kcolw;
        const std::vector<double>& colo = prog ? ctx->h_kpcolo : ctx->h_kcolo;
        CUDA_TRY(pool.upload(&k.colw, colw.data(), colw.size(), st));
        CUDA_TRY(pool.upload(&k.colo, colo.data(), colo.size(), st));
        double* Tbg;
        if (prog) {                 // T[j][v][l] of every statistic
            const long long n = (long long)N * k.n_sv * ctx->kprog.L;
            CUDA_TRY(pool.alloc(&Tbg, (size_t)n));
            k.Tbg = Tbg;
            dks::kmach::km_prog_fit_table_kernel<<<cdiv(n, 256), 256, 0, st>>>(bg, N, width, k, ctx->kprog, Tbg);
            break;
        }
        if (k.head == DKS_KM_HEAD_OVO) {   // the one-vs-one head's class blocks, pair intercepts and calibrations
            KmOvo& ov = ctx->kovo;
            CUDA_TRY(pool.upload(&ov.cls_off, ctx->h_kocls.data(), ctx->h_kocls.size(), st));
            CUDA_TRY(pool.upload(&ov.icpt, ctx->h_koicpt.data(), ctx->h_koicpt.size(), st));
            CUDA_TRY(pool.upload(&ov.cal_a, ctx->h_kocala.data(), ctx->h_kocala.size(), st));
            CUDA_TRY(pool.upload(&ov.cal_b, ctx->h_kocalb.data(), ctx->h_kocalb.size(), st));
        }
        CUDA_TRY(pool.alloc(&Tbg, (size_t)N * k.n_sv));
        k.Tbg = Tbg;
        dks::kmach::km_fit_table_kernel<<<cdiv((long long)N * k.n_sv, 256), 256, 0, st>>>(bg, N, width, k, Tbg);
        break;
    }
    case DKS_GENERAL_MLP: {
        MlpDev& m = ctx->mlp;
        CUDA_TRY(pool.upload(&m.W, ctx->h_mw.data(), ctx->h_mw.size(), st));
        CUDA_TRY(pool.upload(&m.b, ctx->h_mb.data(), ctx->h_mb.size(), st));
        CUDA_TRY(pool.upload(&m.Wf, ctx->h_mwf.data(), ctx->h_mwf.size(), st));
        CUDA_TRY(pool.upload(&m.bp, ctx->h_mbp.data(), ctx->h_mbp.size(), st));
        double* Bbg;
        CUDA_TRY(pool.alloc(&Bbg, (size_t)N * m.width[1]));
        m.Bbg = Bbg;
        dks::mlp::mlp_fit_table_kernel<<<cdiv((long long)N * m.width[1], 256), 256, 0, st>>>(bg, N, width, m, Bbg);
        break;
    }
    case DKS_GENERAL_KNN: {
        KnnDev& k = ctx->knn;
        const std::vector<int32_t> colgrp = column_groups(ctx);
        CUDA_TRY(pool.upload(&k.fitX, ctx->h_nfitX.data(), ctx->h_nfitX.size(), st));
        CUDA_TRY(pool.upload(&k.colw, ctx->h_ncolw.data(), ctx->h_ncolw.size(), st));
        CUDA_TRY(pool.upload(&k.colo, ctx->h_ncolo.data(), ctx->h_ncolo.size(), st));
        CUDA_TRY(pool.upload(&k.y, ctx->h_ny.data(), ctx->h_ny.size(), st));
        CUDA_TRY(pool.upload(&k.colgrp, colgrp.data(), colgrp.size(), st));
        double* Tbg;
        uint64_t* Ebg;
        CUDA_TRY(pool.alloc(&Tbg, (size_t)N * k.n_fit));
        CUDA_TRY(pool.alloc(&Ebg, (size_t)N * k.n_fit));
        k.Tbg = Tbg;
        k.Ebg = Ebg;
        dks::knn::knn_fit_table_kernel<<<cdiv((long long)N * k.n_fit, 256), 256, 0, ctx->stream>>>(bg, N, width, ctx->G, k,
                                                                                                     Tbg, Ebg);
        break;
    }
    case DKS_GENERAL_GAUSS: {
        GaussDev& g = ctx->gauss;
        const bool enc = ctx->enc.E > 0;
        CUDA_TRY(pool.upload(&g.mu, ctx->h_gmu.data(), ctx->h_gmu.size(), st));
        CUDA_TRY(pool.upload(&g.L, ctx->h_gL.data(), ctx->h_gL.size(), st));
        double *Abg, *alpha, *Pbg;
        CUDA_TRY(pool.alloc(&Abg, (size_t)N * g.RT));
        CUDA_TRY(pool.alloc(&alpha, (size_t)N * g.K));
        CUDA_TRY(pool.alloc(&Pbg, (size_t)N * ctx->G * g.RT));
        g.Abg = Abg; g.alpha = alpha; g.Pbg = Pbg;
        dks::gauss::gauss_fit_tables_kernel<<<cdiv((long long)N * g.K, 128), 128, 0, st>>>(
            bg, N, width, ctx->G, enc ? ctx->d_egoff : ctx->d_goff.get(), enc ? ctx->d_egcols : ctx->d_gcols.get(), g, Abg,
            alpha, Pbg);
        break;
    }
    }
    ctx->launches += 1;
    return DKS_OK;
}

// out [n][E] = the column encoding of the raw rows X_dev [n][D] (grid-stride): encode_kernel for a family that refuses no
// raw value, encode_finite_kernel (raw infinities refused) for the others, which sum over columns
int launch_encode(dks_ctx* ctx, const double* X_dev, int n, double* out) {
    const long long total = (long long)n * ctx->enc.E;
    const int grid = (int)std::min<long long>(cdiv(total, 256), (long long)ctx->sm_count * 8);
    auto kern = refusing_kernel(ctx).refuses == REFUSES_NONE ? dks::enc::encode_kernel : dks::enc::encode_finite_kernel;
    kern<<<grid, 256, 0, ctx->stream>>>(X_dev, n, ctx->D, ctx->enc, out, ctx->d_status);
    ctx->launches += 1;
    CUDA_TRY(cudaGetLastError());
    return DKS_OK;
}

// the family's predict kernel over n rows: out [n][C] = f(x) and dlink [n][C] = link(f(x)) - linkfnull, each when not NULL;
// a refused row and a non-finite dlink are reported in the status word.  X holds the rows the model reads or, given Xenc,
// raw rows [n][D] that the column encoding first writes to Xenc [n][E].
int launch_own_predict(dks_ctx* ctx, const double* X, int n, double* Xenc, const double* linkfnull, double* out,
                       double* dlink) {
    if (Xenc) {
        TRY(launch_encode(ctx, X, n, Xenc));
        X = Xenc;
    }
    const int D = ctx->enc.E > 0 ? ctx->enc.E : ctx->D, C = ctx->C, link = ctx->link;
    const cudaStream_t st = ctx->stream;
    switch (ctx->head.family) {
    case DKS_GENERAL_TREES:
        dks::trees::tree_predict_kernel<<<cdiv(n, 128), 128, 0, st>>>(X, n, D, ctx->tree, C, link, linkfnull, out, dlink,
                                                                      ctx->d_status);
        break;
    case DKS_GENERAL_KMACH:
        if (ctx->km.head == DKS_KM_HEAD_OVO)
            dks::kmach::km_ovo_predict_kernel<<<cdiv(n, 128), 128, 0, st>>>(X, n, D, ctx->km, ctx->kovo, C, link, linkfnull,
                                                                            out, dlink, ctx->d_status);
        else if (ctx->km.kernel == DKS_KM_KERNEL_PROGRAM)
            dks::kmach::km_prog_predict_kernel<<<cdiv(n, 128), 128, 0, st>>>(X, n, D, ctx->km, ctx->kprog, C, link,
                                                                             linkfnull, out, dlink, ctx->d_status);
        else
            dks::kmach::km_predict_kernel<<<cdiv(n, 128), 128, 0, st>>>(X, n, D, ctx->km, C, link, linkfnull, out, dlink,
                                                                        ctx->d_status);
        break;
    case DKS_GENERAL_MLP:           // one row per CTA, grid-stride
        dks::mlp::mlp_predict_kernel<<<std::max(1, std::min(n, ctx->sm_count * 8)), dks::mlp::THREADS, 0, st>>>(
            X, n, D, ctx->mlp, C, link, linkfnull, out, dlink, ctx->d_status);
        break;
    case DKS_GENERAL_KNN:
        dks::knn::knn_predict_kernel<<<cdiv(n, 128), 128, 0, st>>>(X, n, D, ctx->knn, C, link, linkfnull, out, dlink,
                                                                   ctx->d_status);
        break;
    case DKS_GENERAL_GAUSS:
        dks::gauss::gauss_predict_kernel<<<cdiv(n, 128), 128, 0, st>>>(X, n, D, ctx->gauss, C, link, linkfnull, out, dlink,
                                                                       ctx->d_status);
        break;
    case DKS_GENERAL_ENSEMBLE: {    // every member's f_k(x) into d_ens_out [K][n][C], then f(x) = sum_k pi_k f_k(x)
        const int K = (int)ctx->ens.size();
        TRY(grow(ctx, ctx->d_ens_out, (size_t)K * n * C));
        for (int k = 0; k < K; ++k) {
            dks_ctx* m = ctx->ens[k];
            double* outk = ctx->d_ens_out + (size_t)k * n * C;
            TRY(on_member(ctx, m, [&] { return launch_own_predict(m, X, n, nullptr, nullptr, outk, nullptr); }));
        }
        dks::ens::ensemble_predict_kernel<<<cdiv(n, 128), 128, 0, st>>>(ctx->d_ens_out, K, ctx->d_ens_pi, n, C, link,
                                                                        linkfnull, out, dlink, ctx->d_status);
        break;
    }
    case DKS_GENERAL_STACKING: {    // every member's outputs into d_ens_out [K][n][C_k], then the final estimator
        const int K = (int)ctx->ens.size();
        size_t width = 0;
        for (const dks_ctx* m : ctx->ens) width += (size_t)m->C;
        TRY(grow(ctx, ctx->d_ens_out, width * n));
        double* outk = ctx->d_ens_out;
        for (int k = 0; k < K; ++k) {
            dks_ctx* m = ctx->ens[k];
            TRY(on_member(ctx, m, [&] { return launch_own_predict(m, X, n, nullptr, nullptr, outk, nullptr); }));
            outk += (size_t)n * m->C;
        }
        dks::stack::stacking_predict_kernel<<<cdiv(n, 128), 128, 0, st>>>(ctx->d_ens_out, ctx->stk, X, n, link, linkfnull,
                                                                          out, dlink, ctx->d_status);
        break;
    }
    case DKS_GENERAL_EXTERNAL:      // the module's outputs on these rows, which the caller handed to dks_external_prepare
        if (ctx->ext_y == nullptr)
            return fail(DKS_ERR_UNSUPPORTED, "module: the engine cannot run a module; run it on the rows and hand its outputs "
                        "to dks_external_prepare, then explain with dks_external_begin / _mask / _reduce / _finish");
        dks::ext::external_load_kernel<<<cdiv(n, 128), 128, 0, st>>>(ctx->ext_y, ctx->ext_y_f64, n, C, link, linkfnull, out,
                                                                     dlink, ctx->d_status);
        break;
    }
    ctx->launches += 1;
    return DKS_OK;
}

// explain_ensemble_tail_kernel over p.list on the background means ey [n][C][S_cap] (L1: the moments of y; complement: the
// logit's 1 - ey_c taken per output, for outputs that need not sum to one)
int launch_tail(dks_ctx* ctx, bool l1, const ExplainParams& p, const dks::SimtL1& q, const double* ey, bool complement,
                cudaStream_t st) {
    const size_t tsm = dks::ens::tail_smem_bytes(p.S_cap, ctx->C);
    auto kern = l1 ? dks::ens::explain_ensemble_tail_kernel<true> : dks::ens::explain_ensemble_tail_kernel<false>;
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tsm));
    kern<<<persistent_grid(ctx, tsm, 1024, 8, ctx->cur_n), dks::ens::THREADS, tsm, st>>>(p, q, ey, complement ? 1 : 0);
    return DKS_OK;
}

int launch_stacking(dks_ctx* ctx, bool l1, const ExplainParams& p, cudaStream_t st);

// the family's explain kernel over p.list (L1: its moments; ea.ey set: a soft-voting ensemble's member adding into its
// workspace, the ACC instantiation; er.ws set: a stacking ensemble's member storing its outputs of every masked row, the
// ROWS instantiation); the tree kernel's per-CTA node scratch is sized for the grid.  A soft-voting ensemble: its members
// in order, then its tail; a stacking ensemble: launch_stacking.
int launch_own_kernel(dks_ctx* ctx, bool l1, const ExplainParams& p, size_t smem, cudaStream_t st,
                      const dks::EnsAcc& ea = dks::EnsAcc{}, const dks::EnsRows& er = dks::EnsRows{}) {
    const int grid = persistent_grid(ctx, smem, 1024, 8, ctx->cur_n);
    const dks::SimtL1 q = l1 ? dks::SimtL1{ctx->d_l1, ctx->d_mom} : dks::SimtL1{};
    const bool acc = ea.ey != nullptr, rows = er.ws != nullptr;
    switch (ctx->head.family) {
    case DKS_GENERAL_TREES: {
        TRY(grow(ctx, ctx->txinfo, (size_t)grid * ctx->tree.nodes));
        ctx->tree.xinfo = ctx->txinfo;
        auto kern = rows ? dks::trees::explain_tree_kernel<false, true, true>
                    : acc ? dks::trees::explain_tree_kernel<false, true>
                    : l1 ? dks::trees::explain_tree_kernel<true> : dks::trees::explain_tree_kernel<false>;
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, dks::trees::THREADS, smem, st>>>(p, q, ctx->tree, ctx->own_X, ctx->own_D, ea, er);
        break;
    }
    case DKS_GENERAL_KMACH: {
        if (ctx->km.head == DKS_KM_HEAD_OVO) {
            auto kern = rows ? dks::kmach::explain_kmach_ovo_kernel<false, true, true>
                        : acc ? dks::kmach::explain_kmach_ovo_kernel<false, true>
                        : l1 ? dks::kmach::explain_kmach_ovo_kernel<true> : dks::kmach::explain_kmach_ovo_kernel<false>;
            CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kern<<<grid, dks::kmach::THREADS, smem, st>>>(p, q, ctx->km, ctx->kovo, ctx->own_X, ctx->own_bg, ctx->own_D,
                                                          ctx->own_goff, ctx->own_gcols, ea, er);
            break;
        }
        auto kern = ctx->km.kernel == DKS_KM_KERNEL_PROGRAM
                    ? (rows ? dks::kmach::explain_kmach_kernel<false, true, true, true>
                       : acc ? dks::kmach::explain_kmach_kernel<false, true, false, true>
                       : l1 ? dks::kmach::explain_kmach_kernel<true, false, false, true>
                            : dks::kmach::explain_kmach_kernel<false, false, false, true>)
                    : rows ? dks::kmach::explain_kmach_kernel<false, true, true>
                    : acc ? dks::kmach::explain_kmach_kernel<false, true>
                    : l1 ? dks::kmach::explain_kmach_kernel<true> : dks::kmach::explain_kmach_kernel<false>;
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, dks::kmach::THREADS, smem, st>>>(p, q, ctx->km, ctx->own_X, ctx->own_bg, ctx->own_D, ctx->own_goff,
                                                      ctx->own_gcols, ea, er, ctx->kprog);
        break;
    }
    case DKS_GENERAL_MLP: {
        auto kern = rows ? dks::mlp::explain_mlp_kernel<false, true, true>
                    : acc ? dks::mlp::explain_mlp_kernel<false, true>
                    : l1 ? dks::mlp::explain_mlp_kernel<true> : dks::mlp::explain_mlp_kernel<false>;
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, dks::mlp::THREADS, smem, st>>>(p, q, ctx->mlp, mlp_warps(ctx, p.S_cap), ctx->own_X, ctx->own_bg,
                                                    ctx->own_D, ctx->own_goff, ctx->own_gcols, ea, er);
        break;
    }
    case DKS_GENERAL_KNN: {
        auto kern = rows ? dks::knn::explain_knn_kernel<false, true, true>
                    : acc ? dks::knn::explain_knn_kernel<false, true>
                    : l1 ? dks::knn::explain_knn_kernel<true> : dks::knn::explain_knn_kernel<false>;
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, dks::knn::THREADS, smem, st>>>(p, q, ctx->knn, knn_chunk(ctx, p.S_cap), ctx->own_X, ctx->own_bg,
                                                    ctx->own_D, ctx->own_goff, ctx->own_gcols, ea, er);
        break;
    }
    case DKS_GENERAL_GAUSS: {       // never an ensemble member (check_members)
        TRY(grow(ctx, ctx->gxp, (size_t)grid * ctx->G * ctx->gauss.RT));
        ctx->gauss.xp = ctx->gxp;
        auto kern = l1 ? dks::gauss::explain_gauss_kernel<true> : dks::gauss::explain_gauss_kernel<false>;
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, dks::gauss::THREADS, smem, st>>>(p, q, ctx->gauss, ctx->own_X, ctx->own_D, ctx->own_goff,
                                                      ctx->own_gcols);
        break;
    }
    case DKS_GENERAL_ENSEMBLE: {
        TRY(grow(ctx, ctx->d_ens_ey, (size_t)ctx->cur_n * ctx->C * p.S_cap));
        for (size_t k = 0; k < ctx->ens.size(); ++k) {
            dks_ctx* m = ctx->ens[k];
            m->cur_n = ctx->cur_n;                  // the rows, background and group CSR of this call
            m->own_X = ctx->own_X; m->own_D = ctx->own_D; m->own_bg = ctx->own_bg;
            m->own_goff = ctx->own_goff; m->own_gcols = ctx->own_gcols;
            const size_t msm = own_kernel(m->head.family).smem(m, p.S_cap);
            const dks::EnsAcc mea{ctx->d_ens_ey, ctx->h_ens_pi[k], k == 0 ? 1 : 0};
            TRY(on_member(ctx, m, [&] { return launch_own_kernel(m, false, p, msm, st, mea); }));
        }
        TRY(launch_tail(ctx, l1, p, q, ctx->d_ens_ey, false, st));
        break;
    }
    case DKS_GENERAL_STACKING:
        TRY(launch_stacking(ctx, l1, p, st));
        break;
    case DKS_GENERAL_EXTERNAL:      // ey from dks_external_reduce; a module's outputs need not sum to one
        TRY(launch_tail(ctx, l1, p, q, ctx->d_ens_ey, true, st));
        break;
    }
    ctx->launches += 1;
    return DKS_OK;
}

// a stacking ensemble's explain over p.list: the background in the fewest chunks [j0, j1) whose members' outputs
// [n][F][j1 - j0][S_cap] fit the workspace budget (at least one row each); per chunk the members' ROWS kernels in order and
// stacking_reduce_kernel, whose chain of ey continues across chunks; then the tail (an identity head's outputs need not sum
// to one: the logit's 1 - ey_c is taken per output).  chunks (K + 1) + 1 launches.
int launch_stacking(dks_ctx* ctx, bool l1, const ExplainParams& p, cudaStream_t st) {
    const int n = ctx->cur_n, N = ctx->N, F = ctx->stk.F;
    const size_t per_row = sizeof(double) * (size_t)F * n * p.S_cap;
    const int width = (int)std::max<long long>(1, std::min<long long>(N, ctx->stk_budget / (long long)per_row));
    TRY(grow(ctx, ctx->d_stk_ws, (size_t)F * n * width * p.S_cap));
    TRY(grow(ctx, ctx->d_ens_ey, (size_t)n * ctx->C * p.S_cap));
    const double* XWg = ctx->stk.Wp != nullptr ? ctx->d_stk_XWg.get() : nullptr;
    int chunks = 0;
    for (int j0 = 0; j0 < N; j0 += width, ++chunks) {
        const int j1 = std::min(N, j0 + width);
        for (size_t k = 0, f0 = 0; k < ctx->ens.size(); f0 += ctx->stk.ccount[k], ++k) {
            dks_ctx* m = ctx->ens[k];
            m->cur_n = n;                           // the rows, background and group CSR of this call
            m->own_X = ctx->own_X; m->own_D = ctx->own_D; m->own_bg = ctx->own_bg;
            m->own_goff = ctx->own_goff; m->own_gcols = ctx->own_gcols;
            ExplainParams pm = p;
            pm.C = m->C;
            const size_t msm = own_kernel(m->head.family).smem(m, p.S_cap);
            const dks::EnsRows mer{ctx->d_stk_ws, p.dlink, ctx->C, F, (int)f0, ctx->stk.cfirst[k], ctx->stk.ccount[k], j0, j1};
            TRY(on_member(ctx, m, [&] { return launch_own_kernel(m, false, pm, msm, st, dks::EnsAcc{}, mer); }));
        }
        dks::stack::stacking_reduce_kernel<<<std::max(1, std::min(n, ctx->sm_count * 8)), dks::stack::THREADS, 0, st>>>(
            p, ctx->stk, ctx->d_stk_ws, j0, j1, XWg, ctx->d_stk_BWg, ctx->d_stk_BWtot, ctx->d_ens_ey, j0 == 0 ? 1 : 0);
        ctx->launches += 1;
        CUDA_TRY(cudaGetLastError());
    }
    ctx->stk_chunks = chunks;
    const dks::SimtL1 q = l1 ? dks::SimtL1{ctx->d_l1, ctx->d_mom} : dks::SimtL1{};
    return launch_tail(ctx, l1, p, q, ctx->d_ens_ey, ctx->stk.head == DKS_STACK_HEAD_IDENTITY, st);
}

// stage 1's instantiation for R score rows: the compile-time bound 1 or 8 (a mixture: DKS_MIX_MAX_R)
template <bool STAGE, bool MAPS>
decltype(&dks::prep_kernel<STAGE, MAPS>) prep_kernel_for(bool mixture, int R) {
    if (mixture) return dks::prep_kernel<STAGE, MAPS, true>;
    return R == 1 ? dks::prep_kernel<STAGE, MAPS, false, 1> : dks::prep_kernel<STAGE, MAPS, false, 8>;
}

int launch_prepare(dks_ctx* ctx, const double* X_dev, int n) {
    ctx->ext_coalitions = -1;           // stage 1 rewrites what a module's call laid out by dks_external_begin reads
    const int G = ctx->G;
    const HeadDesc& h = ctx->head;
    TRY(ensure_workspace(ctx, n));
    // status word, list counters and the histogram of M are adjacent: one memset
    CUDA_TRY(cudaMemsetAsync(ctx->d_status, 0, sizeof(int) * (4 + G + 1), ctx->stream));
    if (!ctx->capturing) ctx->last_was_graph = false;
    CUDA_TRY(record_ev(ctx, 0));
    int ipb = 256 / G;
    if (ipb < 1) ipb = 1;
    const bool maps = ctx->cm.hdr != nullptr;
    const size_t maps_doubles = maps ? (size_t)ctx->cm.n_keys + ctx->cm.n_vals : 0;
    const bool stage = dks::prep_smem_bytes(true, ipb, G, ctx->R, ctx->D, maps_doubles) <= (size_t)96 * 1024;
    const size_t psm = dks::prep_smem_bytes(stage, ipb, G, ctx->R, ctx->D, maps_doubles);
    // the families with their own kernel: stage 1 only decides the varying groups (its scores are those of a zero linear
    // model, one identity output, and unused); the model's predict kernel then writes f(x) and link(f(x)) - link(fnull) of
    // every output
    const bool own = h.own();
    const int R = own ? 1 : ctx->R;
    auto kern = stage ? (maps ? prep_kernel_for<true, true>(h.mixture(), R) : prep_kernel_for<true, false>(h.mixture(), R))
                      : (maps ? prep_kernel_for<false, true>(h.mixture(), R) : prep_kernel_for<false, false>(h.mixture(), R));
    // nibble tables for the shared-plan route: the binary head's at any G, the other heads' up to 128 groups (what their
    // shared-plan route covers)
    double* xt = !own && (h.xt_any || (G <= 128 && ctx->plan_mode == 0)) ? ctx->d_XT.get() : nullptr;
    if (psm > 48 * 1024) CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)psm));
    // a model behind a column encoding: its kernels read the encoded rows, the encoded background and the encoded group CSR
    // (a refused value is reported by the encoding); stage 1 decides the varying groups on the raw rows
    const bool enc = own && ctx->enc.E > 0;
    if (enc) TRY(grow(ctx, ctx->d_Xenc, (size_t)n * ctx->enc.E));
    ctx->own_X = enc ? ctx->d_Xenc : X_dev;
    ctx->own_D = enc ? ctx->enc.E : ctx->D;
    ctx->own_bg = enc ? ctx->d_bg_enc : ctx->d_bg;
    ctx->own_goff = enc ? ctx->d_egoff : ctx->d_goff;
    ctx->own_gcols = enc ? ctx->d_egcols : ctx->d_gcols;
    kern<<<cdiv(n, ipb), 256, psm, ctx->stream>>>(
        X_dev, ctx->d_W, ctx->d_b, ctx->d_bg, ctx->d_goff, ctx->d_gcols, ctx->d_colmin, ctx->d_colmax, ctx->d_colnan,
        ctx->d_linkfnull, n, ctx->N, ctx->D, G, R, own ? 1 : ctx->C, own ? DKS_ACT_IDENTITY : ctx->act, own ? 1.0 : ctx->kappa,
        ctx->link, ipb, ctx->d_XW, ctx->d_vmask, ctx->d_M, ctx->d_dlink, ctx->d_hist, ctx->d_counts, ctx->d_idx_full,
        ctx->d_idx_other, xt, h.xt_scale, h.xt_bbar ? ctx->d_Bbar.get() : nullptr, ctx->d_status, ctx->cm, ctx->d_mix);
    if (own) TRY(launch_own_predict(ctx, X_dev, n, enc ? ctx->d_Xenc.get() : nullptr, ctx->d_linkfnull, nullptr, ctx->d_dlink));
    if (h.family == DKS_GENERAL_STACKING && ctx->stk.Wp != nullptr) {
        // the instances' passthrough per group, over the columns the members read
        TRY(grow(ctx, ctx->d_stk_XWg, (size_t)n * G * ctx->stk.R));
        dks::stack::stacking_pass_kernel<<<cdiv((long long)n * ctx->stk.R, 128), 128, 0, ctx->stream>>>(
            ctx->own_X, n, G, ctx->own_goff, ctx->own_gcols, ctx->stk, ctx->d_stk_XWg, nullptr);
        ctx->launches += 1;
    }
    ctx->launches += 1;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(record_ev(ctx, 1));
    ctx->cur_n = n;
    ctx->cur_X = X_dev;
    ctx->prepared = true;
    return DKS_OK;
}

// dst (+)= pi_k x the member buffer, over the rows of the instances on the shared-plan path
int launch_mix_axpy(dks_ctx* ctx, float* dst, float pi, bool first, int stride, int n) {
    long long grid = cdiv((long long)n * stride, 256);
    if (grid > (long long)ctx->sm_count * 8) grid = (long long)ctx->sm_count * 8;
    if (grid < 1) grid = 1;
    dks::mix::mix_axpy_kernel<<<(int)grid, 256, 0, ctx->stream>>>(ctx->d_mixscr, dst, pi, first ? 1 : 0, ctx->d_idx_full,
                                                                   ctx->d_counts, stride);
    ctx->launches += 1;
    CUDA_TRY(cudaGetLastError());
    return DKS_OK;
}

// what the l1 kernels of both instance lists share
dks::l1::Params l1_params(dks_ctx* ctx, int n, double* phi_dev) {
    dks::l1::Params lp;
    memset(&lp, 0, sizeof(lp));
    lp.n = n; lp.N = ctx->N; lp.G = ctx->G; lp.C = ctx->C; lp.link = ctx->link;
    lp.mode = ctx->l1_mode; lp.kfeat = ctx->l1_k; lp.nout = ctx->head.l1_nout; lp.tabs = ctx->d_l1;
    lp.binary = ctx->head.l1_binary;
    lp.src.act = ctx->act;                           // the exp head's LARS skips tasks with non-finite moments
    lp.dlink = ctx->d_dlink; lp.linkfnull = ctx->d_linkfnull; lp.fnull = ctx->d_fnull;
    lp.mom = ctx->d_mom; lp.phi = phi_dev; lp.status = ctx->d_status;
    return lp;
}

// does the LARS kernel hold one warp's workspace for M groups (its Gram matrix aside)?
bool lars_fits(const dks_ctx* ctx, int M) {
    return dks::l1::lars_smem_per_warp(M) <= (size_t)ctx->max_smem_optin - 2048;
}

// the LARS path + criterion + restricted WLS, one warp per task (at most `tasks`); warps sized for lp.Mmax (lars_fits).
// stage: every task has M = lp.Mmax, whose Gram matrix may then be staged in shared memory.
int launch_lars(dks_ctx* ctx, const dks::l1::Params& lp, int tasks, bool stage, cudaStream_t stream) {
    const int M = lp.Mmax;
    const size_t per_warp = dks::l1::lars_smem_per_warp(M);
    const size_t gram_bytes = sizeof(double) * (size_t)M * M;
    const size_t budget = (size_t)ctx->max_smem_optin - 2048;
    // the Gram matrix of the path goes to shared memory when at least four warps still fit next to it
    const int stage_gram = (stage && gram_bytes + 4 * per_warp <= budget) ? 1 : 0;
    const int wpc = std::min((int)((budget - (stage_gram ? gram_bytes : 0)) / per_warp), 8);
    const size_t lsm = per_warp * wpc + (stage_gram ? gram_bytes : 0);
    const int lgrid = persistent_grid(ctx, lsm, 1024, 4, (tasks + wpc - 1) / wpc);
    CUDA_TRY(cudaFuncSetAttribute(dks::l1::l1_lars_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lsm));
    dks::l1::l1_lars_kernel<<<lgrid, 32 * wpc, lsm, stream>>>(lp, wpc, stage_gram);
    ctx->launches += 1;
    return DKS_OK;
}

// upstream's l1 branch on the shared plan of G groups: moments of y per (instance, output), then the LARS path + criterion +
// restricted WLS, one warp each.  The binary heads: one output, y from the (sum p1, sum p0) buffer; the others: C outputs,
// y from src.
int launch_l1(dks_ctx* ctx, const PlanDev& pg, int n, const dks::shared_path::HeadSource& src, double* phi_dev) {
    dks::l1::Params lp = l1_params(ctx, n, phi_dev);
    lp.S = pg.S; lp.S_pad = pg.S_pad; lp.Mmax = ctx->G; lp.src = src; lp.sums = ctx->d_sums; lp.z = pg.z; lp.w = pg.w;
    lp.list = ctx->d_idx_full; lp.count = ctx->d_counts;
    const size_t msm = sizeof(double) * (size_t)pg.S;
    const int tasks = n * lp.nout;
    const int mgrid = tasks < ctx->sm_count * 2 ? tasks : ctx->sm_count * 2;
#define DKS_MOM(W, MULTI)                                                                                                 \
    CUDA_TRY(cudaFuncSetAttribute(dks::l1::l1_moments_kernel<W, MULTI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)msm)); \
    dks::l1::l1_moments_kernel<W, MULTI><<<mgrid, dks::l1::MOM_THREADS, msm, ctx->stream>>>(lp);
    if (lp.binary) {
        if (pg.W == 1) { DKS_MOM(1, false) } else { DKS_MOM(2, false) }
    } else {
        if (pg.W == 1) { DKS_MOM(1, true) } else { DKS_MOM(2, true) }
    }
#undef DKS_MOM
    ctx->launches += 1;
    return launch_lars(ctx, lp, tasks, true, ctx->stream);
}

// the device copy of the l1 table set (dks::l1::Params::tabs), after any change of h_l1
int sync_l1_tables(dks_ctx* ctx) {
    CUDA_TRY(cudaMemcpyAsync(ctx->d_l1, ctx->h_l1, sizeof(dks::l1::Tables) * (DKS_L1_MAX_GROUPS + 1), cudaMemcpyHostToDevice,
                             ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return DKS_OK;
}

// ---- the explain dispatcher: choose_route decides every kernel of a call before the first one is enqueued --------------
enum RouteShared {                      // the shared-plan route of the instances whose groups all vary
    ROUTE_SHARED_NONE,
    ROUTE_FUSED,                        // binary head: link + projection solve inside the coalition kernel
    ROUTE_BINARY,                       // binary head: (sum p1, sum p0), then a solve
    ROUTE_BINARY_MEMBERS,               // mixture of binary members: the binary head's kernel per member, then a solve
    ROUTE_CLASS_SUMS,                   // softmax / one-vs-rest: per-class sums, then a solve per (instance, class)
    ROUTE_CLASS_MEMBERS,                // mixture of softmax / one-vs-rest members: the class-sum kernel per member
    ROUTE_TABLES,                       // identity / exp: y from the tables, no coalition kernel
};

// per-instance plans drawn on the device: their layout and the sampler's launch configuration
struct SamplerConfig {
    int stride, W, nAmax, fstride, max_left, cap, fw;
    size_t ssm, fsm;
};

struct Route {
    int shared = ROUTE_SHARED_NONE;
    int solve = DKS_SOLVE_NONE;         // of the shared-plan route (DKS_SOLVE_*)
    int general = DKS_GENERAL_NONE;     // the kernel of the other instances (DKS_GENERAL_*)
    bool l1_full = false;               // the instances on the shared-plan route select (l1)
    int l1_Mmax = 0;                    // largest M < G whose instances select on the general list (0: none)
    bool wide_pi = false;               // per-instance plans of 65..128 groups (two-word rows)
    bool draw = false;                  // per-instance plans are drawn on the device first (sc)
    SamplerConfig sc = {};
    int S_cap = 2;                      // the largest S any instance can need
    size_t l1_smem = 0, smem = 0;       // staging of the general list's l1 kernel and of the general kernel
    dks::shared_path::FusedConfig fcfg = {};
};

int sampler_config(const dks_ctx* ctx, bool wide_pi, SamplerConfig* sc) {
    if (ctx->max_plan_S < 2)
        return fail(DKS_ERR_PLAN_MISSING, "per-instance plans need the shared plans of the M values present (their "
                    "enumerated prefix); none is set");
    REQUIRE(ctx->d_sinfo && ctx->d_afix, "per-instance plans: dks_set_plan_sampling has not been called");
    sc->stride = (ctx->max_plan_S + 1) & ~1;
    sc->W = wide_pi ? 2 : 1;                            // 64-bit words per coalition row
    sc->nAmax = ctx->G > 1 ? ctx->G - 1 : 1;
    sc->fstride = sc->nAmax * sc->nAmax;
    // table sized for the largest sampled part among the plans set (a plan's sampled rows <= its S)
    int max_left = 32;
    for (int M = 2; M <= ctx->G && M <= DKS_MAX_GROUPS; ++M)
        if (ctx->h_plans[M].z && ctx->h_sinfo[M].ncdf > 0) max_left = std::max(max_left, ctx->h_plans[M].S - ctx->h_sinfo[M].nfixed);
    sc->max_left = (max_left + 31) / 32 * 32;
    if (sc->max_left > dks::sampler::MAX_SAMPLED)
        return fail(DKS_ERR_UNSUPPORTED, "per-instance plans: %d sampled rows per plan exceed the sampler's limit of %d",
                    sc->max_left, dks::sampler::MAX_SAMPLED);
    int cap = 256;                           // hash slots; its arrays are reused for the bit-transposed plan and pair counts
    while (cap < 2 * sc->max_left || cap < sc->nAmax * (sc->nAmax + 1) / 2) cap <<= 1;
    sc->cap = cap;
    sc->ssm = dks::sampler::smem_bytes(cap, sc->max_left, ctx->G, sc->W);
    if (sc->ssm + 2048 > (size_t)ctx->max_smem_optin)
        return fail(DKS_ERR_UNSUPPORTED, "per-instance plan sampler needs %zu B of shared memory", sc->ssm);
    if (wide_pi) {
        sc->fsm = dks::sampler::wide_factor_smem(sc->nAmax);     // one CTA per instance inverts its normal matrix in place
    } else {
        const size_t per_warp = (size_t)2 * sc->nAmax * sc->nAmax * sizeof(double);
        sc->fw = std::min((int)((size_t)ctx->max_smem_optin / per_warp), dks::sampler::FACTOR_WARPS);
        if (sc->fw < 1)
            return fail(DKS_ERR_UNSUPPORTED, "per-instance plans: normal-matrix workspace does not fit shared memory");
        sc->fsm = (size_t)sc->fw * per_warp;
    }
    return DKS_OK;
}

// a family with its own kernel: every instance on that kernel (up to 64 groups, CUDA-core only), the instances whose M
// selects through the general list's l1 route -- the kernel's moments, then l1_lars_kernel -- whatever their M, G included
int choose_route_own(dks_ctx* ctx, const uint64_t* ext_z, int ext_stride, Route* rt) {
    const OwnKernel ok = own_kernel(ctx->head.family);
    const int G = ctx->G, kernel = ctx->kernel_choice;
    if (kernel != DKS_KERNEL_AUTO && kernel != DKS_KERNEL_SIMT)
        return fail(DKS_ERR_UNSUPPORTED, "%s run on the %s only (kernel 'auto' or 'simt')", ok.family, ok.kernel);
    if (G > 64) return fail(DKS_ERR_UNSUPPORTED, "%s: %d groups; the %s covers at most 64", ok.family, G, ok.kernel);
    rt->draw = ctx->plan_mode == 1 && ext_z == nullptr;
    if (rt->draw) TRY(sampler_config(ctx, false, &rt->sc));
    const bool per_inst = ext_z != nullptr || rt->draw;
    rt->S_cap = std::max(ext_z ? ext_stride : rt->draw ? rt->sc.stride : ctx->max_plan_S, 2);
    rt->smem = ok.smem(ctx, rt->S_cap);
    if ((long long)rt->smem > (long long)ctx->max_smem_optin)
        return fail(DKS_ERR_UNSUPPORTED, "%s needs %zu B of shared memory (> %d): nsamples, outputs or %s too many", ok.kernel,
                    rt->smem, ctx->max_smem_optin, ok.bound);
    if (ctx->l1_mode != 0) {
        if (per_inst) return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection runs on shared plans only");
        for (int M = 2; M <= G; ++M) {
            if (!((ctx->l1_sel[0] >> (M - 1)) & 1ull)) continue;
            if (ctx->h_l1[M].gram_raw == nullptr || ctx->h_l1[M].S != dks_effective_S(M, ctx->nsamples_req) ||
                ctx->h_plans[M].z == nullptr || ctx->h_plans[M].S != ctx->h_l1[M].S)
                return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection needs the shared plan of M=%d and its l1 tables "
                            "(dks_set_l1_tables)", M);
            rt->l1_Mmax = M;
        }
        if (rt->l1_Mmax > 0 && !lars_fits(ctx, rt->l1_Mmax))
            return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection: the %d x %d Cholesky factor does not fit shared memory",
                        rt->l1_Mmax, rt->l1_Mmax);
        rt->l1_smem = rt->smem;
    }
    rt->general = ctx->head.family;
    return DKS_OK;
}

// DKS_ERR_DOMAIN for the row the status word names, worded for what refused it: the family's kernels, or the pipeline in
// front of them; a tree's column encoding; a linear model's column maps
int fail_refused(const dks_ctx* ctx, const char* prefix) {
    const OwnKernel ok = refusing_kernel(ctx);
    const int row = ctx->h_status[1];
    if (ok.refuses != REFUSES_NONE && ctx->enc.E > 0)
        return fail(DKS_ERR_DOMAIN, "%s %d holds a raw value the pipeline refuses (NaN where no imputer fills it, an "
                    "infinity, or a category unseen at fit time), as scikit-learn does", prefix, row);
    if (ok.refuses != REFUSES_NONE)
        return fail(DKS_ERR_DOMAIN, "%s %d holds %s: %s refuse it, as scikit-learn does", prefix, row,
                    ok.refuses == REFUSES_NAN ? "NaN" : "NaN or an infinity", ok.family);
    return fail(DKS_ERR_DOMAIN, "%s %d holds a raw value %s refuses (NaN, or a category unseen at fit time, where the "
                "pipeline raises)", prefix, row, ctx->head.own() ? "the column encoding" : "its column map");
}

// the start of dks_fit for every family: the background, its weights, the linear model's W and b, the groups and the
// column statistics stage 1 decides the varying groups with on the device; fnull's buffers; none of the previous fit's
// arrays (column maps, column encoding, family arrays); status cleared
int fit_begin(dks_ctx* ctx) {
    const int N = ctx->N, D = ctx->D, G = ctx->G, R = ctx->R, C = ctx->C;
    const cudaStream_t st = ctx->stream;
    ctx->ext_coalitions = -1;
    CUDA_TRY(ctx->d_bg.alloc((size_t)N * D));
    CUDA_TRY(ctx->d_wbg.alloc((size_t)N));
    CUDA_TRY(ctx->d_W.alloc((size_t)R * D));
    CUDA_TRY(ctx->d_b.alloc((size_t)R));
    CUDA_TRY(ctx->d_goff.alloc((size_t)G + 1));
    CUDA_TRY(ctx->d_gcols.alloc((size_t)D));
    CUDA_TRY(ctx->d_colmin.alloc((size_t)D));
    CUDA_TRY(ctx->d_colmax.alloc((size_t)D));
    CUDA_TRY(ctx->d_colnan.alloc((size_t)D));
    CUDA_TRY(ctx->d_fnull.alloc((size_t)C));
    CUDA_TRY(ctx->d_linkfnull.alloc((size_t)C));
    ctx->fit_pool.clear();
    ctx->cm = ColumnMapsDev{}; ctx->enc = EncodingDev{};
    ctx->fitted = false;
    ctx->prepared = false;
    CUDA_TRY(cudaMemsetAsync(ctx->d_status, 0, sizeof(int) * 2, st));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_bg, ctx->h_bg.data(), sizeof(double) * N * D, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_wbg, ctx->h_wbg.data(), sizeof(double) * N, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_W, ctx->h_W.data(), sizeof(double) * R * D, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_b, ctx->h_b.data(), sizeof(double) * R, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_goff, ctx->h_goff.data(), sizeof(int32_t) * (G + 1), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_gcols, ctx->h_gcols.data(), sizeof(int32_t) * D, cudaMemcpyHostToDevice, st));
    // varying groups are decided on the raw columns (a tree behind a column encoding reads the encoded background)
    dks::fit_colstats_kernel<<<cdiv(D, 128), 128, 0, st>>>(ctx->d_bg, N, D, ctx->d_colmin, ctx->d_colmax, ctx->d_colnan);
    ctx->launches += 1;
    return DKS_OK;
}

// once the fit kernels are queued: fnull, link(fnull) and the status word back to the host.  A background row the model
// refuses is DKS_ERR_DOMAIN; a family with its own kernel (`family` not NULL) refuses a non-finite link(fnull).
int fit_readback(dks_ctx* ctx, const char* family) {
    const int C = ctx->C;
    const cudaStream_t st = ctx->stream;
    CUDA_TRY(cudaGetLastError());
    ctx->h_fnull.resize(C);
    ctx->h_linkfnull.resize(C);
    CUDA_TRY(cudaMemcpyAsync(ctx->h_fnull.data(), ctx->d_fnull, sizeof(double) * C, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(ctx->h_linkfnull.data(), ctx->d_linkfnull, sizeof(double) * C, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(ctx->h_status, ctx->d_status, sizeof(int) * 2, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (ctx->h_status[0] == DKS_ERR_DOMAIN) return fail_refused(ctx, "background row");
    if (family != nullptr)
        for (int c = 0; c < C; ++c)
            if (!std::isfinite(ctx->h_linkfnull[c]))
                return fail(DKS_ERR_NUMERIC, "%s: link(fnull) of output %d is not finite (fnull = %g): the background's "
                            "mean prediction is 0 or 1 under the logit link, or overflows", family, c, ctx->h_fnull[c]);
    return DKS_OK;
}

// the end of a successful dks_fit: workspace shapes depend on G, R and C, and the plans carry tables derived from the
// background and model: drop them
int fit_done(dks_ctx* ctx) {
    ctx->ws_n = 0;
    ctx->prepared = false;
    for (const DevPool& pool : ctx->plan_pool)
        if (!pool.empty()) { TRY(drop_plans(ctx, -1)); break; }
    ctx->fitted = true;
    ctx->epoch++;
    return DKS_OK;
}

// dks_fit's column encoding, after fit_begin: the device copy, the encoded background d_bg_enc and the encoded group CSR
// (group g owns the encoded columns whose raw source is in g, in increasing encoded index)
int fit_encoding(dks_ctx* ctx) {
    const int E = encoded_columns(ctx), G = ctx->G;
    if (E == 0) return DKS_OK;
    const cudaStream_t st = ctx->stream;
    EncodingDev& en = ctx->enc;
    DevPool& pool = ctx->fit_pool;
    CUDA_TRY(pool.upload(&en.hdr, ctx->h_ehdr.data(), ctx->h_ehdr.size(), st));
    CUDA_TRY(pool.upload(&en.ops, ctx->h_eops.data(), ctx->h_eops.size(), st));
    CUDA_TRY(pool.upload(&en.opv, ctx->h_eopv.data(), ctx->h_eopv.size(), st));
    CUDA_TRY(pool.upload(&en.tab, ctx->h_etab.data(), ctx->h_etab.size(), st));
    en.E = E;
    CUDA_TRY(pool.alloc(&ctx->d_bg_enc, (size_t)ctx->N * E));
    TRY(launch_encode(ctx, ctx->d_bg, ctx->N, ctx->d_bg_enc));
    const std::vector<int32_t> colgrp = column_groups(ctx);
    std::vector<int32_t> goff(G + 1, 0), gcols(E);
    for (int e = 0; e < E; ++e) goff[colgrp[e] + 1] += 1;
    for (int g = 0; g < G; ++g) goff[g + 1] += goff[g];
    std::vector<int32_t> at(goff.begin(), goff.end() - 1);
    for (int e = 0; e < E; ++e) gcols[at[colgrp[e]]++] = e;
    CUDA_TRY(pool.alloc(&ctx->d_egoff, (size_t)G + 1));
    CUDA_TRY(pool.alloc(&ctx->d_egcols, (size_t)E));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_egoff, goff.data(), sizeof(int32_t) * (G + 1), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_egcols, gcols.data(), sizeof(int32_t) * E, cudaMemcpyHostToDevice, st));
    return DKS_OK;
}

int fit_model(dks_ctx* ctx);

// dks_fit of a soft-voting or stacking ensemble's members: every member fitted, in order, on the ensemble's background,
// weights, groups and column encoding, under the identity link (the ensemble takes its own link)
int fit_member_contexts(dks_ctx* ctx) {
    for (size_t k = 0; k < ctx->ens.size(); ++k) {
        dks_ctx* m = ctx->ens[k];
        m->N = ctx->N; m->D = ctx->D; m->G = ctx->G;
        m->h_bg = ctx->h_bg; m->h_wbg = ctx->h_wbg; m->uniform_w = ctx->uniform_w;
        m->h_goff = ctx->h_goff; m->h_gcols = ctx->h_gcols;
        m->h_ehdr = ctx->h_ehdr; m->h_eops = ctx->h_eops; m->h_eopv = ctx->h_eopv; m->h_etab = ctx->h_etab;
        m->link = DKS_LINK_IDENTITY;
        const int rc = on_member(ctx, m, [&] { return fit_model(m); });
        if (rc != DKS_OK)
            return fail(rc, "%s member %d: %s", own_kernel(ctx->head.family).model, (int)k, g_last_error.c_str());
    }
    return DKS_OK;
}

// dks_fit of a soft-voting ensemble, after the common start: its members (fit_member_contexts), then
// fnull = sum_k pi_k fnull_k in member order and pi on the device
int fit_members(dks_ctx* ctx, const OwnKernel& ok) {
    const int C = ctx->C;
    std::vector<double> fnull(C, 0.0), linkfnull(C);
    TRY(fit_member_contexts(ctx));
    for (size_t k = 0; k < ctx->ens.size(); ++k)
        for (int c = 0; c < C; ++c) fnull[c] += ctx->h_ens_pi[k] * ctx->ens[k]->h_fnull[c];
    for (int c = 0; c < C; ++c) {
        linkfnull[c] = ctx->link == DKS_LINK_LOGIT ? std::log(fnull[c] / (1.0 - fnull[c])) : fnull[c];
        if (!std::isfinite(linkfnull[c]))
            return fail(DKS_ERR_NUMERIC, "%s: link(fnull) of output %d is not finite (fnull = %g): the background's "
                        "mean prediction is 0 or 1 under the logit link, or overflows", ok.model, c, fnull[c]);
    }
    const cudaStream_t st = ctx->stream;
    CUDA_TRY(ctx->fit_pool.upload(&ctx->d_ens_pi, ctx->h_ens_pi.data(), ctx->h_ens_pi.size(), st));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_fnull, fnull.data(), sizeof(double) * C, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_linkfnull, linkfnull.data(), sizeof(double) * C, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    ctx->h_fnull = fnull;
    ctx->h_linkfnull = linkfnull;
    return fit_done(ctx);
}

// dks_fit of a stacking ensemble, after the common start and its column encoding: its members (fit_member_contexts), the
// final estimator on the device and the background's passthrough tables over bg [N][width] (encoded behind a column
// encoding)
int fit_stacking(dks_ctx* ctx, const double* bg, int width) {
    TRY(fit_member_contexts(ctx));
    DevPool& pool = ctx->fit_pool;
    const cudaStream_t st = ctx->stream;
    StackDev& sd = ctx->stk;
    CUDA_TRY(pool.upload(&sd.W, ctx->h_stk_W.data(), ctx->h_stk_W.size(), st));
    CUDA_TRY(pool.upload(&sd.b, ctx->h_stk_b.data(), ctx->h_stk_b.size(), st));
    sd.Wp = nullptr;
    sd.D = width;
    ctx->d_stk_BWg = ctx->d_stk_BWtot = nullptr;
    if (!ctx->h_stk_Wp.empty()) {
        CUDA_TRY(pool.upload(&sd.Wp, ctx->h_stk_Wp.data(), ctx->h_stk_Wp.size(), st));
        double *BWg, *BWtot;
        CUDA_TRY(pool.alloc(&BWg, (size_t)ctx->N * ctx->G * sd.R));
        CUDA_TRY(pool.alloc(&BWtot, (size_t)ctx->N * sd.R));
        const bool enc = ctx->enc.E > 0;
        dks::stack::stacking_pass_kernel<<<cdiv((long long)ctx->N * sd.R, 128), 128, 0, st>>>(
            bg, ctx->N, ctx->G, enc ? ctx->d_egoff : ctx->d_goff.get(), enc ? ctx->d_egcols : ctx->d_gcols.get(), sd, BWg,
            BWtot);
        ctx->launches += 1;
        ctx->d_stk_BWg = BWg;
        ctx->d_stk_BWtot = BWtot;
    }
    return DKS_OK;
}

// dks_fit of a family with its own kernel: its column check, the common start, the column encoding, the family's arrays
// and tables, and fnull = sum_j w_j f(bg_j) from its predict kernel
int fit_own(dks_ctx* ctx) {
    const OwnKernel ok = own_kernel(ctx->head.family);
    const int N = ctx->N, C = ctx->C;
    TRY(check_own_columns(ctx, ok));
    TRY(fit_begin(ctx));
    TRY(fit_encoding(ctx));
    if (ctx->head.family == DKS_GENERAL_ENSEMBLE) return fit_members(ctx, ok);
    DevBuf<double> pred;
    const double* bg_pred = pred;
    if (ctx->head.family == DKS_GENERAL_EXTERNAL) {
        // a module: its outputs on the background (dks_set_external_background), and the group of every column for the mask
        REQUIRE(ctx->d_ext_bgy.size() == (size_t)N * C,
                "dks_fit: a module needs its outputs on the %d background rows first (dks_set_external_background)", N);
        const std::vector<int32_t> colgrp = column_groups(ctx);
        CUDA_TRY(ctx->fit_pool.upload(&ctx->d_ext_colgrp, colgrp.data(), colgrp.size(), ctx->stream));
        bg_pred = ctx->d_ext_bgy;
    } else {
        const double* bg = ctx->enc.E > 0 ? ctx->d_bg_enc : ctx->d_bg;
        if (ctx->head.family == DKS_GENERAL_STACKING) TRY(fit_stacking(ctx, bg, model_columns(ctx)));
        else TRY(own_fit_tables(ctx, bg, model_columns(ctx)));
        CUDA_TRY(pred.alloc((size_t)N * C));
        TRY(launch_own_predict(ctx, bg, N, nullptr, nullptr, pred, nullptr));
        bg_pred = pred;
    }
    dks::fit_pred_fnull_kernel<<<1, 32, 0, ctx->stream>>>(bg_pred, ctx->d_wbg, N, C, ctx->link, ctx->d_fnull,
                                                          ctx->d_linkfnull);
    ctx->launches += 1;
    TRY(fit_readback(ctx, ok.model));
    return fit_done(ctx);
}

int choose_route(dks_ctx* ctx, const uint64_t* ext_z, int ext_stride, Route* rt) {
    const HeadDesc& h = ctx->head;
    if (h.own()) {
        *rt = Route{};
        return choose_route_own(ctx, ext_z, ext_stride, rt);
    }
    const int G = ctx->G, N = ctx->N, kernel = ctx->kernel_choice;
    const bool auto_or_shared = kernel == DKS_KERNEL_AUTO || kernel == DKS_KERNEL_SHARED;
    *rt = Route{};
    // the mixture head: one pass of the member head's shared-plan kernel per member for instances whose groups all vary (up
    // to 128 groups), its CUDA-core kernel (dks_mixture.cuh) for the rest (up to 64 groups); no tensor-core kernel
    if (h.mixture() && G > h.shared_max_G)
        return fail(DKS_ERR_UNSUPPORTED, "mixture head: %d groups; it covers at most %d", G, h.shared_max_G);
    if (h.mixture() && kernel == DKS_KERNEL_TCGEN05)
        return fail(DKS_ERR_UNSUPPORTED, "mixture head: no tensor-core kernel (kernel 'auto', 'shared' or 'simt')");
    if (G > 64 && ext_z != nullptr)
        return fail(DKS_ERR_UNSUPPORTED, "more than 64 groups: caller-supplied per-instance plans are not supported");
    // per-instance plans of 65..128 groups (two-word rows): binary-logistic, identity or exp head, CUDA-core kernel
    rt->wide_pi = G > 64 && ctx->plan_mode == 1;
    if (rt->wide_pi) {
        if (G > 128)
            return fail(DKS_ERR_UNSUPPORTED, "per-instance plans cover at most 128 groups (G=%d); use shared plans", G);
        if (!h.wide_pi)
            return fail(DKS_ERR_UNSUPPORTED, "per-instance plans of more than 64 groups: binary-logistic, identity or exp head "
                        "only");
        if (kernel != DKS_KERNEL_AUTO && kernel != DKS_KERNEL_SIMT)
            return fail(DKS_ERR_UNSUPPORTED, "per-instance plans of more than 64 groups run on the CUDA-core kernel (kernel "
                        "'auto' or 'simt')");
        if (ctx->l1_mode != 0) return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection runs on shared plans only");
    }
    // every instance draws its own plan on the device; the explain kernels then read it like a caller-supplied one
    rt->draw = ctx->plan_mode == 1 && ext_z == nullptr;
    if (rt->draw) TRY(sampler_config(ctx, rt->wide_pi, &rt->sc));
    const bool per_inst = ext_z != nullptr || rt->draw;
    rt->S_cap = std::max(ext_z ? ext_stride : rt->draw ? rt->sc.stride : ctx->max_plan_S, 2);

    // shared-plan route: the instances whose varying set is all G groups, on the plan of G groups and its tables
    const PlanDev& pg = ctx->h_plans[G <= DKS_MAX_GROUPS ? G : 0];
    const bool plan_G = pg.z != nullptr && pg.S == dks_effective_S(G, ctx->nsamples_req);
    bool shared = auto_or_shared && !per_inst && G >= 2 && G <= h.shared_max_G && plan_G;
    if (h.shared == HEAD_SHARED_BINARY) shared = shared && pg.dmT != nullptr && (pg.W <= 2 || pg.ptw != nullptr);
    else shared = shared && ctx->full.M == G;
    if (kernel == DKS_KERNEL_SHARED && !shared && !per_inst && pg.z != nullptr)
        return fail(DKS_ERR_UNSUPPORTED, "shared-plan fast path needs the binary-logistic head, or the softmax / one-vs-rest / "
                    "identity / exp head with at most 128 groups");

    // l1 feature selection: on the shared-plan route when M = G selects, and on the general list (CUDA-core kernel for the
    // moments, then l1_lars_kernel) for the instances with a partial varying set whose M selects
    const bool l1 = ctx->l1_mode != 0;
    auto selects = [&](int M) {
        return l1 && M >= 1 && M <= DKS_L1_MAX_GROUPS && ((ctx->l1_sel[(M - 1) >> 6] >> ((M - 1) & 63)) & 1ull) != 0;
    };
    rt->l1_full = selects(G);
    for (int M = 2; M < G && M <= DKS_L1_MAX_GROUPS; ++M) if (selects(M)) rt->l1_Mmax = M;
    if (l1) {
        if (per_inst) return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection runs on shared plans only");
        if (rt->l1_full && pg.W > 2)
            return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection covers plans of at most 128 groups (M=%d)", G);
        if (rt->l1_full && (!shared || ctx->h_l1[G].gram_raw == nullptr || ctx->h_l1[G].S != pg.S))
            return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection needs the shared-plan path (binary-logistic, softmax, "
                        "one-vs-rest, identity, exp or mixture head) and the l1 tables of the M=%d plan (dks_set_l1_tables)", G);
        if (rt->l1_full && sizeof(double) * (size_t)pg.S + 8192 > (size_t)ctx->max_smem_optin)
            return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection: %d coalitions per plan exceed the shared-memory staging",
                        pg.S);
        if (rt->l1_full && !lars_fits(ctx, G))
            return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection: the %d x %d Cholesky factor does not fit shared memory", G, G);
        if (rt->l1_Mmax > 0) {
            const int Mmax = rt->l1_Mmax;
            if (G > 64)
                return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection for partial varying sets covers at most 64 groups (G=%d)", G);
            if (!auto_or_shared)
                return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection needs kernel 'auto' or 'shared' (the CUDA-core kernel "
                            "forms the moments of instances with a partial varying set)");
            for (int M = 2; M <= Mmax; ++M)
                if (selects(M) && (ctx->h_l1[M].gram_raw == nullptr || ctx->h_l1[M].S != dks_effective_S(M, ctx->nsamples_req) ||
                                   ctx->h_plans[M].z == nullptr || ctx->h_plans[M].S != ctx->h_l1[M].S))
                    return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection needs the shared plan of M=%d and its l1 tables "
                                "(dks_set_l1_tables)", M);
            rt->l1_smem = h.mixture() ? dks::mix::smem_bytes(rt->S_cap, N, Mmax, ctx->mix, ctx->C)
                                      : dks::simt_smem_bytes(rt->S_cap, N, Mmax, h.simt_R, h.simt_C);
            if ((long long)rt->l1_smem > (long long)ctx->max_smem_optin)
                return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection: the CUDA-core kernel's staging of instances with up to "
                            "%d varying groups needs %zu B of shared memory (> %d)", Mmax, rt->l1_smem, ctx->max_smem_optin);
            if (!lars_fits(ctx, Mmax))
                return fail(DKS_ERR_UNSUPPORTED, "l1 feature selection: the %d x %d Cholesky factor does not fit shared memory",
                            Mmax, Mmax);
        }
    }

    if (shared) {
        switch (h.shared) {
        case HEAD_SHARED_BINARY: {
            const bool fused = !rt->l1_full && ctx->opt_fused && pg.pmat64 != nullptr && pg.W == 1 &&
                               dks::shared_path::fused_config(N, G, pg.S_pad, ctx->sm_count, ctx->max_smem_optin,
                                                              ctx->opt_fused_warps, ctx->opt_fused_B, &rt->fcfg, !ctx->uniform_w);
            rt->shared = fused ? ROUTE_FUSED : ROUTE_BINARY;
            break;
        }
        case HEAD_SHARED_MIX_BINARY: rt->shared = ROUTE_BINARY_MEMBERS; break;
        case HEAD_SHARED_CLASS_SUMS: rt->shared = ROUTE_CLASS_SUMS; break;
        case HEAD_SHARED_MIX_CLASS: rt->shared = ROUTE_CLASS_MEMBERS; break;
        default: rt->shared = ROUTE_TABLES; break;
        }
        const bool binary = rt->shared == ROUTE_BINARY || rt->shared == ROUTE_BINARY_MEMBERS;
        if (rt->shared == ROUTE_FUSED) rt->solve = DKS_SOLVE_FUSED;
        else if (rt->l1_full) rt->solve = DKS_SOLVE_L1;
        else if (binary && pg.W > 2) rt->solve = DKS_SOLVE_WIDE;   // more than 128 groups: host-supplied projection
        else if (binary && pg.pmat != nullptr) rt->solve = DKS_SOLVE_PMAT;
        else rt->solve = DKS_SOLVE_WLS_SHARED;
    }

    // the kernel of the instances the shared-plan route does not take
    if (rt->wide_pi) {
        // per-instance two-word plans: the instances whose groups all vary run the CUDA-core two-word kernel; a partial
        // varying set is reported, not computed
        rt->smem = dks::iwide::smem_bytes(rt->S_cap);
        if ((long long)rt->smem > (long long)ctx->max_smem_optin)
            return fail(DKS_ERR_UNSUPPORTED, "two-word per-instance kernel needs %zu B of shared memory (> %d): nsamples too "
                        "large", rt->smem, ctx->max_smem_optin);
        rt->general = DKS_GENERAL_SIMT_WIDE;
    } else if (G > 64) {
        // two-word coalition rows exist on the shared-plan path only: anything left over is reported, not computed
        if (!plan_G || (pg.W > 2 && pg.ptw == nullptr)) {
            ctx->h_status[0] = DKS_ERR_PLAN_MISSING; ctx->h_status[1] = G;
            return fail(DKS_ERR_PLAN_MISSING, "no shared plan for M=%d at the current nsamples", G);
        }
        if (!shared)
            return fail(DKS_ERR_UNSUPPORTED, "more than 64 groups needs the shared-plan path (binary-logistic head, or the "
                        "softmax / one-vs-rest / identity head up to 128 groups, or the exp head up to 128 groups; kernel "
                        "'auto' or 'shared', shared plan of M=%d uploaded)", G);
        rt->general = DKS_GENERAL_FLAGGED;
    } else if (auto_or_shared ? dks::tc_supported(ctx, rt->S_cap) : kernel == DKS_KERNEL_TCGEN05) {
        if (!dks::tc_supported(ctx, rt->S_cap))
            return fail(DKS_ERR_UNSUPPORTED, "tensor-core kernel does not support this shape/head (N=%d G=%d act=%d)", N, G,
                        ctx->act);
        rt->general = DKS_GENERAL_TC;
    } else {
        rt->smem = h.mixture() ? dks::mix::smem_bytes(rt->S_cap, N, G, ctx->mix, ctx->C)
                               : dks::simt_smem_bytes(rt->S_cap, N, G, h.simt_R, h.simt_C);
        rt->general = DKS_GENERAL_SIMT;
        if ((long long)rt->smem > (long long)ctx->max_smem_optin) {
            // the shared-plan route took the instances whose groups all vary; the general kernel is sized for the largest
            // plan set and cannot hold it.  The instances left for it (often none) are reported, not computed.
            if (shared) {
                rt->general = DKS_GENERAL_FLAGGED;
            } else if (pg.z == nullptr && auto_or_shared && !per_inst && h.shared != HEAD_SHARED_BINARY && G >= 2 &&
                       G <= h.shared_max_G) {
                // these heads' shared-plan route takes these instances once the plan of G groups is uploaded
                ctx->h_status[0] = DKS_ERR_PLAN_MISSING; ctx->h_status[1] = G;
                return fail(DKS_ERR_PLAN_MISSING, "no shared plan for M=%d at the current nsamples", G);
            } else {
                return fail(DKS_ERR_UNSUPPORTED, "SIMT kernel needs %zu B of shared memory (> %d): N*G or nsamples too large",
                            rt->smem, ctx->max_smem_optin);
            }
        }
    }
    return DKS_OK;
}

// draws every instance's plan on the device and factors its normal matrix; p then reads the plans like caller-supplied ones
int launch_sampler(dks_ctx* ctx, const Route& rt, ExplainParams* p) {
    const SamplerConfig& sc = rt.sc;
    const int n = ctx->cur_n;
    const size_t need = (size_t)n * sc.stride;
    if (need > ctx->d_genw.size() || sc.W != ctx->gen_words) {
        CUDA_TRY(ctx->d_genz.alloc(need * sc.W)); CUDA_TRY(ctx->d_genw.alloc(need));
        ctx->gen_words = sc.W; ctx->epoch++;
    }
    const size_t needf = (size_t)n * sc.fstride;
    if (needf > ctx->d_genchol.size() || (!rt.wide_pi && ctx->d_genainv == nullptr)) {
        // two-word rows keep one matrix per instance (inverted in place); one-word rows its factor and its inverse
        CUDA_TRY(ctx->d_genchol.alloc(needf));
        if (rt.wide_pi) ctx->d_genainv.reset();
        else CUDA_TRY(ctx->d_genainv.alloc(needf));
        ctx->epoch++;
    }
    dks::sampler::SamplerParams sp;
    sp.n = n; sp.G = ctx->G; sp.S_req = ctx->nsamples_req; sp.stride = sc.stride; sp.seed = ctx->sampler_seed;
    sp.table_cap = sc.cap; sp.max_left = sc.max_left; sp.fstride = sc.fstride;
    sp.row_offset = ctx->row_offset; sp.Mcnt = ctx->d_M; sp.plans = ctx->d_plans; sp.info = ctx->d_sinfo;
    sp.afix = ctx->d_afix;
    sp.out_z = ctx->d_genz; sp.out_w = ctx->d_genw; sp.out_chol = ctx->d_genchol; sp.out_ainv = ctx->d_genainv;
    sp.status = ctx->d_status;
    auto skern = sc.W == 1 ? dks::sampler::sample_plans_kernel<1> : dks::sampler::sample_plans_kernel<2>;
    CUDA_TRY(cudaFuncSetAttribute(skern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sc.ssm));
    skern<<<persistent_grid(ctx, sc.ssm, 2048, 6, n), dks::sampler::THREADS, sc.ssm, ctx->stream>>>(sp);
    if (rt.wide_pi) {
        CUDA_TRY(cudaFuncSetAttribute(dks::sampler::factor_wide_plans_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)sc.fsm));
        const int fgrid = n < ctx->sm_count * 2 ? n : ctx->sm_count * 2;
        dks::sampler::factor_wide_plans_kernel<<<fgrid, dks::sampler::WIDE_FACTOR_THREADS, sc.fsm, ctx->stream>>>(
            n, ctx->d_M, ctx->G, sc.fstride, ctx->d_genchol, ctx->d_status);
    } else {
        CUDA_TRY(cudaFuncSetAttribute(dks::sampler::factor_plans_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sc.fsm));
        dks::sampler::factor_plans_kernel<<<(n + sc.fw - 1) / sc.fw, sc.fw * 32, sc.fsm, ctx->stream>>>(
            n, ctx->d_M, sc.fstride, ctx->d_genchol, ctx->d_genainv, sc.nAmax, ctx->d_status);
    }
    ctx->launches += 2;
    CUDA_TRY(cudaGetLastError());
    ctx->gen_stride = sc.stride; ctx->gen_n = n; ctx->gen_plan_words = sc.W;
    p->ext_z = ctx->d_genz; p->ext_w = ctx->d_genw; p->ext_stride = sc.stride;
    p->ext_chol = rt.wide_pi ? nullptr : ctx->d_genchol.get(); p->ext_ainv = rt.wide_pi ? ctx->d_genchol : ctx->d_genainv;
    p->ext_fstride = sc.fstride;
    return DKS_OK;
}

// binary head on the shared-plan route: the fused kernel, or the coalition kernel into (sum p1, sum p0) -- per member, added
// times pi_k, for a mixture of binary members
int launch_shared_binary(dks_ctx* ctx, const Route& rt, const PlanDev& pg, double* phi_dev) {
    const int n = ctx->cur_n, G = ctx->G;
    int32_t* path = ctx->last_path;
    const float* wn = ctx->uniform_w ? nullptr : ctx->d_wn.get();
    if (rt.shared == ROUTE_FUSED) {
        // link + projection solve inside the coalition kernel: no (sum p1, sum p0) buffer, no separate solve launch
        const dks::shared_path::FusedConfig& fcfg = rt.fcfg;
        dks::shared_path::FusedParams fp;
        memset(&fp, 0, sizeof(fp));
        fp.n = n; fp.N = ctx->N; fp.G = G; fp.C = ctx->C; fp.S = pg.S; fp.S_pad = pg.S_pad; fp.link = ctx->link; fp.B = fcfg.B;
        fp.scale = ctx->head.scale; fp.DmT = pg.dmT; fp.dme = pg.dme; fp.z = pg.z; fp.XT = ctx->d_XT; fp.list = ctx->d_idx_full;
        fp.count = ctx->d_counts; fp.pmat64 = pg.pmat64; fp.dvec = pg.dvec64; fp.dlink = ctx->d_dlink;
        fp.linkfnull = ctx->d_linkfnull; fp.fnull = ctx->d_fnull; fp.acc = ctx->d_acc; fp.wn = wn;
        const bool table = ctx->opt_fused_table && pg.ltab != nullptr;
        if (table) {
            fp.ltab = pg.ltab; fp.ltab_rows = pg.ltab_rows; fp.ltab_inv_h = pg.ltab_inv_h; fp.ltab_fb = ctx->d_ltab_fb;
        }
        CUDA_TRY(dks::shared_path::launch_explain_fused(fp, fcfg, ctx->sm_count, ctx->stream));
        // phi from the accumulators the fused kernel filled, sixteen lanes per instance; with push_in_kernel it also
        // stores the rows into the peers' gathered buffers
        dks::PeerPush pp;
        pp.npeers = 0;
        if (ctx->peer_world > 1 && ctx->push_in_kernel) {
            for (int r = 0; r < ctx->peer_world; ++r) {
                double* slab = ctx->peer_base[r] + (long long)ctx->peer_rank * ctx->peer_slab;
                if (slab == phi_dev) continue;               // phi is written in place into the local slab
                pp.dst[pp.npeers++] = slab;
            }
        }
        dks::shared_path::finish_fused_kernel<<<cdiv(n, 16), 256, 0, ctx->stream>>>(
            ctx->d_idx_full, ctx->d_counts, ctx->d_acc, dks::shared_path::fused_kpad(G), pg.dvec64, ctx->d_dlink, n, G, ctx->C,
            phi_dev, pp);
        ctx->launches += 1;          // the fused launch and its finish count as the route's one coalition launch
        path[DKS_PATH_SHARED] = DKS_SHARED_FUSED; path[DKS_PATH_CHUNKS] = 1; path[DKS_PATH_WARPS] = fcfg.warps;
        path[DKS_PATH_GRID] = ctx->sm_count; path[DKS_PATH_FUSED_B] = fcfg.B; path[DKS_PATH_FUSED_NI] = 1;
        path[DKS_PATH_SOLVE] = DKS_SOLVE_FUSED; path[DKS_PATH_FUSED_CTA_WARPS] = fcfg.slices * fcfg.kw;
        path[DKS_PATH_FUSED_TABLE] = table ? 1 : 0;
        CUDA_TRY(cudaGetLastError());
        return DKS_OK;
    }
    const size_t need = (size_t)n * pg.S_pad;
    TRY(grow(ctx, ctx->d_sums, need));
    dks::shared_path::SharedParams sp;
    sp.n = n; sp.N = ctx->N; sp.G = G; sp.S = pg.S; sp.S_pad = pg.S_pad; sp.scale = ctx->head.scale;
    sp.DmT = pg.dmT; sp.dme = pg.dme; sp.z = pg.z; sp.XT = ctx->d_XT; sp.list = ctx->d_idx_full; sp.count = ctx->d_counts; sp.sums = ctx->d_sums; sp.accumulate = 0;
    sp.acache = nullptr; sp.acache_mode = 0; sp.wn = wn;
    if (pg.W > 2 && ctx->N > dks::shared_path::MAXN) {
        // sixteen-word rows, several background chunks: A(i, s) is computed by the first chunk's launch only
        TRY(grow(ctx, ctx->d_acache, need));
        sp.acache = ctx->d_acache;
    }
    if (rt.shared == ROUTE_BINARY) {
        dks::shared_path::SharedLaunch sl;
        const int nl = dks::shared_path::launch_explain_shared(sp, pg.W, ctx->sm_count, ctx->max_smem_optin, ctx->stream, &sl);
        if (nl == 0) return fail(DKS_ERR_CUDA, "shared-plan kernel: %s", cudaGetErrorString(cudaGetLastError()));
        ctx->launches += nl;
        path[DKS_PATH_SHARED] = DKS_SHARED_SMEM; path[DKS_PATH_CHUNKS] = sl.chunks;
        path[DKS_PATH_WARPS] = sl.warps; path[DKS_PATH_GRID] = sl.grid;
        return DKS_OK;
    }
    // binary members: the binary head's kernel per member, into the member buffer, then added times pi_k
    const size_t stride = 2 * (size_t)pg.S_pad;
    TRY(grow(ctx, ctx->d_mixscr, (size_t)n * stride));
    const size_t xt_member = (size_t)n * ((G + 3) / 4) * 16;
    sp.scale = -DKS_LOG2E; sp.sums = reinterpret_cast<float2*>(ctx->d_mixscr.get());
    int chunks = 0, warps = 0, grid = 0;
    for (int k = 0; k < ctx->mix.K; ++k) {
        sp.DmT = ctx->full.dm[k]; sp.dme = ctx->full.dme[k]; sp.XT = ctx->d_XT + k * xt_member;
        dks::shared_path::SharedLaunch sl;
        const int nl = dks::shared_path::launch_explain_shared(sp, pg.W, ctx->sm_count, ctx->max_smem_optin, ctx->stream, &sl);
        if (nl == 0) return fail(DKS_ERR_CUDA, "shared-plan kernel: %s", cudaGetErrorString(cudaGetLastError()));
        ctx->launches += nl;
        chunks += sl.chunks; warps = k == 0 ? sl.warps : std::min(warps, sl.warps); grid = std::max(grid, sl.grid);
        TRY(launch_mix_axpy(ctx, reinterpret_cast<float*>(ctx->d_sums.get()), ctx->mix.pif[k], k == 0, (int)stride, n));
    }
    path[DKS_PATH_SHARED] = DKS_SHARED_MIX; path[DKS_PATH_CHUNKS] = chunks;
    path[DKS_PATH_WARPS] = warps; path[DKS_PATH_GRID] = grid;
    return DKS_OK;
}

// the solve of the binary heads' shared-plan route, from (sum p1, sum p0)
int launch_binary_solve(dks_ctx* ctx, const Route& rt, const PlanDev& pg, double* phi_dev) {
    const int n = ctx->cur_n, G = ctx->G, S = pg.S, S_pad = pg.S_pad;
    if (rt.solve == DKS_SOLVE_L1) {
        TRY(launch_l1(ctx, pg, n, dks::shared_path::HeadSource{}, phi_dev));
    } else if (rt.solve == DKS_SOLVE_WIDE) {
        // more than 128 groups: link, float64 product with the host-supplied projection, remainder (dks_wide.cuh)
        TRY(grow(ctx, ctx->d_yw, (size_t)n * S_pad));
        TRY(grow(ctx, ctx->d_betaw, (size_t)n * pg.kpw));
        dks::wide::WideParams qp;
        memset(&qp, 0, sizeof(qp));
        qp.n = n; qp.N = ctx->N; qp.G = G; qp.C = ctx->C; qp.S = S; qp.S_pad = S_pad; qp.KP = pg.kpw; qp.link = ctx->link;
        qp.sums = ctx->d_sums; qp.PT = pg.ptw; qp.dvec = pg.dvecw; qp.dlink = ctx->d_dlink;
        qp.linkfnull = ctx->d_linkfnull; qp.fnull = ctx->d_fnull; qp.list = ctx->d_idx_full; qp.count = ctx->d_counts;
        qp.y = ctx->d_yw; qp.beta = ctx->d_betaw; qp.phi = phi_dev;
        CUDA_TRY(dks::wide::launch_wide_solve(qp, n, ctx->sm_count, ctx->stream));
        ctx->launches += 3;
    } else if (rt.solve == DKS_SOLVE_PMAT) {
        dks::shared_path::WlsPmatParams pp;
        pp.n = n; pp.N = ctx->N; pp.G = G; pp.C = ctx->C; pp.S = S; pp.S_pad = S_pad; pp.link = ctx->link; pp.uniform_w = 1;
        pp.sums = ctx->d_sums; pp.pmat = pg.pmat; pp.dvec = pg.dvec; pp.dlink = ctx->d_dlink;
        pp.linkfnull = ctx->d_linkfnull; pp.fnull = ctx->d_fnull; pp.list = ctx->d_idx_full; pp.count = ctx->d_counts;
        pp.phi = phi_dev;
        cudaError_t perr = cudaSuccess;
        if (!dks::shared_path::launch_wls_pmat(pp, n, ctx->sm_count, ctx->max_smem_optin, ctx->stream, &perr))
            return fail(DKS_ERR_UNSUPPORTED, "projection solve does not fit shared memory");
        CUDA_TRY(perr);
        ctx->launches += 1;
        ctx->last_path[DKS_PATH_PMAT_KPAD] = dks::shared_path::wls_pmat_kpad(G);
    } else {
        dks::shared_path::WlsSharedParams wp;
        wp.n = n; wp.N = ctx->N; wp.G = G; wp.C = ctx->C; wp.S = S; wp.S_pad = S_pad; wp.link = ctx->link;
        wp.uniform_w = 1; wp.sums = ctx->d_sums; wp.z = pg.z; wp.w = pg.w; wp.ainv = pg.ainv; wp.dlink = ctx->d_dlink;
        wp.linkfnull = ctx->d_linkfnull; wp.fnull = ctx->d_fnull; wp.list = ctx->d_idx_full; wp.count = ctx->d_counts;
        wp.phi = phi_dev; wp.status = ctx->d_status;
        const size_t wsm = dks::shared_path::wls_shared_smem(G);
        const int wgrid = persistent_grid(ctx, wsm, 24 * 1024, 4, n);   // persistent CTAs of 8 warps
        if (pg.W == 1) {
            CUDA_TRY(cudaFuncSetAttribute(dks::shared_path::wls_shared_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsm));
            dks::shared_path::wls_shared_kernel<1><<<wgrid, dks::shared_path::WLS_THREADS, wsm, ctx->stream>>>(wp);
        } else {
            CUDA_TRY(cudaFuncSetAttribute(dks::shared_path::wls_shared_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsm));
            dks::shared_path::wls_shared_kernel<2><<<wgrid, dks::shared_path::WLS_THREADS, wsm, ctx->stream>>>(wp);
        }
        ctx->launches += 1;
    }
    ctx->last_path[DKS_PATH_SOLVE] = rt.solve;
    CUDA_TRY(cudaGetLastError());
    return DKS_OK;
}

// softmax, one-vs-rest, identity, exp and class-member mixture heads on the shared-plan route: the per-class sums of the
// class-sum coalition kernels (dks_multi.cuh; per member, added times pi_k, for a mixture) or the identity / exp head's
// tables.  *src: where the solve reads y.
int launch_class_sums(dks_ctx* ctx, const Route& rt, const PlanDev& pg, dks::shared_path::HeadSource* src) {
    const int n = ctx->cur_n, G = ctx->G, C = ctx->C, S_pad = pg.S_pad;
    int32_t* path = ctx->last_path;
    src->act = ctx->act; src->ntab = (G + 3) / 4; src->msums = nullptr; src->XT = ctx->d_XT; src->ell = ctx->full.ell;
    if (rt.shared == ROUTE_TABLES) {
        // y straight from the tables (and the plan's l(s) for the exp head): no coalition kernel
        path[DKS_PATH_SHARED] = ctx->head.expo ? DKS_SHARED_EXP : DKS_SHARED_AFFINE;
        return DKS_OK;
    }
    // the workspace is C n S_pad floats: the engine explains these heads in row blocks of 2 / C the binary path's
    const bool members = rt.shared == ROUTE_CLASS_MEMBERS;
    const size_t need = (size_t)n * C * S_pad;
    TRY(grow(ctx, ctx->d_msums, need));
    if (members) TRY(grow(ctx, ctx->d_mixscr, need));
    dks::multi::SoftmaxParams mp;
    memset(&mp, 0, sizeof(mp));
    mp.n = n; mp.N = ctx->N; mp.G = G; mp.S = pg.S; mp.S_pad = S_pad; mp.ntab = src->ntab; mp.scale = DKS_LOG2E;
    mp.wn = ctx->d_wn; mp.z = pg.z; mp.list = ctx->d_idx_full; mp.count = ctx->d_counts;
    mp.sums = members ? ctx->d_mixscr : ctx->d_msums;
    const MixHead& mh = ctx->mix;
    const int K = members ? mh.K : 1;
    const size_t xt_member = (size_t)n * mh.Rm * src->ntab * 16;
    int chunks = 0, grid = 0;
    for (int k = 0; k < K; ++k) {
        mp.dm = ctx->full.dm[k]; mp.lo = ctx->full.lo[k];
        if (members) {
            mp.XT = ctx->d_XT + k * xt_member;
            mp.BW = ctx->d_mixBW + (size_t)k * ctx->N * G * mh.Rm; mp.scores = ctx->d_mixsc + (size_t)k * ctx->N * mh.Rm;
        } else {
            mp.XT = ctx->d_XT; mp.BW = ctx->d_BW; mp.scores = ctx->d_scores;
        }
        const int nl = dks::multi::launch_class_sums(mp, ctx->head.ovr, C, pg.W, n, ctx->sm_count, ctx->max_smem_optin,
                                                     ctx->stream, &grid);
        if (nl == 0)
            return fail(DKS_ERR_CUDA, "%s coalition kernel: %s", members ? "mixture member" : ctx->head.ovr ? "one-vs-rest" : "softmax",
                        cudaGetErrorString(cudaGetLastError()));
        ctx->launches += nl;
        chunks += nl;
        if (members) TRY(launch_mix_axpy(ctx, ctx->d_msums, mh.pif[k], k == 0, C * S_pad, n));
    }
    path[DKS_PATH_SHARED] = members ? DKS_SHARED_MIX : ctx->head.ovr ? DKS_SHARED_OVR : DKS_SHARED_SOFTMAX;
    path[DKS_PATH_CHUNKS] = chunks; path[DKS_PATH_WARPS] = dks::multi::MC_WARPS; path[DKS_PATH_GRID] = grid;
    src->msums = ctx->d_msums;
    return DKS_OK;
}

// the solve per (instance, output) of launch_class_sums' route
int launch_class_solve(dks_ctx* ctx, const Route& rt, const PlanDev& pg, const dks::shared_path::HeadSource& src,
                       double* phi_dev) {
    const int n = ctx->cur_n, G = ctx->G, C = ctx->C;
    if (rt.solve == DKS_SOLVE_L1) {
        TRY(launch_l1(ctx, pg, n, src, phi_dev));
    } else {
        dks::shared_path::WlsSharedParams wp;
        memset(&wp, 0, sizeof(wp));
        wp.n = n; wp.N = ctx->N; wp.G = G; wp.C = C; wp.S = pg.S; wp.S_pad = pg.S_pad; wp.link = ctx->link; wp.uniform_w = 1;
        wp.src = src; wp.z = pg.z; wp.w = pg.w; wp.ainv = pg.ainv; wp.dlink = ctx->d_dlink; wp.linkfnull = ctx->d_linkfnull;
        wp.fnull = ctx->d_fnull; wp.list = ctx->d_idx_full; wp.count = ctx->d_counts; wp.phi = phi_dev;
        wp.status = ctx->d_status;
        const size_t wsm = dks::shared_path::wls_shared_smem(G);
        const int wgrid = persistent_grid(ctx, wsm, 24 * 1024, 4, (long long)n * C);
        if (pg.W == 1) {
            CUDA_TRY(cudaFuncSetAttribute(dks::shared_path::wls_shared_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsm));
            dks::shared_path::wls_shared_kernel<1, true><<<wgrid, dks::shared_path::WLS_THREADS, wsm, ctx->stream>>>(wp);
        } else {
            CUDA_TRY(cudaFuncSetAttribute(dks::shared_path::wls_shared_kernel<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsm));
            dks::shared_path::wls_shared_kernel<2, true><<<wgrid, dks::shared_path::WLS_THREADS, wsm, ctx->stream>>>(wp);
        }
        ctx->launches += 1;
    }
    ctx->last_path[DKS_PATH_SOLVE] = rt.solve;
    CUDA_TRY(cudaGetLastError());
    return DKS_OK;
}

// the general list splits into the instances whose M selects -- the CUDA-core kernel stores their moments and
// l1_lars_kernel selects and solves on the shared plan of each one's M -- and the rest, which p then lists
int launch_general_l1(dks_ctx* ctx, const Route& rt, ExplainParams* p, double* phi_dev, cudaStream_t gstream) {
    const int n = ctx->cur_n;
    CUDA_TRY(cudaMemsetAsync(ctx->d_l1_counts, 0, 2 * sizeof(int), gstream));
    int pgrid = cdiv(n, 256);
    if (pgrid > ctx->sm_count * 4) pgrid = ctx->sm_count * 4;
    dks::l1::l1_partition_kernel<<<pgrid, 256, 0, gstream>>>(p->list, p->count, n, ctx->d_M, ctx->l1_sel[0], ctx->l1_sel[1],
                                                             ctx->d_idx_sel, ctx->d_idx_plain, ctx->d_l1_counts);
    ExplainParams ps = *p;
    ps.list = ctx->d_idx_sel; ps.count = ctx->d_l1_counts;
    const bool timed = !ctx->capturing;
    if (ctx->head.own()) {
        if (timed) CUDA_TRY(cudaEventRecord(ctx->ev_l1[0], gstream));
        TRY(launch_own_kernel(ctx, true, ps, rt.l1_smem, gstream));
        ctx->launches += 1;
    } else {
        const bool mixh = ctx->head.mixture();
        auto l1kern = ctx->head.expo ? dks::explain_simt_kernel<true, true> : dks::explain_simt_kernel<true>;
        CUDA_TRY(cudaFuncSetAttribute(mixh ? (const void*)dks::mix::explain_simt_mix_kernel<true> : (const void*)l1kern,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rt.l1_smem));
        const int grid = persistent_grid(ctx, rt.l1_smem, 1024, 8, n);
        if (timed) CUDA_TRY(cudaEventRecord(ctx->ev_l1[0], gstream));
        if (mixh)
            dks::mix::explain_simt_mix_kernel<true><<<grid, 256, rt.l1_smem, gstream>>>(ps, dks::SimtL1{ctx->d_l1, ctx->d_mom},
                                                                                       ctx->mix);
        else
            l1kern<<<grid, 256, rt.l1_smem, gstream>>>(ps, dks::SimtL1{ctx->d_l1, ctx->d_mom},
                                                       ExpBackground{ctx->d_BW, ctx->d_scores});
        ctx->launches += 2;
    }
    if (timed) CUDA_TRY(cudaEventRecord(ctx->ev_l1[1], gstream));
    dks::l1::Params lp = l1_params(ctx, n, phi_dev);
    lp.Mmax = rt.l1_Mmax; lp.Mcnt = ctx->d_M; lp.vmask = ctx->d_vmask; lp.list = ctx->d_idx_sel; lp.count = ctx->d_l1_counts;
    TRY(launch_lars(ctx, lp, n * lp.nout, false, gstream));
    if (timed) CUDA_TRY(cudaEventRecord(ctx->ev_l1[2], gstream));
    ctx->l1_timing_valid = timed;
    CUDA_TRY(cudaGetLastError());
    ctx->last_path[DKS_PATH_GENERAL_L1] = 1;
    p->list = ctx->d_idx_plain;
    p->count = ctx->d_l1_counts + 1;
    return DKS_OK;
}

// the kernel of the instances the shared-plan route and the general list's l1 selection left (p.list)
int launch_general(dks_ctx* ctx, const Route& rt, ExplainParams p, cudaStream_t gstream) {
    const int n = ctx->cur_n, G = ctx->G;
    const ExpBackground eb{ctx->d_BW, ctx->d_scores};
    switch (rt.general) {
    case DKS_GENERAL_SIMT_WIDE: {
        p.list = ctx->d_idx_full; p.count = ctx->d_counts;
        auto wkern = ctx->head.expo ? dks::iwide::explain_wide_instance_kernel<true> : dks::iwide::explain_wide_instance_kernel<false>;
        CUDA_TRY(cudaFuncSetAttribute(wkern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rt.smem));
        wkern<<<persistent_grid(ctx, rt.smem, 1024, 4, n), dks::iwide::THREADS, rt.smem, gstream>>>(p, eb);
        dks::flag_unsupported_kernel<<<1, 1, 0, gstream>>>(ctx->d_counts + 1, G, ctx->d_status);
        ctx->launches += 2;
        break;
    }
    case DKS_GENERAL_FLAGGED:
        dks::flag_unsupported_kernel<<<1, 1, 0, gstream>>>(p.count, G, ctx->d_status);
        ctx->launches += 1;
        break;
    case DKS_GENERAL_TC:
        TRY(dks::tc_launch(ctx, p, gstream));
        break;
    default: {
        if (ctx->head.own()) {
            TRY(launch_own_kernel(ctx, false, p, rt.smem, gstream));
            break;
        }
        const bool mixh = ctx->head.mixture();
        auto skern = ctx->head.expo ? dks::explain_simt_kernel<false, true> : dks::explain_simt_kernel<false>;
        CUDA_TRY(cudaFuncSetAttribute(mixh ? (const void*)dks::mix::explain_simt_mix_kernel<false> : (const void*)skern,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rt.smem));
        const int grid = persistent_grid(ctx, rt.smem, 1024, 8, n);
        if (mixh) dks::mix::explain_simt_mix_kernel<false><<<grid, 256, rt.smem, gstream>>>(p, dks::SimtL1{}, ctx->mix);
        else skern<<<grid, 256, rt.smem, gstream>>>(p, dks::SimtL1{}, eb);
        ctx->launches += 1;
        break;
    }
    }
    ctx->last_path[DKS_PATH_GENERAL] = rt.general;
    CUDA_TRY(cudaGetLastError());
    return DKS_OK;
}

// debug dump of one instance's accumulator tile (tensor-core kernel only)
int prepare_debug_dump(dks_ctx* ctx, int S_cap) {
    const int rows = S_cap, cols = dks::tc_npad(ctx->N);
    if (rows != ctx->dbg_rows || cols != ctx->dbg_cols) {
        CUDA_TRY(ctx->dbg_T.alloc((size_t)rows * cols));
        ctx->dbg_rows = rows; ctx->dbg_cols = cols;
    }
    CUDA_TRY(cudaMemsetAsync(ctx->dbg_T, 0, sizeof(float) * rows * cols, ctx->stream));
    if (!ctx->dbg_time) CUDA_TRY(ctx->dbg_time.alloc(6 * 256));
    CUDA_TRY(cudaMemsetAsync(ctx->dbg_time, 0, sizeof(float) * 6 * 256, ctx->stream));
    return DKS_OK;
}

// the start of an explain call: its route and the explain kernels' parameters, every instance's plan drawn first when the
// device draws them
int explain_setup(dks_ctx* ctx, double* phi_dev, const uint64_t* ext_z, const double* ext_w, int ext_stride, Route* rtp,
                  ExplainParams* pp) {
    REQUIRE(ctx->prepared, "dks_explain: call dks_prepare_* first");
    REQUIRE((ext_z == nullptr) == (ext_w == nullptr), "ext_zbits and ext_w must both be given or both be NULL");
    memset(ctx->last_path, 0, sizeof(ctx->last_path));   // what this call launches (dks_last_path)
    Route& rt = *rtp;
    TRY(choose_route(ctx, ext_z, ext_stride, &rt));
    const int n = ctx->cur_n, G = ctx->G;
    ExplainParams& p = *pp;
    memset(&p, 0, sizeof(p));
    p.n = n; p.N = ctx->N; p.G = G; p.R = ctx->R; p.C = ctx->C;
    p.act = ctx->act; p.link = ctx->link; p.S_req = ctx->nsamples_req;
    p.scale = ctx->head.scale;
    p.BWs = ctx->d_BWs; p.bases = ctx->d_bases; p.wbf = ctx->d_wbf; p.wbg = ctx->d_wbg; p.Bbar = ctx->d_Bbar;
    p.fnull = ctx->d_fnull; p.linkfnull = ctx->d_linkfnull;
    p.XW = ctx->d_XW; p.vmask = ctx->d_vmask; p.Mcnt = ctx->d_M; p.dlink = ctx->d_dlink;
    p.plans = ctx->d_plans; p.ext_z = ext_z; p.ext_w = ext_w; p.ext_stride = ext_stride;
    p.phi = phi_dev; p.status = ctx->d_status;
    p.S_cap = rt.S_cap;
    if (rt.draw) TRY(launch_sampler(ctx, rt, &p));
    return DKS_OK;
}

// the explain kernels of a call explain_setup laid out, phi into p.phi
int explain_launch(dks_ctx* ctx, const Route& rt, ExplainParams p) {
    const int n = ctx->cur_n, G = ctx->G;
    double* phi_dev = p.phi;
    if (ctx->dbg_i >= 0) TRY(prepare_debug_dump(ctx, rt.S_cap));
    CUDA_TRY(record_ev(ctx, 2));
    ctx->l1_timing_valid = false;
    if (ctx->l1_mode != 0) TRY(grow(ctx, ctx->d_mom, (size_t)n * ctx->head.l1_nout * (2 * G + 4)));
    ctx->last_fused = rt.shared == ROUTE_FUSED;
    // the general kernels (instances that are not on the shared-plan route) fork off here and join at the end
    cudaStream_t gstream = ctx->stream;
    if (rt.shared != ROUTE_SHARED_NONE) {
        ctx->last_path[DKS_PATH_BG_WEIGHTS] = ctx->uniform_w ? 0 : 1;
        if (ctx->side_stream != nullptr) {
            CUDA_TRY(cudaEventRecord(ctx->ev_fork, ctx->stream));
            CUDA_TRY(cudaStreamWaitEvent(ctx->side_stream, ctx->ev_fork, 0));
            gstream = ctx->side_stream;
        }
        const PlanDev& pg = ctx->h_plans[G];
        if (rt.shared == ROUTE_FUSED || rt.shared == ROUTE_BINARY || rt.shared == ROUTE_BINARY_MEMBERS) {
            TRY(launch_shared_binary(ctx, rt, pg, phi_dev));
            if (rt.shared != ROUTE_FUSED) TRY(launch_binary_solve(ctx, rt, pg, phi_dev));
        } else {
            dks::shared_path::HeadSource src;
            TRY(launch_class_sums(ctx, rt, pg, &src));
            TRY(launch_class_solve(ctx, rt, pg, src, phi_dev));
        }
        p.list = ctx->d_idx_other;      // the general kernels take the remaining instances
        p.count = ctx->d_counts + 1;
    }
    if (rt.l1_Mmax > 0) TRY(launch_general_l1(ctx, rt, &p, phi_dev, gstream));
    TRY(launch_general(ctx, rt, p, gstream));
    if (gstream != ctx->stream) {
        CUDA_TRY(cudaEventRecord(ctx->ev_join, gstream));
        CUDA_TRY(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    }
    CUDA_TRY(record_ev(ctx, 3));
    return DKS_OK;
}

int launch_explain(dks_ctx* ctx, double* phi_dev, const uint64_t* ext_z, const double* ext_w, int ext_stride) {
    if (ctx->head.family == DKS_GENERAL_EXTERNAL)
        return fail(DKS_ERR_UNSUPPORTED, "module: the caller runs the module between the engine's launches; explain with "
                    "dks_external_begin / _mask / _reduce / _finish");
    Route rt;
    ExplainParams p;
    TRY(explain_setup(ctx, phi_dev, ext_z, ext_w, ext_stride, &rt, &p));
    return explain_launch(ctx, rt, p);
}

int check_status(dks_ctx* ctx) {
    // status was copied to h_status by the caller and the stream synchronised
    if (ctx->h_status[0] == 0) return DKS_OK;
    if (ctx->h_status[0] == DKS_ERR_PLAN_MISSING)
        return fail(DKS_ERR_PLAN_MISSING, "no shared plan for M=%d at the current nsamples", ctx->h_status[1]);
    if (ctx->h_status[0] == DKS_ERR_DOMAIN) return fail_refused(ctx, "instance");
    if (ctx->h_status[0] == DKS_ERR_NUMERIC)
        return fail(DKS_ERR_NUMERIC, "normal matrix not positive definite, or (exp head) a model output that is not finite "
                    "(instance/M %d)", ctx->h_status[1]);
    return fail(ctx->h_status[0], "explain kernel reported status %d (detail %d)", ctx->h_status[0], ctx->h_status[1]);
}

// projection form of the shared-plan solve of the binary head (and of binary mixtures): P = inv(E^T W E) E^T W and d = P z_L,
// when it fits the solve kernel's staging
int build_pmat(dks_ctx* ctx, PlanDev& pd, int M) {
    if (!(pd.W == 1 && M - 1 <= dks::shared_path::PMAT_MAXK &&
          dks::shared_path::wls_pmat_smem(M, pd.S_pad) + 8192 <= (size_t)ctx->max_smem_optin))
        return DKS_OK;
    const int S = pd.S;
    float* pm; double* dv;
    CUDA_TRY(ctx->plan_pool[M].alloc(&pm, (size_t)(M - 1) * pd.S_pad));
    CUDA_TRY(ctx->plan_pool[M].alloc(&dv, (size_t)(M - 1)));
    long long tot = (long long)(M - 1) * pd.S_pad;
    dks::shared_path::plan_pmat_kernel<<<cdiv(tot, 256), 256, 0, ctx->stream>>>(pd.z, pd.w, pd.ainv, S, pd.S_pad, M, pm);
    dks::shared_path::plan_dvec_kernel<<<M - 1, 32, 0, ctx->stream>>>(pd.z, pm, S, pd.S_pad, M, dv);
    ctx->launches += 2;
    CUDA_TRY(cudaGetLastError());
    pd.pmat = pm; pd.dvec = dv;
    return DKS_OK;
}

// Chebyshev nodes of [0, 1] and the inverse of their Vandermonde matrix (Gauss-Jordan, partial pivoting)
dks::shared_path::LinkTabFit make_link_tab_fit() {
    constexpr int K = dks::shared_path::LTAB_NODES;
    dks::shared_path::LinkTabFit f;
    double a[K][2 * K];
    for (int m = 0; m < K; ++m) {
        f.t[m] = 0.5 - 0.5 * cos((2 * m + 1) * 3.14159265358979323846 / (2 * K));
        for (int c = 0; c < K; ++c) { a[m][c] = pow(f.t[m], c); a[m][K + c] = m == c ? 1.0 : 0.0; }
    }
    for (int c = 0; c < K; ++c) {
        int piv = c;
        for (int r = c + 1; r < K; ++r) if (fabs(a[r][c]) > fabs(a[piv][c])) piv = r;
        for (int k = 0; k < 2 * K; ++k) std::swap(a[c][k], a[piv][k]);
        const double d = a[c][c];
        for (int k = 0; k < 2 * K; ++k) a[c][k] /= d;
        for (int r = 0; r < K; ++r) {
            if (r == c) continue;
            const double m = a[r][c];
            for (int k = 0; k < 2 * K; ++k) a[r][k] -= m * a[c][k];
        }
    }
    for (int r = 0; r < K; ++r) for (int c = 0; c < K; ++c) f.vinv[r * K + c] = a[r][K + c];
    return f;
}

// The fused kernel's link table of a plan (dks_fused.cuh) at h = 1/4, refined once to h = 1/8.  pd.ltab stays NULL (the
// plan keeps the exact loop) when both miss LTAB_TOL or the table would pass LTAB_BUDGET.
int build_link_table(dks_ctx* ctx, PlanDev& pd, int M, const uint64_t* dz) {
    using namespace dks::shared_path;
    static const LinkTabFit fit = make_link_tab_fit();
    const int N = ctx->N, S_pad = pd.S_pad;
    cudaStream_t st = ctx->stream;
    DevBuf<double> ld, wd;
    DevBuf<LinkTabRow> rows;
    DevBuf<unsigned long long> merr;
    CUDA_TRY(ld.alloc((size_t)N * S_pad));
    CUDA_TRY(rows.alloc((size_t)S_pad));
    CUDA_TRY(merr.alloc(1));
    if (!ctx->uniform_w) {
        std::vector<double> w(N);
        for (int j = 0; j < N; ++j) w[j] = (double)N * ctx->h_wbg[j];
        CUDA_TRY(wd.alloc((size_t)N));
        CUDA_TRY(cudaMemcpy(wd, w.data(), sizeof(double) * N, cudaMemcpyHostToDevice));
    }
    if (ctx->d_ltab_fb == nullptr) {
        CUDA_TRY(ctx->d_ltab_fb.alloc(1));
        CUDA_TRY(cudaMemset(ctx->d_ltab_fb, 0, sizeof(unsigned long long)));
    }
    std::vector<LinkTabRow> hr(S_pad);
    for (double h : {0.25, 0.125}) {
        plan_ltab_rows_kernel<<<cdiv(S_pad, 128), 128, 0, st>>>(dz, pd.S, S_pad, ctx->d_BW, ctx->d_scores, N, ctx->G, ctx->head.scale,
                                                                pd.dme, wd, h, ld, rows);
        ctx->launches += 1;
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaMemcpyAsync(hr.data(), rows, sizeof(LinkTabRow) * S_pad, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        long long total = 0;
        int maxn = 0;
        for (LinkTabRow& r : hr) { r.off = (int)(total < (1LL << 30) ? total : 0); total += r.nint; maxn = std::max(maxn, r.nint); }
        const size_t bytes = sizeof(LinkTabEntry) * (size_t)total + sizeof(LinkTabRow) * (size_t)S_pad;
        if (bytes > LTAB_BUDGET || maxn > 65535 * 128) return DKS_OK;     // a finer grid only makes it larger
        DevBuf<LinkTabEntry> tab;
        CUDA_TRY(tab.alloc((size_t)total));
        CUDA_TRY(cudaMemcpyAsync(rows, hr.data(), sizeof(LinkTabRow) * S_pad, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemsetAsync(merr, 0, sizeof(unsigned long long), st));
        const dim3 grid(S_pad, cdiv(maxn, 128));
        if (maxn > 0) {
            plan_ltab_fit_kernel<<<grid, 128, 0, st>>>(fit, rows, ld, S_pad, wd, N, ctx->link, h, tab, merr);
            ctx->launches += 1;
            CUDA_TRY(cudaGetLastError());
        }
        unsigned long long bits = 0;
        CUDA_TRY(cudaMemcpyAsync(&bits, merr, sizeof(bits), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        double err;
        memcpy(&err, &bits, sizeof(err));
        if (err <= LTAB_TOL) {
            pd.ltab = tab; pd.ltab_rows = rows; pd.ltab_inv_h = 1.0 / h; pd.ltab_bytes = (long long)bytes;
            ctx->plan_pool[M].adopt(std::move(tab));                 // tab and rows now belong to the plan
            ctx->plan_pool[M].adopt(std::move(rows));
            return DKS_OK;
        }
    }
    return DKS_OK;
}

// dks_fit without the binding (a soft-voting ensemble fits its members through it)
int fit_model(dks_ctx* ctx) {
    REQUIRE(ctx->N > 0 && ctx->R > 0, "dks_fit: background and model must be set first");
    const int N = ctx->N, D = ctx->D, R = ctx->R, C = ctx->C;
    if (ctx->G == 0) {  // default: one singleton group per column (DenseData default)
        if (D > DKS_MAX_GROUPS)
            return fail(DKS_ERR_UNSUPPORTED, "D=%d ungrouped columns; this build handles at most %d groups", D, DKS_MAX_GROUPS);
        ctx->G = D;
        ctx->h_goff.resize(D + 1);
        ctx->h_gcols.resize(D);
        for (int c = 0; c <= D; ++c) ctx->h_goff[c] = c;
        for (int c = 0; c < D; ++c) ctx->h_gcols[c] = c;
    }
    const int G = ctx->G;
    ctx->head = describe_head(ctx);
    const HeadDesc& h = ctx->head;
    if (h.expo && ctx->link == DKS_LINK_LOGIT)
        return fail(DKS_ERR_UNSUPPORTED, "exp head: the logit link is undefined wherever a predicted mean exceeds 1; use the "
                    "identity link");
    if (h.family == DKS_GENERAL_TREES && ctx->tree.head == DKS_TREE_HEAD_IFOREST && ctx->link == DKS_LINK_LOGIT)
        return fail(DKS_ERR_UNSUPPORTED, "anomaly head: an IsolationForest score is not a probability and has no logit; use "
                    "the identity link");
    {   // every column in exactly one group
        std::vector<int> seen(D, 0);
        REQUIRE((int)ctx->h_gcols.size() == D, "groups cover %d columns but the data has %d", (int)ctx->h_gcols.size(), D);
        for (int c : ctx->h_gcols) {
            REQUIRE(c >= 0 && c < D, "group column %d out of range", c);
            REQUIRE(seen[c]++ == 0, "column %d appears in more than one group", c);
        }
    }
    if (h.own()) return fit_own(ctx);
    if (!ctx->h_ehdr.empty())
        return fail(DKS_ERR_UNSUPPORTED, "dks_fit: a column encoding is set, but the model has no kernel of its own (linear "
                    "models read their pipelines through dks_set_column_maps)");
    TRY(fit_begin(ctx));
    CUDA_TRY(ctx->d_BW.alloc((size_t)N * G * R));
    CUDA_TRY(ctx->d_scores.alloc((size_t)N * R));
    CUDA_TRY(ctx->d_Bbar.alloc((size_t)G * R));
    CUDA_TRY(ctx->d_BWs.alloc((size_t)N * G * R));
    CUDA_TRY(ctx->d_bases.alloc((size_t)N * R));
    CUDA_TRY(ctx->d_wbf.alloc((size_t)N));
    CUDA_TRY(ctx->d_wn.alloc((size_t)N));
    CUDA_TRY(ctx->d_mix.alloc(1));
    cudaStream_t st = ctx->stream;
    CUDA_TRY(cudaMemcpyAsync(ctx->d_mix, &ctx->mix, sizeof(MixHead), cudaMemcpyHostToDevice, st));
    const bool maps = !ctx->h_cm_hdr.empty();
    if (maps) {
        ColumnMapsDev& cm = ctx->cm;
        DevPool& pool = ctx->fit_pool;
        CUDA_TRY(pool.upload(&cm.hdr, ctx->h_cm_hdr.data(), ctx->h_cm_hdr.size(), st));
        CUDA_TRY(pool.upload(&cm.keys, ctx->h_cm_keys.data(), ctx->h_cm_keys.size(), st));
        CUDA_TRY(pool.upload(&cm.vals, ctx->h_cm_vals.data(), ctx->h_cm_vals.size(), st));
        cm.n_keys = (int)ctx->h_cm_keys.size();
        cm.n_vals = (int)ctx->h_cm_vals.size();
    }
    {
        // the weighted shared-plan kernels read w'_j = N w_j: their sums then have the magnitude of the uniform ones
        std::vector<float> wn(N);
        for (int j = 0; j < N; ++j) wn[j] = (float)((double)N * ctx->h_wbg[j]);
        CUDA_TRY(cudaMemcpy(ctx->d_wn, wn.data(), sizeof(float) * N, cudaMemcpyHostToDevice));
    }
    (maps ? (R > 8 ? dks::fit_bw_kernel<true, true> : dks::fit_bw_kernel<true>) : dks::fit_bw_kernel<false>)<<<cdiv((long long)N * G * R, 256), 256, 0, st>>>(
        ctx->d_bg, ctx->d_W, ctx->d_goff, ctx->d_gcols, N, D, G, R, ctx->d_BW, ctx->cm, ctx->d_status);
    dks::fit_scores_kernel<<<cdiv((long long)N * R, 256), 256, 0, st>>>(ctx->d_BW, ctx->d_b, N, G, R, ctx->d_scores);
    if (h.mixture()) {
        CUDA_TRY(ctx->d_mixBW.alloc((size_t)N * G * R));
        CUDA_TRY(ctx->d_mixsc.alloc((size_t)N * R));
        dks::mix::mix_split_kernel<<<cdiv((long long)N * G * R, 256), 256, 0, st>>>(ctx->d_BW, ctx->d_scores, N, G, ctx->mix.K,
                                                                                    ctx->mix.Rm, ctx->d_mixBW, ctx->d_mixsc);
        ctx->launches += 1;
    }
    dks::fit_fnull_kernel<<<1, 256, 0, st>>>(ctx->d_scores, ctx->d_BW, ctx->d_wbg, N, G, R, C, ctx->act, ctx->kappa,
                                              ctx->link, ctx->d_fnull, ctx->d_linkfnull, ctx->d_Bbar, ctx->d_mix);
    dks::fit_scale_kernel<<<cdiv((long long)N * G * R, 256), 256, 0, st>>>(ctx->d_BW, ctx->d_scores, ctx->d_wbg, N, G, R,
                                                                              h.scale, ctx->d_BWs, ctx->d_bases, ctx->d_wbf,
                                                                              h.expo ? 1 : 0);
    ctx->launches += 4;
    TRY(fit_readback(ctx, nullptr));
    if (h.expo && !std::isfinite(ctx->h_fnull[0]))
        return fail(DKS_ERR_NUMERIC, "exp head: the background's predictions are not all finite in float64 (fnull = %g)",
                    ctx->h_fnull[0]);
    return fit_done(ctx);
}

// frees the members a soft-voting ensemble owns (their stream and status word are the ensemble's)
void destroy_members(dks_ctx* ctx) {
    for (dks_ctx* m : ctx->ens) {
        m->ens_parent = nullptr;
        dks_destroy(m);
    }
    ctx->ens.clear();
    ctx->h_ens_pi.clear();
}

// the members [K] a soft-voting or stacking ensemble (setter `fn`) is handed: distinct contexts of their own on its device,
// each a tree ensemble, kernel machine, MLP or neighbour model, and (C > 0) each giving C outputs
int check_members(const dks_ctx* ctx, int K, dks_ctx* const* members, const char* fn, int C) {
    for (int k = 0; k < K; ++k) {
        const dks_ctx* m = members[k];
        REQUIRE(m && m != ctx && !m->ens_parent && m->ens.empty(),
                "%s: member %d must be a context of its own, not this one, another ensemble or its member", fn, k);
        for (int k2 = 0; k2 < k; ++k2) REQUIRE(members[k2] != m, "%s: member %d appears twice", fn, k);
        REQUIRE(m->device == ctx->device, "%s: member %d is on device %d, the ensemble on %d", fn, k, m->device,
                ctx->device);
        if (m->act != DKS_ACT_TREES && m->act != DKS_ACT_KMACH && m->act != DKS_ACT_MLP && m->act != DKS_ACT_KNN)
            return fail(DKS_ERR_UNSUPPORTED, "%s: member %d is not a tree ensemble, kernel machine, MLP or neighbour model "
                        "(dks_set_tree_model, dks_set_kernel_machine, dks_set_mlp, dks_set_knn_model)", fn, k);
        if (C > 0 && m->C != C)
            return fail(DKS_ERR_UNSUPPORTED, "%s: member %d gives %d outputs, the ensemble %d", fn, k, m->C, C);
    }
    return DKS_OK;
}

// the ensemble takes the checked members over, in order, in place of any it held: they launch on its stream, report into
// its status word and refuse the C ABI from then on
int adopt_members(dks_ctx* ctx, int K, dks_ctx* const* members) {
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    destroy_members(ctx);
    for (int k = 0; k < K; ++k) {
        dks_ctx* m = members[k];
        CUDA_TRY(cudaStreamSynchronize(m->stream));
        if (m->own_stream && m->stream) CUDA_TRY(cudaStreamDestroy(m->stream));
        m->stream = ctx->stream;
        m->own_stream = false;
        m->status.reset();
        m->d_status = ctx->d_status; m->d_counts = ctx->d_counts; m->d_hist = ctx->d_hist;
        m->head = describe_head(m);
        m->ens_parent = ctx;
        ctx->ens.push_back(m);
    }
    return DKS_OK;
}

}  // namespace

extern "C" {

int dks_version(void) { return DKS_VERSION; }

const char* dks_last_error(void) { return g_last_error.c_str(); }

int dks_device_count(int* count) {
    if (!count) return fail(DKS_ERR_INVALID, "dks_device_count: NULL");
    int c = 0;
    if (cudaGetDeviceCount(&c) != cudaSuccess) { cudaGetLastError(); c = 0; }
    *count = c;
    return DKS_OK;
}

int dks_create(dks_ctx** out, int device) {
    if (!out) return fail(DKS_ERR_INVALID, "dks_create: out is NULL");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(DKS_ERR_CUDA, "dks_create: no CUDA device (%s) -- the engine has no CPU fallback",
                    cudaGetErrorString(e));
    if (device < 0 || device >= count) return fail(DKS_ERR_INVALID, "dks_create: device %d out of range [0,%d)", device, count);
    CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(DKS_ERR_UNSUPPORTED, "dks_create: device %d is sm_%d%d; this library is built for sm_90a only", device,
                    prop.major, prop.minor);
    std::unique_ptr<dks_ctx> ctx(new dks_ctx());   // freed with what it holds on any failure below
    ctx->device = device;
    { const char* e = getenv("DKS_GRAPH"); ctx->graph_enabled = !(e && e[0] == '0'); }
    {
        auto env_int = [](const char* name, int dflt) { const char* e = getenv(name); return e ? atoi(e) : dflt; };
        ctx->opt_fused = env_int("DKS_FUSED", 1);
        ctx->opt_fused_warps = env_int("DKS_FUSED_WARPS", 0);
        ctx->opt_fused_B = env_int("DKS_FUSED_B", 0);
        ctx->push_in_kernel = env_int("DKS_PUSH_IN_KERNEL", 0) != 0;
    }
    ctx->sm_count = prop.multiProcessorCount;
    ctx->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
    memset(ctx->h_plans, 0, sizeof(ctx->h_plans));
    CUDA_TRY(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    ctx->own_stream = true;
    for (int i = 0; i < 4; ++i) CUDA_TRY(cudaEventCreate(&ctx->ev[i]));
    for (int i = 0; i < 3; ++i) CUDA_TRY(cudaEventCreate(&ctx->ev_l1[i]));
    CUDA_TRY(cudaStreamCreateWithFlags(&ctx->side_stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
    CUDA_TRY(ctx->d_plans.alloc(DKS_MAX_GROUPS + 1));
    CUDA_TRY(cudaMemset(ctx->d_plans, 0, sizeof(ctx->h_plans)));
    CUDA_TRY(ctx->status.alloc(4 + DKS_MAX_GROUPS + 1));   // status, list counts, histogram
    ctx->d_status = ctx->status;
    ctx->d_counts = ctx->d_status + 2;
    ctx->d_hist = ctx->d_status + 4;
    CUDA_TRY(cudaMemset(ctx->d_status, 0, sizeof(int) * (4 + DKS_MAX_GROUPS + 1)));
    CUDA_TRY(ctx->d_l1.alloc(DKS_L1_MAX_GROUPS + 1));
    CUDA_TRY(cudaMemset(ctx->d_l1, 0, sizeof(dks::l1::Tables) * (DKS_L1_MAX_GROUPS + 1)));
    CUDA_TRY(ctx->d_l1_counts.alloc(2));
    *out = ctx.release();
    return DKS_OK;
}

int dks_destroy(dks_ctx* ctx) {
    if (!ctx) return DKS_OK;
    if (ctx->ens_parent)
        return fail(DKS_ERR_INVALID, "dks_destroy: this context is a member of a soft-voting ensemble, which frees it");
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    destroy_members(ctx);
    delete ctx;
    return DKS_OK;
}

int dks_set_stream(dks_ctx* ctx, void* stream) {
    BIND(ctx);
    if (ctx->own_stream && ctx->stream) {
        CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        CUDA_TRY(cudaStreamDestroy(ctx->stream));
    }
    ctx->stream = (cudaStream_t)stream;
    ctx->own_stream = false;
    for (dks_ctx* m : ctx->ens) m->stream = ctx->stream;     // a soft-voting ensemble's members launch on its stream
    return DKS_OK;
}

int dks_synchronize(dks_ctx* ctx) {
    BIND(ctx);
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return DKS_OK;
}

int dks_set_background(dks_ctx* ctx, const double* bg_host, int N, int D, const double* weights_host) {
    BIND(ctx);
    REQUIRE(bg_host && N > 0 && D > 0, "dks_set_background: need bg, N > 0, D > 0");
    ctx->N = N; ctx->D = D;
    ctx->h_bg.assign(bg_host, bg_host + (size_t)N * D);
    ctx->h_wbg.assign(N, 1.0 / N);
    ctx->uniform_w = true;
    if (weights_host) {
        for (int j = 1; j < N; ++j) if (weights_host[j] != weights_host[0]) ctx->uniform_w = false;
        double sum = 0;
        for (int j = 0; j < N; ++j) sum += weights_host[j];
        REQUIRE(sum > 0, "dks_set_background: weights must have a positive sum");
        for (int j = 0; j < N; ++j) ctx->h_wbg[j] = weights_host[j] / sum;
    }
    ctx->fitted = false;
    return DKS_OK;
}

int dks_set_groups(dks_ctx* ctx, const int32_t* group_offsets, const int32_t* group_cols, int G) {
    BIND(ctx);
    REQUIRE(group_offsets && group_cols && G > 0, "dks_set_groups: need offsets, cols, G > 0");
    if (G > DKS_MAX_GROUPS)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_groups: G=%d groups; this build handles at most %d (sixteen 64-bit words "
                    "of coalition bits per row)", G, DKS_MAX_GROUPS);
    ctx->G = G;
    ctx->h_goff.assign(group_offsets, group_offsets + G + 1);
    ctx->h_gcols.assign(group_cols, group_cols + group_offsets[G]);
    ctx->fitted = false;
    return DKS_OK;
}

int dks_set_model(dks_ctx* ctx, const double* W_host, const double* b_host, int R, int activation, double kappa,
                  int scalar_out) {
    BIND(ctx);
    REQUIRE(ctx->D > 0, "dks_set_model: call dks_set_background first (D unknown)");
    REQUIRE(W_host && b_host && R > 0, "dks_set_model: need W, b, R > 0");
    if (R > 8) return fail(DKS_ERR_UNSUPPORTED, "dks_set_model: R=%d score rows; at most 8 supported", R);
    if (activation == DKS_ACT_MIX) return fail(DKS_ERR_INVALID, "dks_set_model: the mixture head is set by dks_set_mixture");
    if (activation == DKS_ACT_BINARY_LOGISTIC) {
        REQUIRE(R == 1, "binary-logistic head needs R == 1 (got %d)", R);
        REQUIRE(kappa > 0, "binary-logistic head needs kappa > 0");
        ctx->C = 2;
    } else if (activation == DKS_ACT_IDENTITY) {
        ctx->C = R;
    } else if (activation == DKS_ACT_SOFTMAX) {
        REQUIRE(R >= 2, "softmax head needs at least two score rows (got %d)", R);
        ctx->C = R;
    } else if (activation == DKS_ACT_OVR) {
        REQUIRE(R >= 3, "one-vs-rest head needs at least three score rows (got %d)", R);
        REQUIRE(kappa == 1.0, "one-vs-rest head needs kappa == 1 (got %g)", kappa);
        ctx->C = R;
    } else if (activation == DKS_ACT_EXP) {
        REQUIRE(R == 1, "exp head needs R == 1 (got %d)", R);
        ctx->C = 1;
    } else {
        return fail(DKS_ERR_INVALID, "dks_set_model: unknown activation %d", activation);
    }
    ctx->R = R; ctx->act = activation; ctx->kappa = kappa; ctx->scalar_out = scalar_out;
    ctx->h_cm_hdr.clear(); ctx->h_cm_keys.clear(); ctx->h_cm_vals.clear();   // maps belong to one model
    ctx->h_ehdr.clear(); ctx->h_eops.clear(); ctx->h_eopv.clear(); ctx->h_etab.clear();   // so does a column encoding
    ctx->h_W.assign(W_host, W_host + (size_t)R * ctx->D);
    ctx->h_b.assign(b_host, b_host + R);
    ctx->fitted = false;
    return DKS_OK;
}

int dks_set_mixture(dks_ctx* ctx, int K, int member_act, int R_m, const double* W_host, const double* b_host,
                    const double* pi_host, int scalar_out) {
    BIND(ctx);
    REQUIRE(ctx->D > 0, "dks_set_mixture: call dks_set_background first (D unknown)");
    REQUIRE(W_host && b_host && pi_host, "dks_set_mixture: need W, b, pi");
    REQUIRE(K >= 2, "dks_set_mixture: K=%d members; a single model is set by dks_set_model", K);
    if (member_act == DKS_ACT_BINARY_LOGISTIC) {
        REQUIRE(R_m == 1, "dks_set_mixture: binary-logistic members have one score row (got %d)", R_m);
    } else if (member_act == DKS_ACT_SOFTMAX || member_act == DKS_ACT_OVR) {
        if (R_m < 3 || R_m > 8)
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_mixture: softmax / one-vs-rest members over %d classes; 3..8 supported", R_m);
    } else {
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_mixture: member head %d; binary-logistic, softmax or one-vs-rest only",
                    member_act);
    }
    if ((long long)K * R_m > DKS_MIX_MAX_R)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_mixture: %d members x %d score rows exceed %d rows", K, R_m, DKS_MIX_MAX_R);
    double sum = 0.0;
    for (int k = 0; k < K; ++k) {
        REQUIRE(std::isfinite(pi_host[k]) && pi_host[k] > 0.0, "dks_set_mixture: pi[%d] = %g must be positive and finite", k,
                pi_host[k]);
        sum += pi_host[k];
    }
    const int R = K * R_m;
    MixHead mh = {};
    mh.K = K; mh.Rm = R_m; mh.mact = member_act;
    for (int k = 0; k < K; ++k) { mh.pi[k] = pi_host[k] / sum; mh.pif[k] = (float)mh.pi[k]; }
    ctx->mix = mh;
    ctx->C = member_act == DKS_ACT_BINARY_LOGISTIC ? 2 : R_m;
    ctx->R = R; ctx->act = DKS_ACT_MIX; ctx->kappa = 1.0; ctx->scalar_out = scalar_out;
    ctx->h_cm_hdr.clear(); ctx->h_cm_keys.clear(); ctx->h_cm_vals.clear();
    ctx->h_ehdr.clear(); ctx->h_eops.clear(); ctx->h_eopv.clear(); ctx->h_etab.clear();
    ctx->h_W.assign(W_host, W_host + (size_t)R * ctx->D);
    ctx->h_b.assign(b_host, b_host + R);
    ctx->fitted = false;
    return DKS_OK;
}

int dks_set_tree_model(dks_ctx* ctx, int n_nodes, const int32_t* feature, const double* threshold, const int32_t* left,
                       const int32_t* right, const uint8_t* missing_left, const double* value, int R, int n_trees,
                       const int32_t* roots, const double* base, int head, int cmp, int scalar_out) {
    BIND(ctx);
    REQUIRE(ctx->D > 0, "dks_set_tree_model: call dks_set_background first (D unknown)");
    REQUIRE(n_nodes > 0 && n_trees > 0 && feature && threshold && left && right && missing_left && value && roots && base,
            "dks_set_tree_model: need the node arrays, roots and base");
    if (R < 1 || R > DKS_TREE_MAX_R)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_tree_model: R=%d raw scores; 1..%d supported", R, DKS_TREE_MAX_R);
    if (cmp != DKS_TREE_CMP_F32 && cmp != DKS_TREE_CMP_F64)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_tree_model: unknown comparison %d", cmp);
    int C;
    switch (head) {
    case DKS_TREE_HEAD_IDENTITY: C = R; break;
    case DKS_TREE_HEAD_SIGMOID: REQUIRE(R == 1, "sigmoid tree head needs R == 1 (got %d)", R); C = 2; break;
    case DKS_TREE_HEAD_SOFTMAX: REQUIRE(R >= 2, "softmax tree head needs R >= 2 (got %d)", R); C = R; break;
    case DKS_TREE_HEAD_EXP: REQUIRE(R == 1, "exp tree head needs R == 1 (got %d)", R); C = 1; break;
    case DKS_TREE_HEAD_IFOREST: REQUIRE(R == 1, "anomaly tree head needs R == 1 (got %d)", R); C = 1; break;
    default: return fail(DKS_ERR_UNSUPPORTED, "dks_set_tree_model: unknown head %d", head);
    }
    const int width = model_columns(ctx);
    for (int nd = 0; nd < n_nodes; ++nd) {
        const int f = feature[nd];
        if (f < 0) {
            for (int q = 0; q < R; ++q)
                if (!std::isfinite(value[(size_t)nd * R + q]))
                    return fail(DKS_ERR_UNSUPPORTED, "dks_set_tree_model: leaf %d has a non-finite value", nd);
            continue;
        }
        if (f >= width || std::isnan(threshold[nd]) || left[nd] <= nd || right[nd] <= nd || left[nd] >= n_nodes ||
            right[nd] >= n_nodes)
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_tree_model: node %d is malformed (feature %d of %d, children %d / %d "
                        "must follow it)", nd, f, width, left[nd], right[nd]);
    }
    for (int k = 0; k < n_trees; ++k)
        if (roots[k] < 0 || roots[k] >= n_nodes) return fail(DKS_ERR_UNSUPPORTED, "dks_set_tree_model: root %d out of range", k);
    for (int q = 0; q < R; ++q)
        if (!std::isfinite(base[q])) return fail(DKS_ERR_UNSUPPORTED, "dks_set_tree_model: base must be finite");
    ctx->h_tfeat.assign(feature, feature + n_nodes);
    ctx->h_tthr.assign(threshold, threshold + n_nodes);
    ctx->h_tleft.assign(left, left + n_nodes);
    ctx->h_tright.assign(right, right + n_nodes);
    ctx->h_tmiss.assign(missing_left, missing_left + n_nodes);
    ctx->h_tval.assign(value, value + (size_t)n_nodes * R);
    ctx->h_troots.assign(roots, roots + n_trees);
    ctx->h_tbase.assign(base, base + R);
    ctx->tree.nodes = n_nodes; ctx->tree.T = n_trees; ctx->tree.R = R; ctx->tree.head = head; ctx->tree.cmp = cmp;
    ctx->tree.offset = 0.0;
    return set_own_model(ctx, DKS_ACT_TREES, C, scalar_out);
}

int dks_set_tree_offset(dks_ctx* ctx, double offset) {
    BIND(ctx);
    REQUIRE(ctx->act == DKS_ACT_TREES && ctx->tree.head == DKS_TREE_HEAD_IFOREST,
            "dks_set_tree_offset: needs a tree ensemble with the anomaly head (dks_set_tree_model, DKS_TREE_HEAD_IFOREST)");
    if (!std::isfinite(offset)) return fail(DKS_ERR_UNSUPPORTED, "dks_set_tree_offset: the offset must be finite");
    ctx->tree.offset = offset;
    ctx->fitted = false;
    return DKS_OK;
}

int dks_set_kernel_machine(dks_ctx* ctx, int K, const int32_t* sv_off, const double* sv, const double* dual, int R,
                           const double* intercept, const double* colw, const double* colo, const double* gamma, int kernel,
                           double degree, double coef0, int head, const double* cal_a, const double* cal_b,
                           const double* pi, int scalar_out) {
    BIND(ctx);
    REQUIRE(ctx->D > 0, "dks_set_kernel_machine: call dks_set_background first (D unknown)");
    REQUIRE(sv_off && sv && dual && intercept && colw && colo && gamma,
            "dks_set_kernel_machine: need the support vectors, dual coefficients, intercepts, column weights and gamma");
    const int D = model_columns(ctx);
    if (K < 1 || K > DKS_KM_MAX_K)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: K=%d members; 1..%d supported", K, DKS_KM_MAX_K);
    if (R < 1 || R > DKS_KM_MAX_R)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: R=%d outputs; 1..%d supported", R, DKS_KM_MAX_R);
    if (kernel < DKS_KM_KERNEL_RBF || kernel > DKS_KM_KERNEL_PROGRAM)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: unknown kernel %d", kernel);
    if (kernel == DKS_KM_KERNEL_PROGRAM && (K != 1 || head != DKS_KM_HEAD_IDENTITY))
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: the program kernel takes one member and the identity head");
    if (!std::isfinite(coef0) || !std::isfinite(degree) ||
        (kernel == DKS_KM_KERNEL_POLY && (degree < 0 || degree != std::floor(degree))))
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: degree %g / coef0 %g (degree: an integer >= 0)", degree, coef0);
    int C;
    if (head == DKS_KM_HEAD_IDENTITY) {
        if (K != 1) return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: the identity head takes one member (K=%d)", K);
        C = R;
    } else if (head == DKS_KM_HEAD_CALIBRATED) {
        if (R != 1) return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: the calibrated head needs R == 1 (got %d)", R);
        if (!cal_a || !cal_b || !pi || !all_finite(cal_a, K) || !all_finite(cal_b, K))
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: the calibrated head needs finite a, b and pi");
        C = 2;
    } else {
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: unknown head %d", head);
    }
    if (sv_off[0] != 0) return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: sv_off[0] must be 0");
    for (int m = 0; m < K; ++m)
        if (sv_off[m + 1] < sv_off[m])
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: sv_off must not decrease (member %d)", m);
    const int n_sv = sv_off[K];
    if (n_sv < 1) return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: no support vectors");
    if (!all_finite(sv, (size_t)n_sv * D) || !all_finite(dual, (size_t)n_sv * R) || !all_finite(intercept, (size_t)K * R) ||
        !all_finite(colw, (size_t)K * D) || !all_finite(colo, (size_t)K * D) || !all_finite(gamma, K))
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: the arrays must be finite");
    for (size_t e = 0; e < (size_t)K * D; ++e)
        if (!(colw[e] > 0)) return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: column weights must be positive");
    double pisum = 0;
    for (int m = 0; m < K; ++m) {
        if (!(gamma[m] >= 0)) return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: gamma must be >= 0");
        if (head == DKS_KM_HEAD_CALIBRATED) {
            if (!(pi[m] > 0) || !std::isfinite(pi[m]))
                return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_machine: pi must be positive and finite");
            pisum += pi[m];
        }
    }
    KmDev& k = ctx->km;
    for (int m = 0; m <= K; ++m) k.sv_off[m] = sv_off[m];
    for (int m = 0; m < K; ++m) {
        k.gamma[m] = gamma[m];
        for (int q = 0; q < R; ++q) k.icpt[m * R + q] = intercept[m * R + q];
        k.cal_a[m] = head == DKS_KM_HEAD_CALIBRATED ? cal_a[m] : 0.0;
        k.cal_b[m] = head == DKS_KM_HEAD_CALIBRATED ? cal_b[m] : 0.0;
        k.pi[m] = head == DKS_KM_HEAD_CALIBRATED ? pi[m] / pisum : 1.0;
    }
    k.degree = degree; k.coef0 = coef0; k.K = K; k.R = R; k.n_sv = n_sv; k.kernel = kernel; k.head = head;
    ctx->h_ksv.assign(sv, sv + (size_t)n_sv * D);
    ctx->h_kdual.assign(dual, dual + (size_t)n_sv * R);
    ctx->h_kcolw.assign(colw, colw + (size_t)K * D);
    ctx->h_kcolo.assign(colo, colo + (size_t)K * D);
    ctx->kprog = KmProg{};
    ctx->h_kpcolw.clear(); ctx->h_kpcolo.clear();
    return set_own_model(ctx, DKS_ACT_KMACH, C, scalar_out);
}

int dks_set_kernel_program(dks_ctx* ctx, int L, const int32_t* kinds, const double* colw, const double* colo, int n_ops,
                           const int32_t* ops, const int32_t* args, const double* a, const double* b) {
    BIND(ctx);
    REQUIRE(ctx->act == DKS_ACT_KMACH && ctx->km.kernel == DKS_KM_KERNEL_PROGRAM,
            "dks_set_kernel_program: needs a kernel machine set with DKS_KM_KERNEL_PROGRAM (dks_set_kernel_machine)");
    REQUIRE(kinds && colw && colo && ops && args && a && b,
            "dks_set_kernel_program: need the statistic kinds, column weights and origins and the instructions");
    const int D = model_columns(ctx);
    if (L < 1 || L > DKS_KM_MAX_STATS)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: L=%d statistics; 1..%d supported", L, DKS_KM_MAX_STATS);
    if (n_ops < 1 || n_ops > DKS_KM_MAX_OPS)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: %d instructions; 1..%d supported", n_ops, DKS_KM_MAX_OPS);
    for (int l = 0; l < L; ++l)
        if (kinds[l] != DKS_KM_STAT_SQDIST && kinds[l] != DKS_KM_STAT_DOT)
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: unknown statistic kind %d", kinds[l]);
    if (!all_finite(colw, (size_t)L * D) || !all_finite(colo, (size_t)L * D))
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: the column weights and origins must be finite");
    for (size_t e = 0; e < (size_t)L * D; ++e)
        if (!(colw[e] > 0)) return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: column weights must be positive");
    int depth = 0;
    for (int i = 0; i < n_ops; ++i) {
        const int op = ops[i];
        if (op < DKS_KM_OP_CONST || op > DKS_KM_OP_MULC)
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: unknown instruction %d at %d", op, i);
        if (!std::isfinite(a[i]) || !std::isfinite(b[i]))
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: non-finite constant at instruction %d", i);
        if (op == DKS_KM_OP_EXPSINE && (a[i] == 0.0 || b[i] == 0.0))
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: zero periodicity or length scale at instruction %d", i);
        if (op >= DKS_KM_OP_CONST && op <= DKS_KM_OP_EXPSINE) {
            if (op != DKS_KM_OP_CONST && (args[i] < 0 || args[i] >= L))
                return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: statistic %d at instruction %d (L=%d)", args[i], i, L);
            if (++depth > DKS_KM_MAX_STACK)
                return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: more than %d operands at instruction %d",
                            DKS_KM_MAX_STACK, i);
        } else if (op == DKS_KM_OP_ADD || op == DKS_KM_OP_MUL) {
            if (--depth < 1) return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: stack underflow at instruction %d", i);
        } else if (depth < 1) {
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: stack underflow at instruction %d", i);
        }
    }
    if (depth != 1)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_kernel_program: the expression leaves %d values (1 expected)", depth);
    KmProg g = {};
    g.L = L; g.n = n_ops;
    for (int l = 0; l < L; ++l) g.kind[l] = kinds[l];
    for (int i = 0; i < n_ops; ++i) {
        g.op[i] = (signed char)ops[i];
        g.arg[i] = (signed char)(ops[i] == DKS_KM_OP_CONST || ops[i] > DKS_KM_OP_EXPSINE ? 0 : args[i]);
        g.a[i] = a[i]; g.b[i] = b[i];
    }
    ctx->kprog = g;
    ctx->h_kpcolw.assign(colw, colw + (size_t)L * D);
    ctx->h_kpcolo.assign(colo, colo + (size_t)L * D);
    ctx->fitted = false;
    return DKS_OK;
}

int dks_set_svc_multiclass(dks_ctx* ctx, int K, int classes, const int32_t* sv_off, const int32_t* cls_off, const double* sv,
                           const double* dual, const double* intercept, const double* colw, const double* colo,
                           const double* gamma, int kernel, double degree, double coef0, int mode, const double* cal_a,
                           const double* cal_b, const double* pi, int scalar_out) {
    BIND(ctx);
    REQUIRE(ctx->D > 0, "dks_set_svc_multiclass: call dks_set_background first (D unknown)");
    REQUIRE(sv_off && cls_off && sv && dual && intercept && colw && colo && gamma,
            "dks_set_svc_multiclass: need the support vectors, class offsets, dual coefficients, intercepts, column weights "
            "and gamma");
    const int D = model_columns(ctx);
    if (K < 1 || K > DKS_KM_MAX_K)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: K=%d members; 1..%d supported", K, DKS_KM_MAX_K);
    if (classes < 3 || classes > DKS_KM_OVO_MAX_CLASSES)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: %d classes; 3..%d supported", classes,
                    DKS_KM_OVO_MAX_CLASSES);
    if (kernel != DKS_KM_KERNEL_RBF && kernel != DKS_KM_KERNEL_POLY && kernel != DKS_KM_KERNEL_SIGMOID)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: kernel %d; rbf, poly and sigmoid supported", kernel);
    if (!std::isfinite(coef0) || !std::isfinite(degree) ||
        (kernel == DKS_KM_KERNEL_POLY && (degree < 0 || degree != std::floor(degree))))
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: degree %g / coef0 %g (degree: an integer >= 0)", degree,
                    coef0);
    const int P = classes * (classes - 1) / 2, R = classes - 1;
    int C;
    if (mode == DKS_KM_OVO_DECISION) {
        if (K != 1) return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: the pair values take one member (K=%d)", K);
        if (P > DKS_KM_MAX_R)
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: %d pair values over %d classes; up to %d outputs", P,
                        classes, DKS_KM_MAX_R);
        C = P;
    } else if (mode == DKS_KM_OVO_PROBA) {
        if (!cal_a || !cal_b || !pi || !all_finite(cal_a, (size_t)K * classes) || !all_finite(cal_b, (size_t)K * classes))
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: the probabilities need finite a, b and pi");
        C = classes;
    } else {
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: unknown mode %d", mode);
    }
    if (sv_off[0] != 0) return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: sv_off[0] must be 0");
    for (int m = 0; m < K; ++m) {
        if (sv_off[m + 1] < sv_off[m])
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: sv_off must not decrease (member %d)", m);
        const int32_t* co = cls_off + (size_t)m * (classes + 1);
        if (co[0] != sv_off[m] || co[classes] != sv_off[m + 1])
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: the class blocks of member %d must span its support "
                        "vectors", m);
        for (int c = 0; c < classes; ++c)
            if (co[c + 1] < co[c])
                return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: cls_off must not decrease (member %d, class %d)",
                            m, c);
    }
    const int n_sv = sv_off[K];
    if (n_sv < 1) return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: no support vectors");
    if (!all_finite(sv, (size_t)n_sv * D) || !all_finite(dual, (size_t)n_sv * R) || !all_finite(intercept, (size_t)K * P) ||
        !all_finite(colw, (size_t)K * D) || !all_finite(colo, (size_t)K * D) || !all_finite(gamma, K))
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: the arrays must be finite");
    for (size_t e = 0; e < (size_t)K * D; ++e)
        if (!(colw[e] > 0)) return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: column weights must be positive");
    double pisum = 0;
    for (int m = 0; m < K; ++m) {
        if (!(gamma[m] >= 0)) return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: gamma must be >= 0");
        if (mode == DKS_KM_OVO_PROBA) {
            if (!(pi[m] > 0) || !std::isfinite(pi[m]))
                return fail(DKS_ERR_UNSUPPORTED, "dks_set_svc_multiclass: pi must be positive and finite");
            pisum += pi[m];
        }
    }
    KmDev& k = ctx->km;
    for (int m = 0; m <= K; ++m) k.sv_off[m] = sv_off[m];
    for (int m = 0; m < K; ++m) {
        k.gamma[m] = gamma[m];
        k.icpt[m] = k.cal_a[m] = k.cal_b[m] = 0.0;      // the one-vs-one head reads its own (KmOvo)
        k.pi[m] = mode == DKS_KM_OVO_PROBA ? pi[m] / pisum : 1.0;
    }
    k.degree = degree; k.coef0 = coef0; k.K = K; k.R = R; k.n_sv = n_sv; k.kernel = kernel; k.head = DKS_KM_HEAD_OVO;
    ctx->h_ksv.assign(sv, sv + (size_t)n_sv * D);
    ctx->h_kdual.assign(dual, dual + (size_t)n_sv * R);
    ctx->h_kcolw.assign(colw, colw + (size_t)K * D);
    ctx->h_kcolo.assign(colo, colo + (size_t)K * D);
    ctx->kprog = KmProg{};
    ctx->h_kpcolw.clear(); ctx->h_kpcolo.clear();
    ctx->h_kocls.assign(cls_off, cls_off + (size_t)K * (classes + 1));
    ctx->h_koicpt.assign(intercept, intercept + (size_t)K * P);
    if (mode == DKS_KM_OVO_PROBA) {
        ctx->h_kocala.assign(cal_a, cal_a + (size_t)K * classes);
        ctx->h_kocalb.assign(cal_b, cal_b + (size_t)K * classes);
    } else {
        ctx->h_kocala.assign((size_t)K * classes, 0.0);
        ctx->h_kocalb.assign((size_t)K * classes, 0.0);
    }
    ctx->kovo = KmOvo{};
    ctx->kovo.classes = classes; ctx->kovo.P = P; ctx->kovo.mode = mode;
    return set_own_model(ctx, DKS_ACT_KMACH, C, scalar_out);
}

int dks_set_mlp(dks_ctx* ctx, int n_hidden, const int32_t* widths, const double* W_host, const double* b_host, int activation,
                int head, int scalar_out) {
    BIND(ctx);
    REQUIRE(ctx->D > 0, "dks_set_mlp: call dks_set_background first (D unknown)");
    REQUIRE(widths && W_host && b_host, "dks_set_mlp: need the widths, weights and biases");
    const int E = encoded_columns(ctx), D = model_columns(ctx);
    if (n_hidden < 1 || n_hidden > DKS_MLP_MAX_HIDDEN)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_mlp: %d hidden layers; 1..%d supported", n_hidden, DKS_MLP_MAX_HIDDEN);
    const int L = n_hidden + 1, R = widths[L];
    if (widths[0] != D)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_mlp: the first layer reads %d columns, the %s has %d", widths[0],
                    E > 0 ? "column encoding" : "background", D);
    for (int l = 1; l < L; ++l)
        if (widths[l] < 1 || widths[l] > DKS_MLP_MAX_WIDTH)
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_mlp: hidden layer %d has %d units; 1..%d supported", l, widths[l],
                        DKS_MLP_MAX_WIDTH);
    if (R < 1 || R > DKS_MLP_MAX_OUT)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_mlp: %d output units; 1..%d supported", R, DKS_MLP_MAX_OUT);
    if (activation < DKS_MLP_ACT_IDENTITY || activation > DKS_MLP_ACT_RELU)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_mlp: unknown activation %d", activation);
    int C;
    switch (head) {
    case DKS_MLP_HEAD_IDENTITY: C = R; break;
    case DKS_MLP_HEAD_SIGMOID:
        if (R != 1) return fail(DKS_ERR_UNSUPPORTED, "dks_set_mlp: the sigmoid head needs one output unit (got %d)", R);
        C = 2;
        break;
    case DKS_MLP_HEAD_SOFTMAX:
        if (R < 2) return fail(DKS_ERR_UNSUPPORTED, "dks_set_mlp: the softmax head needs at least two output units (got %d)", R);
        C = R;
        break;
    default: return fail(DKS_ERR_UNSUPPORTED, "dks_set_mlp: unknown head %d", head);
    }
    MlpDev m = {};
    m.L = L; m.act = activation; m.head = head; m.R = R;
    size_t nw = 0, nb = 0, nwf = 0, nbp = 0;
    for (int l = 0; l <= L; ++l) {
        m.width[l] = widths[l];
        m.pad[l] = l == 0 ? D : l == L ? 8 : dks::mlp::pad16(widths[l]);
    }
    for (int l = 0; l < L; ++l) {
        m.woff[l] = (int)nw; m.boff[l] = (int)nb; m.wfoff[l] = (int)nwf; m.bpoff[l] = (int)nbp;
        nw += (size_t)widths[l] * widths[l + 1];
        nb += (size_t)widths[l + 1];
        if (l > 0) nwf += (size_t)m.pad[l] * m.pad[l + 1];
        nbp += (size_t)m.pad[l + 1];
    }
    if (nw > (size_t)INT32_MAX) return fail(DKS_ERR_UNSUPPORTED, "dks_set_mlp: %zu weights are too many", nw);
    if (!all_finite(W_host, nw)) return fail(DKS_ERR_UNSUPPORTED, "dks_set_mlp: the weights must be finite");
    if (!all_finite(b_host, nb)) return fail(DKS_ERR_UNSUPPORTED, "dks_set_mlp: the biases must be finite");
    m.nbuf = n_hidden >= 2 ? 2 : 1;
    m.hmax = 16;
    for (int l = 1; l < L; ++l) m.hmax = std::max(m.hmax, m.pad[l]);
    // layers 1 .. L - 1 in B-fragment order: element (k, n) of layer l at ((k / 16) * (pad / 8) + n / 8) * 32 + lane, lane =
    // (n % 8) * 4 + k % 4, entry (k % 16) / 4; zero rows and columns pad it.  Every layer's biases zero-padded.
    ctx->h_mwf.assign(nwf, 0.0);
    ctx->h_mbp.assign(nbp, 0.0);
    for (int l = 0; l < L; ++l) {
        const int K = widths[l], H = widths[l + 1], NT = m.pad[l + 1] / 8;
        for (int n = 0; n < H; ++n) ctx->h_mbp[m.bpoff[l] + n] = b_host[m.boff[l] + n];
        if (l == 0) continue;
        for (int k = 0; k < K; ++k)
            for (int n = 0; n < H; ++n) {
                const int kk = k & 15;
                const size_t at = (((size_t)(k >> 4) * NT + (n >> 3)) * 32 + (n & 7) * 4 + (kk & 3)) * 4 + (kk >> 2);
                ctx->h_mwf[m.wfoff[l] + at] = W_host[m.woff[l] + (size_t)k * H + n];
            }
    }
    ctx->h_mw.assign(W_host, W_host + nw);
    ctx->h_mb.assign(b_host, b_host + nb);
    ctx->mlp = m;
    return set_own_model(ctx, DKS_ACT_MLP, C, scalar_out);
}

int dks_set_knn_model(dks_ctx* ctx, int n_fit, const double* fitX, const double* colw, const double* colo, int k, int metric,
                      double p, int weights, int R, const double* labels_or_targets, int head, int scalar_out) {
    BIND(ctx);
    REQUIRE(ctx->D > 0, "dks_set_knn_model: call dks_set_background first (D unknown)");
    REQUIRE(fitX && colw && colo && labels_or_targets, "dks_set_knn_model: need the training rows, column map and labels");
    const int D = model_columns(ctx);
    if (k < 1 || k > DKS_KNN_MAX_K)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_knn_model: k=%d neighbours; 1..%d supported", k, DKS_KNN_MAX_K);
    if (n_fit < k)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_knn_model: %d training rows for k=%d neighbours (need n_fit >= k)", n_fit, k);
    if (metric < DKS_KNN_METRIC_EUCLIDEAN || metric > DKS_KNN_METRIC_SQEUCLIDEAN)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_knn_model: unknown metric %d", metric);
    if (metric == DKS_KNN_METRIC_MINKOWSKI && !(std::isfinite(p) && p >= 1))
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_knn_model: minkowski p=%g (a finite p >= 1)", p);
    if (weights != DKS_KNN_WEIGHTS_UNIFORM && weights != DKS_KNN_WEIGHTS_DISTANCE)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_knn_model: unknown weights %d", weights);
    if (head != DKS_KNN_HEAD_CLASSIFY && head != DKS_KNN_HEAD_REGRESS)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_knn_model: unknown head %d", head);
    const int Rmin = head == DKS_KNN_HEAD_CLASSIFY ? 2 : 1;
    if (R < Rmin || R > DKS_KNN_MAX_R)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_knn_model: R=%d %s; %d..%d supported", R,
                    head == DKS_KNN_HEAD_CLASSIFY ? "classes" : "targets", Rmin, DKS_KNN_MAX_R);
    const size_t ny = head == DKS_KNN_HEAD_CLASSIFY ? (size_t)n_fit : (size_t)n_fit * R;
    if (!all_finite(fitX, (size_t)n_fit * D) || !all_finite(colw, D) || !all_finite(colo, D) || !all_finite(labels_or_targets, ny))
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_knn_model: the arrays must be finite");
    for (int c = 0; c < D; ++c)
        if (colw[c] == 0) return fail(DKS_ERR_UNSUPPORTED, "dks_set_knn_model: column weights must be non-zero");
    if (head == DKS_KNN_HEAD_CLASSIFY)
        for (int v = 0; v < n_fit; ++v) {
            const double l = labels_or_targets[v];
            if (!(l >= 0 && l < R && l == std::floor(l)))
                return fail(DKS_ERR_UNSUPPORTED, "dks_set_knn_model: the label of row %d is not a class index 0..%d", v, R - 1);
        }
    KnnDev& kd = ctx->knn;
    kd.n_fit = n_fit; kd.k = k; kd.metric = metric; kd.p = p; kd.weights = weights; kd.R = R; kd.head = head;
    ctx->h_nfitX.assign(fitX, fitX + (size_t)n_fit * D);
    ctx->h_ncolw.assign(colw, colw + D);
    ctx->h_ncolo.assign(colo, colo + D);
    ctx->h_ny.assign(labels_or_targets, labels_or_targets + ny);
    return set_own_model(ctx, DKS_ACT_KNN, R, scalar_out);
}

int dks_set_gaussian_model(dks_ctx* ctx, int K, int D, const int32_t* r_off, const double* mu, const double* L,
                           const double* gamma, const double* c, int head, int scalar_out) {
    BIND(ctx);
    REQUIRE(ctx->D > 0, "dks_set_gaussian_model: call dks_set_background first (D unknown)");
    REQUIRE(r_off && mu && L && gamma && c, "dks_set_gaussian_model: need r_off, mu, L, gamma and c");
    if (K < 1 || K > DKS_GAUSS_MAX_K)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_gaussian_model: K=%d components; 1..%d supported", K, DKS_GAUSS_MAX_K);
    if (D < 1) return fail(DKS_ERR_UNSUPPORTED, "dks_set_gaussian_model: D=%d columns", D);
    if (head < DKS_GAUSS_HEAD_SOFTMAX || head > DKS_GAUSS_HEAD_DIFF)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_gaussian_model: unknown head %d", head);
    if (head == DKS_GAUSS_HEAD_DIFF && K != 2)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_gaussian_model: the difference head needs K = 2 (K=%d)", K);
    if (r_off[0] != 0)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_gaussian_model: r_off must start at 0");
    for (int k = 0; k < K; ++k)
        if (r_off[k + 1] <= r_off[k])
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_gaussian_model: component %d has rank %d (at least 1)", k,
                        r_off[k + 1] - r_off[k]);
    const int RT = r_off[K];
    if (!all_finite(mu, (size_t)K * D) || !all_finite(L, (size_t)RT * D) || !all_finite(gamma, K) || !all_finite(c, K))
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_gaussian_model: the arrays must be finite");
    for (int k = 0; k < K; ++k)
        if (!(gamma[k] > 0)) return fail(DKS_ERR_UNSUPPORTED, "dks_set_gaussian_model: gamma of component %d is not positive", k);
    GaussDev& g = ctx->gauss;
    g = GaussDev{};
    g.K = K; g.RT = RT; g.head = head;
    for (int k = 0; k <= K; ++k) g.r_off[k] = r_off[k];
    for (int k = 0; k < K; ++k) { g.gamma[k] = gamma[k]; g.c[k] = c[k]; }
    ctx->h_gmu.assign(mu, mu + (size_t)K * D);
    ctx->h_gL.assign(L, L + (size_t)RT * D);
    const int C = head == DKS_GAUSS_HEAD_SOFTMAX || head == DKS_GAUSS_HEAD_IDENTITY ? K : 1;
    return set_own_model(ctx, DKS_ACT_GAUSS, C, scalar_out);
}

int dks_set_ensemble(dks_ctx* ctx, int K, dks_ctx* const* members, const double* weights, int C, int scalar_out) {
    BIND(ctx);
    REQUIRE(ctx->D > 0, "dks_set_ensemble: call dks_set_background first (D unknown)");
    REQUIRE(members && weights, "dks_set_ensemble: need the members and their weights");
    if (K < 1 || K > DKS_ENS_MAX_MEMBERS)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_ensemble: K=%d members; 1..%d supported", K, DKS_ENS_MAX_MEMBERS);
    if (C < 1 || C > DKS_ENS_MAX_OUT)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_ensemble: C=%d outputs; 1..%d supported", C, DKS_ENS_MAX_OUT);
    double wsum = 0;
    for (int k = 0; k < K; ++k) {
        if (!std::isfinite(weights[k]) || weights[k] < 0)
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_ensemble: weights must be finite and non-negative");
        wsum += weights[k];
    }
    if (!(wsum > 0) || !std::isfinite(wsum))
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_ensemble: the weights must have a positive finite sum");
    TRY(check_members(ctx, K, members, "dks_set_ensemble", C));
    TRY(adopt_members(ctx, K, members));
    for (int k = 0; k < K; ++k) ctx->h_ens_pi.push_back(weights[k] / wsum);
    return set_own_model(ctx, DKS_ACT_ENSEMBLE, C, scalar_out);
}

int dks_set_stacking(dks_ctx* ctx, int K, dks_ctx* const* members, const int32_t* col_first, const int32_t* col_count,
                     const double* W, const double* b, int R, int head, const double* W_pass, int C, int scalar_out,
                     int64_t workspace_bytes) {
    BIND(ctx);
    REQUIRE(ctx->D > 0, "dks_set_stacking: call dks_set_background first (D unknown)");
    REQUIRE(members && col_first && col_count && W && b, "dks_set_stacking: need the members, their columns, W and b");
    if (K < 1 || K > DKS_ENS_MAX_MEMBERS)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_stacking: K=%d members; 1..%d supported", K, DKS_ENS_MAX_MEMBERS);
    if (C < 1 || C > DKS_ENS_MAX_OUT)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_stacking: C=%d outputs; 1..%d supported", C, DKS_ENS_MAX_OUT);
    const bool heads_ok = (head == DKS_STACK_HEAD_IDENTITY && R == C) || (head == DKS_STACK_HEAD_SIGMOID && R == 1 && C == 2) ||
                          (head == DKS_STACK_HEAD_SOFTMAX && R == C && R >= 2);
    if (!heads_ok)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_stacking: head %d with R=%d scores and C=%d outputs (identity: R = C; "
                    "sigmoid: R = 1, C = 2; softmax: R = C >= 2)", head, R, C);
    REQUIRE(workspace_bytes > 0, "dks_set_stacking: the workspace budget must be positive");
    int F = 0;
    TRY(check_members(ctx, K, members, "dks_set_stacking", 0));
    for (int k = 0; k < K; ++k) {
        const dks_ctx* m = members[k];
        if (col_count[k] < 1 || col_first[k] < 0 || col_first[k] + col_count[k] > m->C)
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_stacking: member %d keeps outputs %d..%d of its %d", k, col_first[k],
                        col_first[k] + col_count[k] - 1, m->C);
        F += col_count[k];
    }
    if (F > DKS_STACK_MAX_F)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_stacking: F=%d meta columns; at most %d", F, DKS_STACK_MAX_F);
    const int width = model_columns(ctx);
    if (!all_finite(W, (size_t)R * F) || !all_finite(b, R) || (W_pass && !all_finite(W_pass, (size_t)R * width)))
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_stacking: the final estimator's weights must be finite");
    TRY(adopt_members(ctx, K, members));
    StackDev& sd = ctx->stk;
    sd = StackDev{};
    sd.K = K; sd.F = F; sd.R = R; sd.C = C; sd.head = head; sd.D = width;
    for (int k = 0; k < K; ++k) {
        sd.ck[k] = members[k]->C; sd.cfirst[k] = col_first[k]; sd.ccount[k] = col_count[k];
    }
    ctx->h_stk_W.assign(W, W + (size_t)R * F);
    ctx->h_stk_b.assign(b, b + R);
    if (W_pass) ctx->h_stk_Wp.assign(W_pass, W_pass + (size_t)R * width);
    else ctx->h_stk_Wp.clear();
    ctx->stk_budget = workspace_bytes;
    return set_own_model(ctx, DKS_ACT_STACKING, C, scalar_out);
}

int dks_set_column_maps(dks_ctx* ctx, int D, int R, const int32_t* hdr_host, const double* keys_host, int n_keys,
                        const double* vals_host, int n_vals) {
    BIND(ctx);
    ctx->fitted = false;
    if (hdr_host == nullptr) {             // back to the scores W x + b
        ctx->h_cm_hdr.clear(); ctx->h_cm_keys.clear(); ctx->h_cm_vals.clear();
        return DKS_OK;
    }
    REQUIRE(ctx->R > 0, "dks_set_column_maps: call dks_set_model first");
    const OwnKernel ok = own_kernel(describe_head(ctx).family);
    if (ok.family) return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_maps: not for %s%s", ok.family, ok.maps_note);
    if (D != ctx->D || R != ctx->R)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_maps: maps of %d columns x %d score rows, model has %d x %d", D, R,
                    ctx->D, ctx->R);
    if (n_keys < 0 || n_vals < 1 || (n_keys > 0 && !keys_host) || !vals_host)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_maps: bad table sizes");
    for (int c = 0; c < D; ++c) {
        const int flags = hdr_host[4 * c], m = hdr_host[4 * c + 1], ko = hdr_host[4 * c + 2], vo = hdr_host[4 * c + 3];
        const bool cat = flags & DKS_CM_CATEGORICAL;
        const long long nk = cat ? m : (long long)m - 1;
        const long long nv = (long long)R * (cat ? m + 2 : 2 * (long long)m + 1);
        if ((flags & ~(DKS_CM_CATEGORICAL | DKS_CM_NAN_ERROR | DKS_CM_UNKNOWN_ERROR)) || (!cat && (flags & DKS_CM_UNKNOWN_ERROR)) ||
            m < 1 || ko < 0 || vo < 0 || ko + nk > n_keys || vo + nv > n_vals)
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_maps: malformed header of column %d", c);
        for (long long k = 0; k < nk; ++k) {
            const double t = keys_host[ko + k];
            if (!std::isfinite(t) || (k > 0 && !(keys_host[ko + k - 1] < t)))
                return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_maps: column %d: %s must be finite and strictly increasing",
                            c, cat ? "keys" : "breakpoints");
        }
        for (long long k = 0; k < nv; ++k)
            if (!std::isfinite(vals_host[vo + k]))
                return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_maps: column %d: values must be finite", c);
    }
    ctx->h_cm_hdr.assign(hdr_host, hdr_host + 4 * (size_t)D);
    ctx->h_cm_keys.assign(keys_host, keys_host + n_keys);
    ctx->h_cm_vals.assign(vals_host, vals_host + n_vals);
    return DKS_OK;
}

int dks_set_column_encoding(dks_ctx* ctx, int E, const int32_t* hdr_host, const int32_t* ops_host, const double* opvals_host,
                            int n_ops, const double* tab_host, int n_tab) {
    BIND(ctx);
    ctx->fitted = false;
    if (hdr_host == nullptr) {
        ctx->h_ehdr.clear(); ctx->h_eops.clear(); ctx->h_eopv.clear(); ctx->h_etab.clear();
        return DKS_OK;
    }
    REQUIRE(ctx->D > 0, "dks_set_column_encoding: call dks_set_background first (D unknown)");
    if (ctx->act >= 0 && !describe_head(ctx).own())
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_encoding: for models with their own kernels only (linear models read "
                    "their pipelines through dks_set_column_maps)");
    if (E < 1 || n_ops < 0 || n_tab < 0 || (n_ops > 0 && (!ops_host || !opvals_host)) || (n_tab > 0 && !tab_host))
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_encoding: bad sizes");
    for (int e = 0; e < E; ++e) {
        const int src = hdr_host[3 * e], first = hdr_host[3 * e + 1], count = hdr_host[3 * e + 2];
        if (src < 0 || src >= ctx->D || first < 0 || count < 0 || (long long)first + count > n_ops)
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_encoding: malformed header of encoded column %d (source %d of "
                        "%d, ops %d + %d of %d)", e, src, ctx->D, first, count, n_ops);
    }
    for (int k = 0; k < n_ops; ++k) {
        const int code = ops_host[4 * k], flags = ops_host[4 * k + 1], m = ops_host[4 * k + 2], off = ops_host[4 * k + 3];
        const double c0 = opvals_host[2 * k], c1 = opvals_host[2 * k + 1];
        if (code < DKS_ENC_OP_SUB || code > DKS_ENC_OP_TABLE)
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_encoding: op %d: unknown code %d", k, code);
        if (code < DKS_ENC_OP_PIECES) {
            if (flags != 0 || !std::isfinite(c0) || (code == DKS_ENC_OP_CLIP && !(std::isfinite(c1) && c0 <= c1)))
                return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_encoding: op %d: flags must be 0 and constants finite", k);
            continue;
        }
        const int allowed = DKS_ENC_NAN_ERROR | (code == DKS_ENC_OP_TABLE ? DKS_ENC_UNKNOWN_ERROR : 0);
        if ((flags & ~allowed) || m < 0 || off < 0 || (long long)off + 2 * (long long)m + 2 > n_tab)
            return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_encoding: op %d: malformed lookup (flags %d, m %d, offset %d of "
                        "%d)", k, flags, m, off, n_tab);
        for (int q = 0; q < m; ++q) {
            const double t = tab_host[off + q];
            if (!std::isfinite(t) || (q > 0 && !(tab_host[off + q - 1] < t)))
                return fail(DKS_ERR_UNSUPPORTED, "dks_set_column_encoding: op %d: %s must be finite and strictly increasing",
                            k, code == DKS_ENC_OP_PIECES ? "edges" : "keys");
        }
    }
    ctx->h_ehdr.assign(hdr_host, hdr_host + 3 * (size_t)E);
    ctx->h_eops.assign(ops_host, ops_host + 4 * (size_t)n_ops);
    ctx->h_eopv.assign(opvals_host, opvals_host + 2 * (size_t)n_ops);
    ctx->h_etab.assign(tab_host, tab_host + n_tab);
    if (ctx->h_eops.empty()) ctx->h_eops.assign(4, 0), ctx->h_eopv.assign(2, 0.0);   // device copies are never empty
    if (ctx->h_etab.empty()) ctx->h_etab.assign(1, 0.0);
    return DKS_OK;
}

int dks_encode_host(dks_ctx* ctx, const double* X_host, int n, double* out_host) {
    BIND(ctx);
    REQUIRE(ctx->fitted && ctx->enc.E > 0, "dks_encode_host: call dks_fit with a column encoding set first");
    REQUIRE(X_host && out_host && n > 0, "dks_encode_host: bad arguments");
    const int E = ctx->enc.E;
    DevBuf<double> dX, dO;
    CUDA_TRY(dX.alloc((size_t)n * ctx->D));
    CUDA_TRY(dO.alloc((size_t)n * E));
    CUDA_TRY(cudaMemcpyAsync(dX, X_host, sizeof(double) * n * ctx->D, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(ctx->d_status, 0, sizeof(int) * 2, ctx->stream));
    TRY(launch_encode(ctx, dX, n, dO));
    CUDA_TRY(cudaMemcpyAsync(out_host, dO, sizeof(double) * n * E, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(ctx->h_status, ctx->d_status, sizeof(int) * 2, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (ctx->h_status[0] == DKS_ERR_DOMAIN) return fail_refused(ctx, "row");
    return DKS_OK;
}

int dks_set_link(dks_ctx* ctx, int link) {
    BIND(ctx);
    REQUIRE(link == DKS_LINK_IDENTITY || link == DKS_LINK_LOGIT, "dks_set_link: unknown link %d", link);
    ctx->link = link;
    ctx->fitted = false;
    return DKS_OK;
}

int dks_fit(dks_ctx* ctx) {
    BIND(ctx);
    return fit_model(ctx);
}
int dks_num_outputs(dks_ctx* ctx, int* C) {
    BIND(ctx);
    REQUIRE(C, "dks_num_outputs: NULL");
    *C = ctx->C;
    return DKS_OK;
}

int dks_get_fnull(dks_ctx* ctx, double* fnull_host, double* expected_value_host) {
    BIND(ctx);
    REQUIRE(ctx->fitted, "dks_get_fnull: call dks_fit first");
    for (int c = 0; c < ctx->C; ++c) {
        if (fnull_host) fnull_host[c] = ctx->h_fnull[c];
        if (expected_value_host) expected_value_host[c] = ctx->h_linkfnull[c];
    }
    return DKS_OK;
}

int dks_predict_host(dks_ctx* ctx, const double* X_host, int n, double* out_host) {
    BIND(ctx);
    REQUIRE(ctx->fitted, "dks_predict_host: call dks_fit first");
    REQUIRE(X_host && out_host && n > 0, "dks_predict_host: bad arguments");
    DevBuf<double> dX, dO;
    CUDA_TRY(dX.alloc((size_t)n * ctx->D));
    CUDA_TRY(dO.alloc((size_t)n * ctx->C));
    CUDA_TRY(cudaMemcpyAsync(dX, X_host, sizeof(double) * n * ctx->D, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(ctx->d_status, 0, sizeof(int) * 2, ctx->stream));
    DevBuf<double> dXe;                // a model with its own kernel behind a column encoding reads the encoded rows
    if (ctx->head.own()) {
        if (ctx->enc.E > 0) CUDA_TRY(dXe.alloc((size_t)n * ctx->enc.E));
        TRY(launch_own_predict(ctx, dX, n, dXe, nullptr, dO, nullptr));
    } else {
        (ctx->cm.hdr ? dks::predict_kernel<true> : dks::predict_kernel<false>)<<<cdiv(n, 128), 128, 0, ctx->stream>>>(
            dX, ctx->d_W, ctx->d_b, n, ctx->D, ctx->R, ctx->C, ctx->act, ctx->kappa, dO, ctx->cm, ctx->d_status, ctx->d_mix);
        ctx->launches += 1;
    }
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(out_host, dO, sizeof(double) * n * ctx->C, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(ctx->h_status, ctx->d_status, sizeof(int) * 2, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (ctx->h_status[0] == DKS_ERR_DOMAIN) return fail_refused(ctx, "row");
    return DKS_OK;
}

int dks_set_nsamples(dks_ctx* ctx, int nsamples) {
    BIND(ctx);
    REQUIRE(nsamples >= 0, "dks_set_nsamples: nsamples must be >= 0 (0 = auto)");
    ctx->nsamples_req = nsamples;
    return DKS_OK;
}

int dks_effective_nsamples(dks_ctx* ctx, int M, int* S) {
    REQUIRE(ctx && S && M >= 0, "dks_effective_nsamples: bad arguments");
    *S = dks_effective_S(M, ctx->nsamples_req);
    return DKS_OK;
}

// uploads a plan of M groups and factors its normal matrix (plans of more than 128 groups: the host hands the projection
// over with dks_set_plan_projection)
static int upload_plan(dks_ctx* ctx, int M, int S, const uint64_t* zbits_host, const double* w_host, PlanDev* out) {
    DevPool& pool = ctx->plan_pool[M];
    uint64_t* dz; double* dw; double* dc = nullptr; double* di = nullptr;
    const int W = dks_plan_words(M);                        // 64-bit words per coalition row
    const size_t S_even = ((size_t)S + 1) & ~(size_t)1;     // TMA bulk copies move 16-byte multiples
    CUDA_TRY(pool.alloc(&dz, S_even * W));
    CUDA_TRY(pool.alloc(&dw, S_even));
    CUDA_TRY(cudaMemsetAsync(dz, 0, sizeof(uint64_t) * S_even * W, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(dw, 0, sizeof(double) * S_even, ctx->stream));
    if (W <= 2) {
        CUDA_TRY(pool.alloc(&dc, (size_t)(M - 1) * (M - 1)));
        CUDA_TRY(pool.alloc(&di, (size_t)(M - 1) * (M - 1)));
    }
    CUDA_TRY(cudaMemcpyAsync(dz, zbits_host, sizeof(uint64_t) * S * W, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(dw, w_host, sizeof(double) * S, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(ctx->d_status, 0, sizeof(int) * 2, ctx->stream));
    if (W == 1) {
        size_t smem = 2 * sizeof(double) * (size_t)(M - 1) * (M - 1);
        CUDA_TRY(cudaFuncSetAttribute(dks::plan_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        dks::plan_factor_kernel<<<1, 256, smem, ctx->stream>>>(dz, dw, S, M, dc, di, ctx->d_status);
        ctx->launches += 1;
    } else if (W == 2) {
        double* scratch;
        CUDA_TRY(pool.alloc(&scratch, (size_t)(M - 1) * (M - 1)));
        size_t smem = sizeof(double) * (size_t)(M - 1) * (M - 1);
        CUDA_TRY(cudaFuncSetAttribute(dks::plan_factor_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        dks::plan_factor_wide_kernel<<<1, 1024, smem, ctx->stream>>>(dz, dw, S, M, dc, di, scratch, ctx->d_status);
        ctx->launches += 1;
    }
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(ctx->h_status, ctx->d_status, sizeof(int) * 2, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (ctx->h_status[0] != 0)
        return fail(DKS_ERR_NUMERIC, "dks_set_shared_plan: normal matrix of the M=%d plan is not positive definite", M);
    PlanDev& pd = *out;
    memset(&pd, 0, sizeof(pd));
    pd.z = dz; pd.w = dw; pd.chol = dc; pd.ainv = di; pd.S = S; pd.W = W;
    pd.S_pad = (S + 31) / 32 * 32;
    return DKS_OK;
}

// the binary head's Dm table and row exponents of a plan, from background contributions BW and scores (one member's for
// a mixture)
static int build_dm_tables(dks_ctx* ctx, const PlanDev& pd, int M, const double* BW, const double* scores, double scale,
                           const float** dm_out, const double** dme_out) {
    const int N = ctx->N;
    float* dm;
    double* dme;
    CUDA_TRY(ctx->plan_pool[M].alloc(&dm, (size_t)N * pd.S_pad));
    CUDA_TRY(ctx->plan_pool[M].alloc(&dme, (size_t)pd.S_pad));
    const long long total = (long long)N * pd.S_pad;
    dks::shared_path::plan_dme_kernel<<<cdiv(pd.S_pad, 128), 128, 0, ctx->stream>>>(pd.z, pd.W, pd.S, pd.S_pad, BW, scores, N,
                                                                                   M, scale, dme);
    dks::shared_path::plan_dm_kernel<<<cdiv(total, 256), 256, 0, ctx->stream>>>(pd.z, pd.W, pd.S, pd.S_pad, BW, scores, N, M,
                                                                                  scale, dme, dm);
    ctx->launches += 2;
    CUDA_TRY(cudaGetLastError());
    *dm_out = dm; *dme_out = dme;
    return DKS_OK;
}

// the softmax / one-vs-rest tables of a plan over C classes (dks_multi.cuh): per-class Dm [CS][N][S_pad] and row bounds
// [CS][S_pad], the one-vs-rest head keeping one more slot of each (CS = C + 1: nd per element, hi per row)
static int build_class_tables(dks_ctx* ctx, const PlanDev& pd, int M, const double* BW, const double* scores, int C,
                              double scale, const float** dm_out, const float** lo_out) {
    const bool ovr = ctx->head.ovr;
    const int CS = ovr ? C + 1 : C;
    float* sd; float* sl;
    CUDA_TRY(ctx->plan_pool[M].alloc(&sd, (size_t)CS * ctx->N * pd.S_pad));
    CUDA_TRY(ctx->plan_pool[M].alloc(&sl, (size_t)CS * pd.S_pad));
    auto kern = ovr ? (pd.W == 1 ? dks::multi::plan_ovr_kernel<1> : dks::multi::plan_ovr_kernel<2>)
                    : (pd.W == 1 ? dks::multi::plan_softmax_kernel<1> : dks::multi::plan_softmax_kernel<2>);
    kern<<<cdiv(pd.S_pad, 128), 128, 0, ctx->stream>>>(pd.z, pd.S, pd.S_pad, BW, scores, ctx->N, M, C, scale, sd, sl);
    ctx->launches += 1;
    CUDA_TRY(cudaGetLastError());
    *dm_out = sd; *lo_out = sl;
    return DKS_OK;
}

// what the shared-plan route of the head reads besides the plan, for the full varying set (M == G)
static int build_full_set_tables(dks_ctx* ctx, PlanDev& pd, int M) {
    const HeadDesc& h = ctx->head;
    FullSetTables& ft = ctx->full;
    ft = FullSetTables{};
    const MixHead& mh = ctx->mix;
    const int N = ctx->N;
    switch (h.shared) {
    case HEAD_SHARED_BINARY:
        TRY(build_dm_tables(ctx, pd, M, ctx->d_BW, ctx->d_scores, h.scale, &pd.dmT, &pd.dme));
        TRY(build_pmat(ctx, pd, M));
        // float64 P, row-major per coalition, for the fused kernel (link + solve inside the coalition kernel)
        if (pd.W == 1 && M <= 16) {
            const int kpad = dks::shared_path::fused_kpad(M);
            double* pm64; double* dv64;
            CUDA_TRY(ctx->plan_pool[M].alloc(&pm64, (size_t)kpad * pd.S_pad));
            CUDA_TRY(ctx->plan_pool[M].alloc(&dv64, (size_t)kpad));
            long long tot = (long long)kpad * pd.S_pad;
            dks::shared_path::plan_pmat64_kernel<<<cdiv(tot, 256), 256, 0, ctx->stream>>>(pd.z, pd.w, pd.ainv, pd.S, pd.S_pad, M,
                                                                                          kpad, pm64);
            dks::shared_path::plan_dvec64_kernel<<<kpad, 32, 0, ctx->stream>>>(pd.z, pm64, pd.S, M, kpad, dv64);
            ctx->launches += 2;
            CUDA_TRY(cudaGetLastError());
            pd.pmat64 = pm64; pd.dvec64 = dv64; pd.kpad = kpad;
            if (N <= dks::shared_path::MAXN) TRY(build_link_table(ctx, pd, M, pd.z));
        }
        break;
    case HEAD_SHARED_MIX_BINARY:
        // each member's tables from its own rows of the background (dks_fit split them per member)
        for (int k = 0; k < mh.K; ++k)
            TRY(build_dm_tables(ctx, pd, M, ctx->d_mixBW + (size_t)k * N * M * mh.Rm, ctx->d_mixsc + (size_t)k * N * mh.Rm,
                                -DKS_LOG2E, &ft.dm[k], &ft.dme[k]));
        TRY(build_pmat(ctx, pd, M));
        break;
    case HEAD_SHARED_CLASS_SUMS:
        TRY(build_class_tables(ctx, pd, M, ctx->d_BW, ctx->d_scores, ctx->C, h.scale, &ft.dm[0], &ft.lo[0]));
        break;
    case HEAD_SHARED_MIX_CLASS:
        for (int k = 0; k < mh.K; ++k)
            TRY(build_class_tables(ctx, pd, M, ctx->d_mixBW + (size_t)k * N * M * mh.Rm, ctx->d_mixsc + (size_t)k * N * mh.Rm,
                                   mh.Rm, DKS_LOG2E, &ft.dm[k], &ft.lo[k]));
        break;
    case HEAD_SHARED_TABLES:
        if (h.expo) {
            // exp head: l(s) = log2 sum_j w_j 2^(log2 e d(s, j)) (head_y, dks_shared.cuh)
            double* el;
            CUDA_TRY(ctx->plan_pool[M].alloc(&el, (size_t)pd.S_pad));
            auto kern = pd.W == 1 ? dks::shared_path::plan_exp_kernel<1> : dks::shared_path::plan_exp_kernel<2>;
            kern<<<cdiv(pd.S_pad, 128), 128, 0, ctx->stream>>>(pd.z, pd.S, pd.S_pad, ctx->d_BW, ctx->d_scores, ctx->d_wbg, N, M,
                                                              h.scale, el);
            ctx->launches += 1;
            CUDA_TRY(cudaGetLastError());
            ft.ell = el;
        }
        break;
    }
    ft.M = M;
    return DKS_OK;
}

int dks_set_shared_plan(dks_ctx* ctx, int M, int S, const uint64_t* zbits_host, const double* w_host) {
    BIND(ctx);
    REQUIRE(M >= 2 && M <= DKS_MAX_GROUPS, "dks_set_shared_plan: M=%d out of [2,%d]", M, DKS_MAX_GROUPS);
    REQUIRE(S >= 1 && zbits_host && w_host, "dks_set_shared_plan: bad arguments");
    if (!ctx->plan_pool[M].empty()) TRY(drop_plans(ctx, M));     // replacing the plan of this M (another nsamples)
    PlanDev pd;
    TRY(upload_plan(ctx, M, S, zbits_host, w_host, &pd));
    if (M == ctx->G && ctx->fitted && M <= ctx->head.shared_max_G) TRY(build_full_set_tables(ctx, pd, M));
    ctx->h_plans[M] = pd;
    ctx->epoch++;
    CUDA_TRY(cudaMemcpyAsync(ctx->d_plans, ctx->h_plans, sizeof(ctx->h_plans), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (S > ctx->max_plan_S) ctx->max_plan_S = S;
    return DKS_OK;
}

int dks_clear_plans(dks_ctx* ctx) {
    BIND(ctx);
    return drop_plans(ctx, -1);
}

int dks_has_shared_plan(dks_ctx* ctx, int M, int* present) {
    REQUIRE(ctx && present && M >= 0 && M <= DKS_MAX_GROUPS, "dks_has_shared_plan: bad arguments");
    const PlanDev& pd = ctx->h_plans[M];
    *present = (pd.z != nullptr && pd.S == dks_effective_S(M, ctx->nsamples_req) && (pd.W <= 2 || pd.ptw != nullptr)) ? 1 : 0;
    return DKS_OK;
}

int dks_set_plan_projection(dks_ctx* ctx, int M, const double* pt_host, const double* dvec_host) {
    BIND(ctx);
    REQUIRE(M > 128 && M <= DKS_MAX_GROUPS, "dks_set_plan_projection: for plans of 129..%d groups (got M=%d); narrower plans "
            "are factored on the device", DKS_MAX_GROUPS, M);
    REQUIRE(pt_host && dvec_host, "dks_set_plan_projection: NULL table");
    PlanDev& pd = ctx->h_plans[M];
    REQUIRE(pd.z != nullptr && pd.W > 2, "dks_set_plan_projection: set the shared plan of M=%d first", M);
    REQUIRE(pd.ptw == nullptr, "dks_set_plan_projection: the M=%d plan already has its projection (replace the plan first)", M);
    const int nA = M - 1, kp = dks::wide::kpad(M);
    double* pt; double* dv;
    CUDA_TRY(ctx->plan_pool[M].alloc(&pt, (size_t)pd.S_pad * kp));
    CUDA_TRY(ctx->plan_pool[M].alloc(&dv, (size_t)kp));
    CUDA_TRY(cudaMemsetAsync(pt, 0, sizeof(double) * (size_t)pd.S_pad * kp, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(dv, 0, sizeof(double) * kp, ctx->stream));
    // host [S][M-1] -> device [S_pad][kp] (zero padded rows and columns)
    CUDA_TRY(cudaMemcpy2DAsync(pt, sizeof(double) * kp, pt_host, sizeof(double) * nA, sizeof(double) * nA, (size_t)pd.S,
                               cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(dv, dvec_host, sizeof(double) * nA, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    pd.ptw = pt; pd.dvecw = dv; pd.kpw = kp;
    ctx->epoch++;
    CUDA_TRY(cudaMemcpy(ctx->d_plans, ctx->h_plans, sizeof(ctx->h_plans), cudaMemcpyHostToDevice));
    return DKS_OK;
}

int dks_set_l1(dks_ctx* ctx, int mode, int k, uint64_t sel_lo, uint64_t sel_hi) {
    REQUIRE(ctx && mode >= 0 && mode <= 3, "dks_set_l1: mode must be 0 (off), 1 (aic), 2 (bic) or 3 (num_features)");
    REQUIRE(mode != 3 || k >= 1, "dks_set_l1: num_features needs k >= 1");
    REQUIRE((sel_lo & 1ull) == 0, "dks_set_l1: M = 1 has nothing to select");
    if (mode != ctx->l1_mode || k != ctx->l1_k || sel_lo != ctx->l1_sel[0] || sel_hi != ctx->l1_sel[1]) ctx->epoch++;
    ctx->l1_mode = mode; ctx->l1_k = k; ctx->l1_sel[0] = sel_lo; ctx->l1_sel[1] = sel_hi;
    return DKS_OK;
}

int dks_set_l1_tables(dks_ctx* ctx, int M, const double* gram_raw, const double* gram_norm, const double* colsum,
                      const double* scale, const double* bz, const double* gram_w, const double* b_rows,
                      const double* sqab_rows, double sum_b, double sum_sqb, int n_aug) {
    BIND(ctx);
    REQUIRE(M >= 2 && M <= DKS_L1_MAX_GROUPS, "dks_set_l1_tables: M out of range (the selection covers at most %d groups)",
            DKS_L1_MAX_GROUPS);
    REQUIRE(gram_raw && gram_norm && colsum && scale && bz && gram_w && b_rows && sqab_rows, "dks_set_l1_tables: NULL table");
    const PlanDev& pd = ctx->h_plans[M];
    REQUIRE(pd.z != nullptr && n_aug == 2 * pd.S, "dks_set_l1_tables: set the shared plan of M=%d first (n_aug = 2 S)", M);
    const size_t mm = (size_t)M * M, S = (size_t)pd.S;
    const size_t total = 3 * mm + 3 * (size_t)M + 2 * S;
    double* base;
    CUDA_TRY(ctx->plan_pool[M].alloc(&base, total));
    dks::l1::Tables d;
    memset(&d, 0, sizeof(d));
    double* q = base;
    auto put = [&](const double* src, size_t cnt, const double** dst) -> cudaError_t {
        *dst = q;
        cudaError_t e = cudaMemcpyAsync(q, src, sizeof(double) * cnt, cudaMemcpyHostToDevice, ctx->stream);
        q += cnt;
        return e;
    };
    CUDA_TRY(put(gram_raw, mm, &d.gram_raw)); CUDA_TRY(put(gram_norm, mm, &d.gram_norm)); CUDA_TRY(put(gram_w, mm, &d.gram_w));
    CUDA_TRY(put(colsum, M, &d.colsum)); CUDA_TRY(put(scale, M, &d.scale)); CUDA_TRY(put(bz, M, &d.bz));
    CUDA_TRY(put(b_rows, S, &d.b)); CUDA_TRY(put(sqab_rows, S, &d.sqab));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    d.sum_b = sum_b; d.sum_sqb = sum_sqb; d.n_aug = n_aug; d.S = pd.S;
    ctx->h_l1[M] = d;
    ctx->epoch++;
    return sync_l1_tables(ctx);
}

int dks_set_plan_sampling(dks_ctx* ctx, int M, int nfixed, int n_full, int n_paired, int ncdf, const double* cdf_host,
                          double weight_left) {
    REQUIRE(ctx && M >= 2 && M <= DKS_MAX_GROUPS, "dks_set_plan_sampling: M out of range");
    REQUIRE(ncdf >= 0 && ncdf <= dks::sampler::MAX_SIZES && (ncdf == 0 || cdf_host),
            "dks_set_plan_sampling: at most 64 sampled subset sizes");
    if (M > 128) return fail(DKS_ERR_UNSUPPORTED, "dks_set_plan_sampling: per-instance plans cover at most 128 groups");
    REQUIRE(nfixed >= 0 && n_full >= 0 && n_paired >= 0, "dks_set_plan_sampling: bad arguments");
    DksSamplingInfo& inf = ctx->h_sinfo[M];
    memset(&inf, 0, sizeof(inf));
    inf.nfixed = nfixed; inf.n_full = n_full; inf.n_paired = n_paired; inf.ncdf = ncdf; inf.weight_left = weight_left;
    for (int k = 0; k < ncdf; ++k) inf.cdf[k] = cdf_host[k];
    // normal matrix of the enumerated prefix: the per-instance sampler adds the sampled rows' part to it
    const PlanDev& pd = ctx->h_plans[M];
    REQUIRE(pd.z != nullptr && nfixed <= pd.S, "dks_set_plan_sampling: set the shared plan of M=%d first", M);
    BIND(ctx);
    double* af;
    CUDA_TRY(ctx->plan_pool[M].alloc(&af, (size_t)(M - 1) * (M - 1)));
    if (M <= 64) dks::plan_prefix_normal_kernel<<<1, 256, sizeof(double) * (M - 1) * (M - 1), ctx->stream>>>(pd.z, pd.w, nfixed, M, af);
    else dks::plan_prefix_normal_wide_kernel<<<1, 1024, 0, ctx->stream>>>(pd.z, pd.w, nfixed, M, af);
    ctx->launches += 1;
    CUDA_TRY(cudaGetLastError());
    ctx->h_afix[M] = af;
    // device copies of the tables the sampler reads (kept current here, not per explain call)
    if (!ctx->d_sinfo) CUDA_TRY(ctx->d_sinfo.alloc(DKS_MAX_GROUPS + 1));
    if (!ctx->d_afix) CUDA_TRY(ctx->d_afix.alloc(DKS_MAX_GROUPS + 1));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_sinfo, ctx->h_sinfo, sizeof(ctx->h_sinfo), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_afix, ctx->h_afix, sizeof(ctx->h_afix), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    ctx->epoch++;
    return DKS_OK;
}

int dks_set_plan_mode(dks_ctx* ctx, int mode, uint64_t seed) {
    REQUIRE(ctx && (mode == 0 || mode == 1), "dks_set_plan_mode: mode must be 0 (shared per M) or 1 (per instance, device-drawn)");
    ctx->plan_mode = mode;
    ctx->sampler_seed = seed;
    return DKS_OK;
}

int dks_set_row_offset(dks_ctx* ctx, int64_t offset) {
    REQUIRE(ctx && offset >= 0, "dks_set_row_offset: bad arguments");
    ctx->row_offset = (long long)offset;
    return DKS_OK;
}

int dks_get_instance_plans(dks_ctx* ctx, uint64_t* zbits_host, double* w_host, int* n_out, int* stride_out) {
    BIND(ctx);
    REQUIRE(n_out && stride_out, "dks_get_instance_plans: bad arguments");
    *n_out = ctx->gen_n; *stride_out = ctx->gen_stride;
    REQUIRE(!(zbits_host && w_host && ctx->gen_n > 0 && ctx->gen_plan_words != 1),
            "dks_get_instance_plans: the last plans have two-word rows; use dks_get_instance_plans_w");
    if (zbits_host && w_host && ctx->gen_n > 0) {
        const size_t cnt = (size_t)ctx->gen_n * ctx->gen_stride;
        CUDA_TRY(cudaMemcpyAsync(zbits_host, ctx->d_genz, sizeof(uint64_t) * cnt, cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(cudaMemcpyAsync(w_host, ctx->d_genw, sizeof(double) * cnt, cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    }
    return DKS_OK;
}

int dks_get_instance_plans_w(dks_ctx* ctx, uint64_t* zbits_host, double* w_host, int* n_out, int* stride_out,
                             int* words_out) {
    BIND(ctx);
    REQUIRE(n_out && stride_out && words_out, "dks_get_instance_plans_w: bad arguments");
    *n_out = ctx->gen_n; *stride_out = ctx->gen_stride; *words_out = ctx->gen_plan_words;
    if (zbits_host && w_host && ctx->gen_n > 0) {
        const size_t cnt = (size_t)ctx->gen_n * ctx->gen_stride;
        CUDA_TRY(cudaMemcpyAsync(zbits_host, ctx->d_genz, sizeof(uint64_t) * cnt * ctx->gen_plan_words,
                                 cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(cudaMemcpyAsync(w_host, ctx->d_genw, sizeof(double) * cnt, cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    }
    return DKS_OK;
}

int dks_prepare_dev(dks_ctx* ctx, const double* X_dev, int n) {
    BIND(ctx);
    REQUIRE(ctx->fitted, "dks_prepare: call dks_fit first");
    REQUIRE(X_dev && n > 0, "dks_prepare: need X and n > 0");
    return launch_prepare(ctx, X_dev, n);
}

int dks_prepare_host(dks_ctx* ctx, const double* X_host, int n) {
    BIND(ctx);
    REQUIRE(ctx->fitted, "dks_prepare: call dks_fit first");
    REQUIRE(X_host && n > 0, "dks_prepare: need X and n > 0");
    size_t need = (size_t)n * ctx->D;
    if (need > ctx->d_X.size()) CUDA_TRY(ctx->d_X.alloc(need));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_X, X_host, sizeof(double) * need, cudaMemcpyHostToDevice, ctx->stream));
    return launch_prepare(ctx, ctx->d_X, n);
}

int dks_get_m_histogram(dks_ctx* ctx, int32_t* hist_host) {
    BIND(ctx);
    REQUIRE(ctx->prepared && hist_host, "dks_get_m_histogram: call dks_prepare_* first");
    CUDA_TRY(cudaMemcpyAsync(hist_host, ctx->d_hist, sizeof(int) * (ctx->G + 1), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return DKS_OK;
}

int dks_get_varying(dks_ctx* ctx, int32_t* M_host, uint64_t* mask_host) {
    BIND(ctx);
    REQUIRE(ctx->prepared, "dks_get_varying: call dks_prepare_* first");
    if (M_host) CUDA_TRY(cudaMemcpyAsync(M_host, ctx->d_M, sizeof(int) * ctx->cur_n, cudaMemcpyDeviceToHost, ctx->stream));
    if (mask_host)
        CUDA_TRY(cudaMemcpyAsync(mask_host, ctx->d_vmask, sizeof(uint64_t) * ctx->cur_n, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return DKS_OK;
}

int dks_get_link_fx(dks_ctx* ctx, double* out_host, int n) {
    BIND(ctx);
    REQUIRE(ctx->prepared && out_host, "dks_get_link_fx: call dks_prepare_* / dks_explain_* first");
    REQUIRE(n == ctx->cur_n, "dks_get_link_fx: the last stage 1 ran over %d rows, the caller expects %d", ctx->cur_n, n);
    const size_t cnt = (size_t)ctx->cur_n * ctx->C;
    CUDA_TRY(cudaMemcpyAsync(out_host, ctx->d_dlink, sizeof(double) * cnt, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < cnt; ++i) out_host[i] += ctx->h_linkfnull[i % ctx->C];   // stage 1 keeps link(f(x)) - link(fnull)
    return DKS_OK;
}

int dks_explain_dev(dks_ctx* ctx, double* phi_dev, const uint64_t* ext_zbits_dev, const double* ext_w_dev, int ext_stride) {
    BIND(ctx);
    REQUIRE(phi_dev, "dks_explain_dev: phi is NULL");
    TRY(launch_explain(ctx, phi_dev, ext_zbits_dev, ext_w_dev, ext_stride));
    return DKS_OK;
}

// after the solve: this rank's phi goes to every peer's gathered buffer (no-op without dks_set_peers)
static int launch_push(dks_ctx* ctx, const double* phi_dev) {
    if (ctx->peer_world <= 1) return DKS_OK;
    dks::PeerPush pp;
    pp.npeers = 0;
    for (int r = 0; r < ctx->peer_world; ++r) {
        double* slab = ctx->peer_base[r] + (long long)ctx->peer_rank * ctx->peer_slab;
        if (r == ctx->peer_rank && slab == phi_dev) continue;        // phi was written in place into the local slab
        pp.dst[pp.npeers++] = slab;
    }
    if (pp.npeers == 0) return DKS_OK;
    if (ctx->last_fused && ctx->push_in_kernel) {
        // the fused route's finish kernel stored its instances into the peers' buffers: only the general kernels' rows are left
        dks::push_rows_kernel<<<8, 256, 0, ctx->stream>>>(phi_dev, pp, ctx->d_idx_other, ctx->d_counts + 1, ctx->cur_n, ctx->G, ctx->C);
        ctx->launches += 1;
        CUDA_TRY(cudaGetLastError());
        return DKS_OK;
    }
    dim3 grid(8, pp.npeers);
    dks::push_phi_kernel<<<grid, 256, 0, ctx->stream>>>(phi_dev, pp, ctx->peer_slab);
    ctx->launches += 1;
    CUDA_TRY(cudaGetLastError());
    return DKS_OK;
}

// after the pushes: signal every peer and wait for theirs (no-op without dks_set_peer_flags)
static int launch_peer_sync(dks_ctx* ctx) {
    if (ctx->peer_world <= 1 || !ctx->peer_flags_set) return DKS_OK;
    dks::PeerFlags f;
    memset(&f, 0, sizeof(f));
    f.world = ctx->peer_world; f.rank = ctx->peer_rank; f.step = ctx->d_step;
    f.mine = ctx->peer_flags[ctx->peer_rank];
    for (int r = 0; r < ctx->peer_world; ++r) f.peer[r] = ctx->peer_flags[r];
    dks::peer_sync_kernel<<<1, 32, 0, ctx->stream>>>(f, ctx->d_status);
    ctx->launches += 1;
    CUDA_TRY(cudaGetLastError());
    return DKS_OK;
}

static void drop_graph(dks_ctx* ctx) {
    if (ctx->gexec) { cudaGraphExecDestroy(ctx->gexec); ctx->gexec = nullptr; }
}

int dks_run_dev(dks_ctx* ctx, const double* X_dev, int n, double* phi_dev) {
    BIND(ctx);
    REQUIRE(ctx->fitted, "dks_run_dev: call dks_fit first");
    REQUIRE(X_dev && phi_dev && n > 0, "dks_run_dev: bad arguments");
    dks_ctx::GraphKey key{X_dev, phi_dev, n, ctx->nsamples_req, ctx->kernel_choice, ctx->plan_mode, ctx->row_offset,
                          (unsigned long long)ctx->sampler_seed, ctx->epoch, ctx->stream};
    if (ctx->graph_enabled && ctx->gexec && key == ctx->graph_key && ctx->dbg_i < 0) {
        CUDA_TRY(cudaGraphLaunch(ctx->gexec, ctx->stream));
        ctx->graph_launches++;
        ctx->launches += ctx->graph_kernels;
        ctx->last_was_graph = true;
        return DKS_OK;                          // the status word stays on the device until dks_last_status asks for it
    }
    // the second identical call is captured (the first one sized every workspace, so nothing allocates during capture)
    // (the legacy default stream cannot be captured: callers that want graph replay pass their own stream)
    const bool capturable = ctx->stream != nullptr && ctx->stream != cudaStreamLegacy && ctx->stream != cudaStreamPerThread;
    bool capture = ctx->graph_enabled && capturable && ctx->have_last_key && key == ctx->last_key && ctx->dbg_i < 0;
    ctx->last_key = key; ctx->have_last_key = true;
    if (capture) {
        drop_graph(ctx);
        if (cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeRelaxed) != cudaSuccess) {
            cudaGetLastError();
            ctx->graph_enabled = false;          // this stream cannot be captured: plain launches from now on
            capture = false;
        } else {
            ctx->capturing = true;
        }
    }
    const int64_t launches_before = ctx->launches;
    int rc = launch_prepare(ctx, X_dev, n);
    if (rc == DKS_OK) rc = launch_explain(ctx, phi_dev, nullptr, nullptr, 0);
    if (rc == DKS_OK) rc = launch_push(ctx, phi_dev);
    if (rc == DKS_OK) rc = launch_peer_sync(ctx);
    ctx->last_was_graph = capture;          // the captured sequence runs as a graph launch below
    if (capture) {
        ctx->capturing = false;
        cudaGraph_t graph = nullptr;
        cudaError_t ce = cudaStreamEndCapture(ctx->stream, &graph);
        if (rc == DKS_OK && ce == cudaSuccess && graph) {
            ce = cudaGraphInstantiate(&ctx->gexec, graph, 0);
            if (ce == cudaSuccess) {
                ctx->graph_key = key;
                ctx->graph_kernels = ctx->launches - launches_before;
                ce = cudaGraphLaunch(ctx->gexec, ctx->stream);      // capturing did not execute anything
                ctx->graph_launches++;
            }
        }
        if (graph) cudaGraphDestroy(graph);
        if (rc != DKS_OK) return rc;
        if (ce != cudaSuccess) {
            drop_graph(ctx);
            cudaGetLastError();
            ctx->graph_enabled = false;                              // fall back to plain launches for good
            ctx->launches = launches_before;
            TRY(launch_prepare(ctx, X_dev, n));
            TRY(launch_explain(ctx, phi_dev, nullptr, nullptr, 0));
            TRY(launch_push(ctx, phi_dev));
            TRY(launch_peer_sync(ctx));
        }
    } else if (rc != DKS_OK) {
        return rc;
    }
    return DKS_OK;
}

int dks_set_peers(dks_ctx* ctx, int world, int rank, const uint64_t* gathered_ptrs_host, int64_t slab_doubles) {
    REQUIRE(ctx, "dks_set_peers: ctx is NULL");
    ctx->epoch++;
    if (world <= 1 || gathered_ptrs_host == nullptr) { ctx->peer_world = 0; ctx->peer_flags_set = false; return DKS_OK; }
    REQUIRE(world <= 16 && rank >= 0 && rank < world && slab_doubles > 0, "dks_set_peers: bad arguments (at most 16 ranks)");
    for (int r = 0; r < world; ++r) {
        REQUIRE(gathered_ptrs_host[r] != 0 && (gathered_ptrs_host[r] & 15) == 0, "dks_set_peers: peer buffers must be 16-byte aligned");
        ctx->peer_base[r] = reinterpret_cast<double*>(gathered_ptrs_host[r]);
    }
    REQUIRE((slab_doubles & 1) == 0, "dks_set_peers: slab size must be even (128-bit stores)");
    ctx->peer_world = world; ctx->peer_rank = rank; ctx->peer_slab = slab_doubles;
    return DKS_OK;
}

int dks_set_peer_flags(dks_ctx* ctx, const uint64_t* flag_ptrs_host) {
    BIND(ctx);
    ctx->epoch++;
    if (flag_ptrs_host == nullptr) { ctx->peer_flags_set = false; return DKS_OK; }
    REQUIRE(ctx->peer_world > 1, "dks_set_peer_flags: call dks_set_peers first");
    for (int r = 0; r < ctx->peer_world; ++r) {
        REQUIRE(flag_ptrs_host[r] != 0 && (flag_ptrs_host[r] & 7) == 0, "dks_set_peer_flags: flag arrays must be 8-byte aligned");
        ctx->peer_flags[r] = reinterpret_cast<unsigned long long*>(flag_ptrs_host[r]);
    }
    if (!ctx->d_step) {
        CUDA_TRY(ctx->d_step.alloc(1));
        CUDA_TRY(cudaMemset(ctx->d_step, 0, sizeof(unsigned long long)));
    }
    ctx->peer_flags_set = true;
    return DKS_OK;
}

int dks_graph_launches(dks_ctx* ctx, int64_t* count) {
    REQUIRE(ctx && count, "dks_graph_launches: bad arguments");
    *count = ctx->graph_launches;
    return DKS_OK;
}

// caller-supplied plans [n][ext_stride] from host memory into the context's buffers (*dz, *dw; NULL without plans)
static int stage_ext_plans(dks_ctx* ctx, int n, const uint64_t* ext_zbits_host, const double* ext_w_host, int ext_stride,
                           const uint64_t** dz, const double** dw) {
    *dz = nullptr; *dw = nullptr;
    if (!ext_zbits_host) return DKS_OK;
    REQUIRE(ext_w_host && ext_stride > 0, "dks_explain_host: ext_w / ext_stride missing");
    size_t need = (size_t)n * ext_stride;
    if (need > ctx->d_extw.size()) { CUDA_TRY(ctx->d_extz.alloc(need)); CUDA_TRY(ctx->d_extw.alloc(need)); }
    CUDA_TRY(cudaMemcpyAsync(ctx->d_extz, ext_zbits_host, sizeof(uint64_t) * need, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(ctx->d_extw, ext_w_host, sizeof(double) * need, cudaMemcpyHostToDevice, ctx->stream));
    *dz = ctx->d_extz; *dw = ctx->d_extw;
    return DKS_OK;
}

// d_phi [C][n][G] of the call just enqueued into phi_host and the status word back; synchronises
static int phi_to_host(dks_ctx* ctx, int n, double* phi_host) {
    const size_t need_phi = (size_t)ctx->C * n * ctx->G;
    ctx->phi_rows = n;                      // dks_summarise_host works off this buffer
    // results travel through a pinned staging buffer: one asynchronous DMA + one host memcpy instead of the driver's
    // chunked pageable path (the caller's array is ordinary NumPy memory)
    bool direct = false;                    // the caller's array is page-locked: one DMA straight into it
    {
        cudaPointerAttributes attr;
        if (cudaPointerGetAttributes(&attr, phi_host) == cudaSuccess) direct = attr.type == cudaMemoryTypeHost;
        else cudaGetLastError();
    }
    if (!direct && need_phi > ctx->h_phi_pin.size()) CUDA_TRY(ctx->h_phi_pin.alloc(need_phi));
    CUDA_TRY(cudaMemcpyAsync(direct ? phi_host : ctx->h_phi_pin, ctx->d_phi, sizeof(double) * need_phi, cudaMemcpyDeviceToHost,
                             ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(ctx->h_status, ctx->d_status, sizeof(int) * 2, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (!direct) memcpy(phi_host, ctx->h_phi_pin, sizeof(double) * need_phi);
    return check_status(ctx);
}

int dks_explain_host(dks_ctx* ctx, const double* X_host, int n, double* phi_host, const uint64_t* ext_zbits_host,
                     const double* ext_w_host, int ext_stride) {
    BIND(ctx);
    REQUIRE(ctx->fitted, "dks_explain_host: call dks_fit first");
    REQUIRE(X_host && phi_host && n > 0, "dks_explain_host: bad arguments");
    TRY(dks_prepare_host(ctx, X_host, n));
    size_t need_phi = (size_t)ctx->C * n * ctx->G;
    if (need_phi > ctx->d_phi.size()) CUDA_TRY(ctx->d_phi.alloc(need_phi));
    const uint64_t* dz; const double* dw;
    TRY(stage_ext_plans(ctx, n, ext_zbits_host, ext_w_host, ext_stride, &dz, &dw));
    TRY(launch_explain(ctx, ctx->d_phi, dz, dw, ext_stride));
    return phi_to_host(ctx, n, phi_host);
}

// ---- a model the caller evaluates (DKS_ACT_EXTERNAL, dks_external.cuh) -------------------------------------------------
static int external_dtype(int dtype, const char* what) {
    if (dtype != DKS_EXTERNAL_FLOAT32 && dtype != DKS_EXTERNAL_FLOAT64)
        return fail(DKS_ERR_UNSUPPORTED, "%s: dtype %d; DKS_EXTERNAL_FLOAT32 or DKS_EXTERNAL_FLOAT64 only", what, dtype);
    return DKS_OK;
}

int dks_set_external_model(dks_ctx* ctx, int C, int scalar_out, int dtype) {
    BIND(ctx);
    REQUIRE(ctx->D > 0, "dks_set_external_model: call dks_set_background first (D unknown)");
    if (C < 1 || C > DKS_ENS_MAX_OUT)
        return fail(DKS_ERR_UNSUPPORTED, "dks_set_external_model: C=%d outputs; 1..%d supported", C, DKS_ENS_MAX_OUT);
    REQUIRE(!scalar_out || C == 1, "dks_set_external_model: a scalar output is one output (C=%d)", C);
    TRY(external_dtype(dtype, "dks_set_external_model"));
    ctx->ext_in_f64 = dtype == DKS_EXTERNAL_FLOAT64;
    ctx->d_ext_bgy.reset();
    return set_own_model(ctx, DKS_ACT_EXTERNAL, C, scalar_out);
}

int dks_set_external_background(dks_ctx* ctx, const void* y_dev, int y_dtype) {
    BIND(ctx);
    REQUIRE(ctx->act == DKS_ACT_EXTERNAL, "dks_set_external_background: call dks_set_external_model first");
    REQUIRE(y_dev, "dks_set_external_background: y is NULL");
    TRY(external_dtype(y_dtype, "dks_set_external_background"));
    const int N = ctx->N, C = ctx->C;
    CUDA_TRY(ctx->d_ext_bgy.alloc((size_t)N * C));
    dks::ext::external_load_kernel<<<cdiv(N, 128), 128, 0, ctx->stream>>>(y_dev, y_dtype == DKS_EXTERNAL_FLOAT64, N, C,
                                                                         ctx->link, nullptr, ctx->d_ext_bgy, nullptr, nullptr);
    ctx->launches += 1;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));       // the caller may free y_dev once this returns
    ctx->fitted = false;
    return DKS_OK;
}

// what an external call's steps after dks_external_begin depend on: the rows, the phi buffer, the options that decide the
// route and plans, the epoch (fit, plans, l1 tables, buffers moved) and the stream
static dks_ctx::GraphKey external_key(const dks_ctx* ctx) {
    return {ctx->cur_X, ctx->d_phi.get(), ctx->cur_n, ctx->nsamples_req, ctx->kernel_choice, ctx->plan_mode,
            ctx->row_offset, (unsigned long long)ctx->sampler_seed, ctx->epoch, ctx->stream};
}

// the call dks_external_begin laid out is still the one the context would run
static int require_begun(dks_ctx* ctx, const char* what) {
    REQUIRE(ctx->ext_coalitions >= 0 && ctx->prepared, "%s: call dks_external_begin first", what);
    if (!(external_key(ctx) == ctx->ext_key)) {
        ctx->ext_coalitions = -1;
        return fail(DKS_ERR_INVALID, "%s: the rows, plans, options, stream or fit changed since dks_external_begin; "
                    "prepare and begin the call again", what);
    }
    return DKS_OK;
}

static int require_external(dks_ctx* ctx, const char* what) {
    REQUIRE(ctx->fitted && ctx->act == DKS_ACT_EXTERNAL, "%s: needs a fitted context with a module (dks_set_external_model, "
            "dks_fit)", what);
    return DKS_OK;
}

int dks_external_prepare(dks_ctx* ctx, const double* X_dev, int n, const void* fx_dev, int fx_dtype) {
    BIND(ctx);
    TRY(require_external(ctx, "dks_external_prepare"));
    REQUIRE(X_dev && fx_dev && n > 0, "dks_external_prepare: need X, the module's outputs on it and n > 0");
    TRY(external_dtype(fx_dtype, "dks_external_prepare"));
    ctx->ext_coalitions = -1;
    ctx->ext_y = fx_dev; ctx->ext_y_f64 = fx_dtype == DKS_EXTERNAL_FLOAT64;
    const int rc = launch_prepare(ctx, X_dev, n);
    ctx->ext_y = nullptr;                   // the caller's buffer: read by the launch just enqueued, not kept
    return rc;
}

int dks_external_begin(dks_ctx* ctx, const uint64_t* ext_zbits_host, const double* ext_w_host, int ext_stride,
                       int64_t* rows_total) {
    BIND(ctx);
    TRY(require_external(ctx, "dks_external_begin"));
    REQUIRE(ctx->prepared && rows_total, "dks_external_begin: call dks_external_prepare first");
    const int n = ctx->cur_n;
    ctx->ext_coalitions = -1;
    const size_t need_phi = (size_t)ctx->C * n * ctx->G;
    if (need_phi > ctx->d_phi.size()) CUDA_TRY(ctx->d_phi.alloc(need_phi));
    const uint64_t* dz; const double* dw;
    TRY(stage_ext_plans(ctx, n, ext_zbits_host, ext_w_host, ext_stride, &dz, &dw));
    Route rt;
    ExplainParams p;
    TRY(explain_setup(ctx, ctx->d_phi, dz, dw, ext_stride, &rt, &p));
    TRY(grow(ctx, ctx->d_ens_ey, (size_t)n * ctx->C * p.S_cap));
    TRY(grow(ctx, ctx->d_ext_soff, (size_t)n + 1));
    dks::ext::external_offsets_kernel<<<1, dks::ext::SCAN_THREADS, 0, ctx->stream>>>(p, ctx->d_ext_soff);
    ctx->launches += 1;
    CUDA_TRY(cudaGetLastError());
    long long total = 0;
    CUDA_TRY(cudaMemcpyAsync(&total, ctx->d_ext_soff.get() + n, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(ctx->h_status, ctx->d_status, sizeof(int) * 2, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    TRY(check_status(ctx));
    ctx->ext_p = p;
    ctx->ext_call_z = dz; ctx->ext_call_stride = ext_stride;
    ctx->ext_coalitions = total;
    ctx->ext_key = external_key(ctx);
    *rows_total = (int64_t)total * ctx->N;
    return DKS_OK;
}

// the coalitions [*q0, *q1) of rows row0 .. row0 + rows - 1 of the call dks_external_begin laid out
static int external_rows(dks_ctx* ctx, const char* what, int64_t row0, int64_t rows, const void* buf, long long* q0,
                         long long* q1) {
    BIND(ctx);
    TRY(require_external(ctx, what));
    TRY(require_begun(ctx, what));
    const int64_t N = ctx->N;
    REQUIRE(buf && rows > 0 && row0 >= 0 && row0 % N == 0 && rows % N == 0 && row0 + rows <= ctx->ext_coalitions * N,
            "%s: rows %lld .. %lld are not whole coalitions of N=%lld rows within the call's %lld rows", what,
            (long long)row0, (long long)(row0 + rows), (long long)N, (long long)(ctx->ext_coalitions * N));
    *q0 = row0 / N; *q1 = (row0 + rows) / N;
    return DKS_OK;
}

int dks_external_mask(dks_ctx* ctx, int64_t row0, int64_t rows, void* out_dev) {
    long long q0, q1;
    TRY(external_rows(ctx, "dks_external_mask", row0, rows, out_dev, &q0, &q1));
    const int grid = cdiv(q1 - q0, dks::ext::MASK_COALITIONS);
    const cudaStream_t st = ctx->stream;
    if (ctx->ext_in_f64)
        dks::ext::external_mask_kernel<double><<<grid, dks::ext::MASK_THREADS, 0, st>>>(
            ctx->ext_p, ctx->d_ext_soff, q0, q1, ctx->cur_X, ctx->d_bg, ctx->D, ctx->d_ext_colgrp, (double*)out_dev);
    else
        dks::ext::external_mask_kernel<float><<<grid, dks::ext::MASK_THREADS, 0, st>>>(
            ctx->ext_p, ctx->d_ext_soff, q0, q1, ctx->cur_X, ctx->d_bg, ctx->D, ctx->d_ext_colgrp, (float*)out_dev);
    ctx->launches += 1;
    CUDA_TRY(cudaGetLastError());
    return DKS_OK;
}

int dks_external_reduce(dks_ctx* ctx, int64_t row0, int64_t rows, const void* y_dev, int y_dtype) {
    long long q0, q1;
    TRY(external_rows(ctx, "dks_external_reduce", row0, rows, y_dev, &q0, &q1));
    TRY(external_dtype(y_dtype, "dks_external_reduce"));
    constexpr int wpc = dks::ext::REDUCE_THREADS / 32;
    const int grid = (int)std::min<long long>(cdiv(q1 - q0, wpc), (long long)ctx->sm_count * 16);
    const ExplainParams& p = ctx->ext_p;
    if (y_dtype == DKS_EXTERNAL_FLOAT64)
        dks::ext::external_reduce_kernel<double><<<grid, dks::ext::REDUCE_THREADS, 0, ctx->stream>>>(
            ctx->d_ext_soff, p.n, ctx->N, ctx->C, p.S_cap, q0, q1, (const double*)y_dev, ctx->d_wbg, ctx->d_ens_ey);
    else
        dks::ext::external_reduce_kernel<float><<<grid, dks::ext::REDUCE_THREADS, 0, ctx->stream>>>(
            ctx->d_ext_soff, p.n, ctx->N, ctx->C, p.S_cap, q0, q1, (const float*)y_dev, ctx->d_wbg, ctx->d_ens_ey);
    ctx->launches += 1;
    CUDA_TRY(cudaGetLastError());
    return DKS_OK;
}

int dks_external_finish(dks_ctx* ctx, double* phi_host) {
    BIND(ctx);
    TRY(require_external(ctx, "dks_external_finish"));
    REQUIRE(phi_host, "dks_external_finish: phi is NULL");
    TRY(require_begun(ctx, "dks_external_finish"));
    ctx->ext_coalitions = -1;
    Route rt;                               // the route begin chose (the same state decides it; nothing is launched)
    TRY(choose_route(ctx, ctx->ext_call_z, ctx->ext_call_stride, &rt));
    TRY(explain_launch(ctx, rt, ctx->ext_p));
    return phi_to_host(ctx, ctx->cur_n, phi_host);
}

int dks_summarise_host(dks_ctx* ctx, int n, const int32_t* seg_offsets_host, int Gp, double* phi_sum_host,
                       double* mean_abs_host, int32_t* order_host, int32_t* argmax_host) {
    BIND(ctx);
    REQUIRE(ctx->prepared && ctx->d_phi != nullptr && n == ctx->cur_n && n == ctx->phi_rows,
            "dks_summarise_host: the last dks_explain_host call covered %d rows, the caller expects %d", ctx->phi_rows, n);
    const int G = ctx->G, C = ctx->C;
    REQUIRE(Gp >= 1 && Gp <= G, "dks_summarise_host: Gp out of range");
    if (seg_offsets_host) {
        REQUIRE(seg_offsets_host[0] == 0 && seg_offsets_host[Gp] == G, "dks_summarise_host: segments must cover the %d groups", G);
        for (int g = 0; g < Gp; ++g) REQUIRE(seg_offsets_host[g + 1] > seg_offsets_host[g], "dks_summarise_host: empty segment");
    } else {
        REQUIRE(Gp == G, "dks_summarise_host: without segments Gp must equal the number of groups");
    }
    DevBuf<int> d_seg, d_ord, d_arg;
    DevBuf<double> d_sum, d_mean;
    DevBuf<unsigned long long> d_abs;
    const size_t cells = (size_t)C * Gp;
    CUDA_TRY(d_abs.alloc(cells)); CUDA_TRY(d_mean.alloc((size_t)(C + 1) * Gp)); CUDA_TRY(d_ord.alloc((size_t)(C + 1) * Gp));
    CUDA_TRY(d_arg.alloc((size_t)n));
    if (seg_offsets_host) {
        CUDA_TRY(d_seg.alloc((size_t)Gp + 1));
        CUDA_TRY(cudaMemcpyAsync(d_seg, seg_offsets_host, sizeof(int) * (Gp + 1), cudaMemcpyHostToDevice, ctx->stream));
    }
    if (phi_sum_host) CUDA_TRY(d_sum.alloc(cells * n));
    CUDA_TRY(cudaMemsetAsync(d_abs, 0, sizeof(unsigned long long) * cells, ctx->stream));
    const long long total = (long long)cells * n;
    int grid = cdiv(total, 256);
    if (grid > ctx->sm_count * 4) grid = ctx->sm_count * 4;
    dks::phi_summary_kernel<<<grid, 256, sizeof(unsigned long long) * cells, ctx->stream>>>(
        ctx->d_phi, C, n, G, d_seg, Gp, d_sum, d_abs, ctx->d_dlink, ctx->d_linkfnull, d_arg);
    dks::phi_rank_kernel<<<1, 128, 0, ctx->stream>>>(d_abs, C, n, Gp, d_mean, d_ord);
    ctx->launches += 2;
    CUDA_TRY(cudaGetLastError());
    if (phi_sum_host) CUDA_TRY(cudaMemcpyAsync(phi_sum_host, d_sum, sizeof(double) * cells * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (mean_abs_host) CUDA_TRY(cudaMemcpyAsync(mean_abs_host, d_mean, sizeof(double) * (C + 1) * Gp, cudaMemcpyDeviceToHost, ctx->stream));
    if (order_host) CUDA_TRY(cudaMemcpyAsync(order_host, d_ord, sizeof(int) * (C + 1) * Gp, cudaMemcpyDeviceToHost, ctx->stream));
    if (argmax_host) CUDA_TRY(cudaMemcpyAsync(argmax_host, d_arg, sizeof(int) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return DKS_OK;
}

int dks_host_alloc(void** out, uint64_t bytes) {
    if (!out || bytes == 0) return fail(DKS_ERR_INVALID, "dks_host_alloc: bad arguments");
    CUDA_TRY(cudaHostAlloc(out, (size_t)bytes, cudaHostAllocDefault));
    return DKS_OK;
}

int dks_host_free(void* p) {
    if (p) CUDA_TRY(cudaFreeHost(p));
    return DKS_OK;
}

int dks_last_status(dks_ctx* ctx, int* detail) {
    BIND(ctx);
    CUDA_TRY(cudaMemcpyAsync(ctx->h_status, ctx->d_status, sizeof(int) * 2, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (detail) *detail = ctx->h_status[1];
    return check_status(ctx);
}

int dks_set_option(dks_ctx* ctx, const char* name, int value) {
    REQUIRE(ctx && name, "dks_set_option: bad arguments");
    const std::string key(name);
    if (key == "fused") ctx->opt_fused = value;
    else if (key == "fused_warps") ctx->opt_fused_warps = value;
    else if (key == "fused_batch") ctx->opt_fused_B = value;
    else if (key == "fused_table") ctx->opt_fused_table = value != 0;
    else if (key == "push_in_kernel") ctx->push_in_kernel = value != 0;
    else if (key == "graph") ctx->graph_enabled = value != 0;
    else if (key == "graph_timing") ctx->opt_graph_timing = value != 0;
    else return fail(DKS_ERR_INVALID, "dks_set_option: unknown option '%s'", name);
    ctx->epoch++;                      // a captured graph holds the old launch sequence
    return DKS_OK;
}

int dks_set_kernel(dks_ctx* ctx, int kernel) {
    REQUIRE(ctx && kernel >= DKS_KERNEL_AUTO && kernel <= DKS_KERNEL_SHARED, "dks_set_kernel: unknown kernel %d", kernel);
    ctx->kernel_choice = kernel;
    return DKS_OK;
}

int dks_kernel_launches(dks_ctx* ctx, int64_t* count) {
    REQUIRE(ctx && count, "dks_kernel_launches: bad arguments");
    *count = ctx->launches;
    return DKS_OK;
}

int dks_live_allocations(int64_t* count) {
    REQUIRE(count, "dks_live_allocations: NULL");
    *count = dks::g_live_allocations.load();
    return DKS_OK;
}

int dks_last_timings(dks_ctx* ctx, float* ms3) {
    BIND(ctx);
    REQUIRE(ms3 && ctx->prepared, "dks_last_timings: nothing to report");
    REQUIRE(ctx->timing_valid && !(ctx->last_was_graph && !ctx->opt_graph_timing),
            "dks_last_timings: the last call was a graph replay without timing nodes (dks_set_option \"graph_timing\" 1, or \"graph\" 0)");
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    CUDA_TRY(cudaEventElapsedTime(&ms3[0], ctx->ev[0], ctx->ev[1]));
    CUDA_TRY(cudaEventElapsedTime(&ms3[1], ctx->ev[2], ctx->ev[3]));
    CUDA_TRY(cudaEventElapsedTime(&ms3[2], ctx->ev[0], ctx->ev[3]));
    return DKS_OK;
}

int dks_last_general_l1_timings(dks_ctx* ctx, float* ms2) {
    BIND(ctx);
    REQUIRE(ms2 && ctx->l1_timing_valid, "dks_last_general_l1_timings: the last explain ran no general-list l1 selection "
            "outside a graph capture");
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    CUDA_TRY(cudaEventElapsedTime(&ms2[0], ctx->ev_l1[0], ctx->ev_l1[1]));
    CUDA_TRY(cudaEventElapsedTime(&ms2[1], ctx->ev_l1[1], ctx->ev_l1[2]));
    return DKS_OK;
}

int dks_last_path(dks_ctx* ctx, int32_t* out, int n) {
    REQUIRE(ctx && out && n >= 0, "dks_last_path: bad arguments");
    for (int k = 0; k < n; ++k) out[k] = k < DKS_PATH_FIELDS ? ctx->last_path[k] : 0;
    return DKS_OK;
}

int dks_fused_table_info(dks_ctx* ctx, int M, int64_t* table_bytes, int64_t* fallback_passes) {
    BIND(ctx);
    REQUIRE(M >= 0 && M <= DKS_MAX_GROUPS && table_bytes && fallback_passes, "dks_fused_table_info: bad arguments");
    *table_bytes = ctx->h_plans[M].ltab != nullptr ? ctx->h_plans[M].ltab_bytes : 0;
    unsigned long long fb = 0;
    if (ctx->d_ltab_fb != nullptr) {
        CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        CUDA_TRY(cudaMemcpy(&fb, ctx->d_ltab_fb, sizeof(fb), cudaMemcpyDeviceToHost));
    }
    *fallback_passes = (int64_t)fb;
    return DKS_OK;
}

int dks_debug_score_dump(dks_ctx* ctx, int instance) {
    REQUIRE(ctx, "null ctx");
    ctx->dbg_i = instance;
    return DKS_OK;
}

int dks_debug_get_scores(dks_ctx* ctx, float* out_host, int max_floats, int* rows, int* cols) {
    BIND(ctx);
    REQUIRE(ctx->dbg_T && out_host && rows && cols, "dks_debug_get_scores: no dump available");
    *rows = ctx->dbg_rows; *cols = ctx->dbg_cols;
    REQUIRE((long long)ctx->dbg_rows * ctx->dbg_cols <= max_floats, "dks_debug_get_scores: buffer too small");
    CUDA_TRY(cudaMemcpyAsync(out_host, ctx->dbg_T, sizeof(float) * ctx->dbg_rows * ctx->dbg_cols, cudaMemcpyDeviceToHost,
                             ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return DKS_OK;
}

int dks_debug_get_timeline(dks_ctx* ctx, float* out_host /* [6][256] */) {
    BIND(ctx);
    REQUIRE(ctx->dbg_time && out_host, "dks_debug_get_timeline: no timeline available");
    CUDA_TRY(cudaMemcpyAsync(out_host, ctx->dbg_time, sizeof(float) * 6 * 256, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return DKS_OK;
}

}  // extern "C"
