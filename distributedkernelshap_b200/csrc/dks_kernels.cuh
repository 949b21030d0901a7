// Device code of the H100 KernelSHAP engine: fit kernels (K0), per-instance preparation, and the fused
// coalition kernel (mask/impute + predict + background reduction + link + constrained WLS).
//
// Algebra used throughout (DESIGN.md §3): the model head sees linear scores, so a masked row's score is
//     score(s, j) = base_j + sum_{k in varying} z_sk * (XW_i[k] - BW[j][k])
// with XW_i[k] = sum_{col in group k} x_i[col] W[col]  and  BW[j][k] likewise for background row j.  The
// masked batch (S*N x D, KernelExplainer.allocate/addsample) is therefore never materialised.
#pragma once

#include <cuda_pipeline.h>

#include "dks_common.cuh"
#include "dks_linkmath.cuh"

namespace dks {

// ------------------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---- cheap link arithmetic (per-row log around a 64-entry table): dks_linkmath.cuh

// fixed-point accumulation of E^T W y: v -> round(v * 2^40) as int64 (|v| = w |y| < 8e6 fits), integer adds are exact and
// order-independent (bit-reproducible whatever the reduction order); resolution 2^-40 ~ 9e-13 per row.  (64-bit integer
// adds run at ~30 lanes/clk/SM, half the DADD rate: used where order-independence matters, not for speed.)
#define DKS_FIX_SCALE 1099511627776.0          /* 2^40 */
#define DKS_FIX_INV 9.094947017729282379150390625e-13   /* 2^-40 */
__device__ __forceinline__ long long to_fix(double v) { return __double2ll_rn(v * DKS_FIX_SCALE); }
__device__ __forceinline__ double from_fix(long long t) { return (double)t * DKS_FIX_INV; }
__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// np.isclose(a, b, rtol=1e-5, atol=1e-8, equal_nan=True) as used by KernelExplainer.not_equal
__device__ __forceinline__ bool np_isclose(double a, double b) {
    if (a == b) return true;
    if (isnan(a) && isnan(b)) return true;
    if (!isfinite(a) || !isfinite(b)) return false;
    return fabs(a - b) <= 1e-8 + 1e-5 * fabs(b);
}

// link(p): shap.common.LogitLink.f / IdentityLink.f
__device__ __forceinline__ double link_f(double p, int link) {
    return link == DKS_LINK_LOGIT ? log(p / (1.0 - p)) : p;
}

// model head in float64 on R scores -> C outputs (C = 2 for the binary head, else R).
// RB: a compile-time bound on R.  The loops then unroll over RB with r < R guards, so that a caller's z and out arrays
// stay in registers; 0: the loops run to the run-time R.  The same operations in the same order either way.
template <int RB = 0>
__device__ inline void head_f64(const double* z, int R, int act, double kappa, double* out) {
    constexpr bool fixed = RB > 0;
    if (act == DKS_ACT_BINARY_LOGISTIC) {
        // softmax([-kz/2, kz/2]) evaluated the numerically stable way sklearn does
        double t = kappa * z[0];
        double e = exp(-fabs(t));
        double big = 1.0 / (1.0 + e), small = e / (1.0 + e);
        out[1] = t >= 0 ? big : small;
        out[0] = t >= 0 ? small : big;
    } else if (act == DKS_ACT_SOFTMAX) {
        double m = z[0];
#pragma unroll
        for (int r = 1; r < (fixed ? RB : R); ++r) if (!fixed || r < R) m = fmax(m, z[r]);
        double sum = 0;
#pragma unroll
        for (int r = 0; r < (fixed ? RB : R); ++r) if (!fixed || r < R) { out[r] = exp(z[r] - m); sum += out[r]; }
#pragma unroll
        for (int r = 0; r < (fixed ? RB : R); ++r) if (!fixed || r < R) out[r] /= sum;
    } else if (act == DKS_ACT_OVR) {
        // one-vs-rest: sigmoid(z_r) / sum_r' sigmoid(z_r'), formed from log sigmoid so that no class underflows to 0/0
        double m = -INFINITY;
#pragma unroll
        for (int r = 0; r < (fixed ? RB : R); ++r) {
            if (fixed && r >= R) continue;
            out[r] = fmin(z[r], 0.0) - log1p(exp(-fabs(z[r])));
            m = fmax(m, out[r]);
        }
        double sum = 0;
#pragma unroll
        for (int r = 0; r < (fixed ? RB : R); ++r) if (!fixed || r < R) { out[r] = exp(out[r] - m); sum += out[r]; }
#pragma unroll
        for (int r = 0; r < (fixed ? RB : R); ++r) if (!fixed || r < R) out[r] /= sum;
    } else if (act == DKS_ACT_EXP) {
        out[0] = exp(z[0]);          // log-link GLM: predict = exp(z)
    } else {
#pragma unroll
        for (int r = 0; r < (fixed ? RB : R); ++r) if (!fixed || r < R) out[r] = z[r];
    }
}

// mixture head in float64: sum_k pi_k h(z_k) over the members' score rows z[k R_m ..] (2 outputs for binary members, else R_m)
__device__ inline void mix_head_f64(const double* z, const MixHead& mh, double* out) {
    const int Co = mh.mact == DKS_ACT_BINARY_LOGISTIC ? 2 : mh.Rm;
    for (int c = 0; c < Co; ++c) out[c] = 0.0;
    for (int k = 0; k < mh.K; ++k) {
        double o[8];
        head_f64(z + (size_t)k * mh.Rm, mh.Rm, mh.mact, 1.0, o);
        for (int c = 0; c < Co; ++c) out[c] = fma(mh.pi[k], o[c], out[c]);
    }
}

// column maps: adds f_col(x), the R score contributions of one raw value, to acc.  A binary search over the column's
// breakpoints (numpy's searchsorted side='right': a value on a breakpoint takes the piece on its right) then R FMAs, or over
// its keys (exact match, else the unknown row) then R loads.  Returns false, adding nothing, where the map's policy is
// "error" (NaN, or a category unseen at fit time).  RB: a compile-time bound on R, as for head_f64.
template <int RB = 0>
__device__ __forceinline__ bool cm_add(const int* __restrict__ h, const double* __restrict__ keys,
                                       const double* __restrict__ vals, double x, int R, double* acc) {
    constexpr bool fixed = RB > 0;
    const int flags = h[0], m = h[1];
    const double* t = keys + h[2];
    const double* v = vals + h[3];
    const double* row;
    if (isnan(x)) {
        if (flags & DKS_CM_NAN_ERROR) return false;
        row = v + (size_t)((flags & DKS_CM_CATEGORICAL) ? m + 1 : 2 * m) * R;
    } else if (flags & DKS_CM_CATEGORICAL) {
        int lo = 0, hi = m;                       // first key >= x
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (t[mid] < x) lo = mid + 1; else hi = mid; }
        if (lo < m && t[lo] == x) row = v + (size_t)lo * R;
        else if (flags & DKS_CM_UNKNOWN_ERROR) return false;
        else row = v + (size_t)m * R;
    } else {
        int lo = 0, hi = m - 1;                   // piece = breakpoints <= x
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (t[mid] <= x) lo = mid + 1; else hi = mid; }
        const double* p = v + (size_t)2 * lo * R;
#pragma unroll
        for (int r = 0; r < (fixed ? RB : R); ++r) if (!fixed || r < R) acc[r] += fma(p[r], x, p[R + r]);
        return true;
    }
#pragma unroll
    for (int r = 0; r < (fixed ? RB : R); ++r) if (!fixed || r < R) acc[r] += row[r];
    return true;
}

// reports the first instance / background row whose raw value a column map refuses
__device__ __forceinline__ void cm_report(int* status, int row) {
    if (atomicCAS(&status[0], 0, DKS_ERR_DOMAIN) == 0) status[1] = row;
}

// ------------------------------------------------------------------------------------------------------
// K0: fit (DenseData + KernelExplainer.__init__)
// ------------------------------------------------------------------------------------------------------
// BW[j][g][r] = sum_{col in g} bg[j][col] * W[r][col]; MAPS: sum_{col in g} f_{r,col}(bg[j][col]) (column maps)
// WIDE: up to DKS_MIX_MAX_R score rows per column map (a pipeline ending in a mixture head); the other instantiation eight
template <bool MAPS, bool WIDE = false>
__global__ void fit_bw_kernel(const double* __restrict__ bg, const double* __restrict__ W,
                              const int32_t* __restrict__ goff, const int32_t* __restrict__ gcols, int N, int D,
                              int G, int R, double* __restrict__ BW, ColumnMapsDev cm, int* __restrict__ status) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * G * R) return;
    int r = idx % R, g = (idx / R) % G, j = idx / (R * G);
    if (MAPS) {
        double acc[WIDE ? DKS_MIX_MAX_R : 8];     // every score row of the column
        for (int q = 0; q < R; ++q) acc[q] = 0;
        for (int c = goff[g]; c < goff[g + 1]; ++c) {
            const int col = gcols[c];
            if (!cm_add(cm.hdr + 4 * col, cm.keys, cm.vals, bg[(size_t)j * D + col], R, acc)) cm_report(status, j);
        }
        BW[idx] = acc[r];
        return;
    }
    double acc = 0;
    for (int c = goff[g]; c < goff[g + 1]; ++c) {
        int col = gcols[c];
        acc += bg[(size_t)j * D + col] * W[(size_t)r * D + col];
    }
    BW[idx] = acc;
}

__global__ void fit_scores_kernel(const double* __restrict__ BW, const double* __restrict__ b, int N, int G, int R,
                                  double* __restrict__ scores) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * R) return;
    int r = idx % R, j = idx / R;
    double acc = b[r];
    for (int g = 0; g < G; ++g) acc += BW[((size_t)j * G + g) * R + r];
    scores[idx] = acc;
}

__global__ void fit_colstats_kernel(const double* __restrict__ bg, int N, int D, double* __restrict__ colmin,
                                    double* __restrict__ colmax, int* __restrict__ colnan) {
    int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= D) return;
    double mn = INFINITY, mx = -INFINITY;
    int nan = 0;
    for (int j = 0; j < N; ++j) {
        double v = bg[(size_t)j * D + col];
        if (isnan(v)) nan = 1;
        else { mn = fmin(mn, v); mx = fmax(mx, v); }
    }
    colmin[col] = mn; colmax[col] = mx; colnan[col] = nan;
}

// fnull[c] = sum_j w_j f(bg_j)[c]; linkfnull = link(fnull); Bbar[g][r] = sum_j w_j BW[j][g][r].  One block.
__global__ void fit_fnull_kernel(const double* __restrict__ scores, const double* __restrict__ BW,
                                 const double* __restrict__ wbg, int N, int G, int R, int C, int act, double kappa,
                                 int link, double* __restrict__ fnull, double* __restrict__ linkfnull,
                                 double* __restrict__ Bbar, const MixHead* __restrict__ mix) {
    int t = threadIdx.x;
    if (t < C) {
        double acc = 0;
        for (int j = 0; j < N; ++j) {
            double out[DKS_MAX_OUT];
            if (act == DKS_ACT_MIX) mix_head_f64(scores + (size_t)j * R, *mix, out);
            else head_f64(scores + (size_t)j * R, R, act, kappa, out);
            acc += out[t] * wbg[j];
        }
        fnull[t] = acc;
        linkfnull[t] = link_f(acc, link);
    }
    for (int idx = t; idx < G * R; idx += blockDim.x) {
        double acc = 0;
        for (int j = 0; j < N; ++j) acc += wbg[j] * BW[(size_t)j * G * R + idx];
        Bbar[idx] = acc;
    }
}

// fnull[c] = sum_j w_j pred[j][c] in row order and linkfnull = link(fnull), from the background's predictions of a model with
// its own kernel; one block
__global__ void fit_pred_fnull_kernel(const double* __restrict__ pred, const double* __restrict__ wbg, int N, int C, int link,
                                      double* __restrict__ fnull, double* __restrict__ linkfnull) {
    const int c = threadIdx.x;
    if (c >= C) return;
    double acc = 0;
    for (int j = 0; j < N; ++j) acc += pred[(size_t)j * C + c] * wbg[j];
    fnull[c] = acc;
    linkfnull[c] = link_f(acc, link);
}

// scaled float copies consumed by the fused kernel: BWs[r][g][j] = scale*BW[j][g][r], bases[r][j] = scale*score
// (fold_w, the exp head: bases[j] = scale*score + log2 w_j, so that 2^t carries the weight and a zero weight gives 2^-inf = 0)
__global__ void fit_scale_kernel(const double* __restrict__ BW, const double* __restrict__ scores,
                                 const double* __restrict__ wbg, int N, int G, int R, double scale,
                                 float* __restrict__ BWs, float* __restrict__ bases, float* __restrict__ wbf, int fold_w) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < N * G * R) {
        int j = idx % N, g = (idx / N) % G, r = idx / (N * G);
        BWs[idx] = (float)(scale * BW[((size_t)j * G + g) * R + r]);
    }
    if (idx < N * R) {
        int j = idx % N, r = idx / N;
        const double v = scale * scores[(size_t)j * R + r];
        bases[idx] = (float)(fold_w ? v + log2(wbg[j]) : v);
    }
    if (idx < N) wbf[idx] = (float)wbg[idx];
}

// f(X) for n rows, float64 (model check against the Python callable); MAPS: the scores through the column maps
template <bool MAPS>
__global__ void predict_kernel(const double* __restrict__ X, const double* __restrict__ W,
                               const double* __restrict__ b, int n, int D, int R, int C, int act, double kappa,
                               double* __restrict__ out, ColumnMapsDev cm, int* __restrict__ status,
                               const MixHead* __restrict__ mix) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double z[DKS_MAX_OUT], o[DKS_MAX_OUT];
    if (MAPS) {
        for (int r = 0; r < R; ++r) z[r] = b[r];
        for (int c = 0; c < D; ++c)
            if (!cm_add(cm.hdr + 4 * c, cm.keys, cm.vals, X[(size_t)i * D + c], R, z)) cm_report(status, i);
    } else {
        for (int r = 0; r < R; ++r) {
            double acc = b[r];
            for (int c = 0; c < D; ++c) acc += X[(size_t)i * D + c] * W[(size_t)r * D + c];
            z[r] = acc;
        }
    }
    if (act == DKS_ACT_MIX) mix_head_f64(z, *mix, o);
    else head_f64(z, R, act, kappa, o);
    for (int c = 0; c < C; ++c) out[(size_t)i * C + c] = o[c];
}

// Two fp32 lanes handled together.  Hopper has no packed fp32 instructions, so each lane is one scalar
// round-to-nearest op (explicit intrinsics: no contraction, the same rounding per lane as a packed op).
struct f32x2 { float lo, hi; };
__device__ __forceinline__ f32x2 f2_pack(float lo, float hi) { return f32x2{lo, hi}; }
__device__ __forceinline__ void f2_unpack(f32x2 v, float& lo, float& hi) { lo = v.lo; hi = v.hi; }
__device__ __forceinline__ f32x2 f2_mul(f32x2 a, f32x2 b) { return f32x2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f32x2 f2_add(f32x2 a, f32x2 b) { return f32x2{__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f32x2 f2_fma(f32x2 a, f32x2 b, f32x2 c) {
    return f32x2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)};
}


// ------------------------------------------------------------------------------------------------------
// Preparation: grouped instance contributions, varying_groups(), f(x), link deltas
// ------------------------------------------------------------------------------------------------------
// Fused preparation: a block handles `ipb` instances.  Phase 1, one thread per (instance, group): grouped
// contribution XW[i][g][r] and the "group varies" flag (KernelExplainer.varying_groups); phase 2, one thread per
// instance: varying bit-mask, M, histogram of M, f(x), link(f(x)) - link(fnull).
// The two instance lists and the histogram are counted per block in shared memory first: one global atomic per block and
// counter, and each instance takes the slot at its block's base plus its rank in the block.  The order of a list is
// therefore unspecified (it already was with one atomic per instance); every consumer works per instance.
// STAGE: the block first copies what phase 1 reads -- its instances' rows of X, W, the column statistics and the group
// tables -- into shared memory with coalesced loads, so the per-(instance, group) loop runs without dependent global loads.
// The host picks STAGE when the tables fit shared memory.  (Measured on the Adult shape, 2560 instances: 7.5 us per launch
// under torch.profiler on an H100 80GB HBM3 at 700 W, against 12.9 us with local-memory arrays, per-instance atomics and
// synchronous staging; DESIGN.md 5.0.)
// MAPS: the contributions come from the column maps `cm` instead of W -- per column a binary search and R FMAs or loads
// (cm_add); STAGE then stages the maps' tables where W would be.  A raw value a map refuses is reported as DKS_ERR_DOMAIN
// with the instance index and contributes nothing.
// MIX: the mixture head (up to DKS_MIX_MAX_R score rows; f(x) = sum_k pi_k h(z_k) from `mix`).  The other instantiations
// never read `mix`.
// RB: the compile-time bound on R (1 or 8; MIX: DKS_MIX_MAX_R).  The loops over score rows unroll over RB, so the per-thread
// contributions and scores live in registers rather than in a local-memory stack frame.
template <bool STAGE, bool MAPS, bool MIX = false, int RB = MIX ? DKS_MIX_MAX_R : 8>
__global__ void prep_kernel(const double* __restrict__ X, const double* __restrict__ W, const double* __restrict__ b,
                            const double* __restrict__ bg, const int32_t* __restrict__ goff,
                            const int32_t* __restrict__ gcols, const double* __restrict__ colmin,
                            const double* __restrict__ colmax, const int* __restrict__ colnan,
                            const double* __restrict__ linkfnull, int n, int N, int D, int G, int R, int C, int act,
                            double kappa, int link, int ipb, double* __restrict__ XW, uint64_t* __restrict__ vmask,
                            int* __restrict__ Mcnt, double* __restrict__ dlink, int* __restrict__ hist,
                            int* __restrict__ counts, int* __restrict__ idx_full, int* __restrict__ idx_other,
                            double* __restrict__ XT, double xt_scale, const double* __restrict__ xt_sub,
                            int* __restrict__ status, ColumnMapsDev cm, const MixHead* __restrict__ mix) {
    constexpr int CB = MIX ? 8 : (RB == 1 ? 2 : RB);    // outputs: C = 2 (binary head) or R; mixtures at most 8
    extern __shared__ __align__(16) unsigned char prep_smem[];
    double* sXW = reinterpret_cast<double*>(prep_smem);                        // [ipb][G][R]
    double* sX = sXW + (size_t)ipb * G * R;                                    // STAGE: [ipb][D]
    double* sW = sX + (STAGE ? (size_t)ipb * D : 0);                           //        [R][D] (MAPS: keys, values)
    double* sMin = sW + (STAGE ? (MAPS ? (size_t)cm.n_keys + cm.n_vals : (size_t)R * D) : 0);   //        [D]
    double* sMax = sMin + (STAGE ? D : 0);                                     //        [D]
    int* sNan = reinterpret_cast<int*>(sMax + (STAGE ? D : 0));                //        [D]
    int* sCols = sNan + (STAGE ? D : 0);                                       //        [D]
    int* sOff = sCols + (STAGE ? D : 0);                                       //        [G + 1]
    int* sHdr = sOff + (STAGE ? G + 1 : 0);                                    // MAPS:  [D][4]
    int* sCnt = sHdr + (STAGE && MAPS ? 4 * D : 0);     // the block's counts of the two lists, their bases, hist [G + 1]
    int* sHist = sCnt + 4;
    unsigned char* sflag = reinterpret_cast<unsigned char*>(sHist + G + 1);   // [ipb][G]
    for (int idx = threadIdx.x; idx < G + 5; idx += blockDim.x) sCnt[idx] = 0;
    if (threadIdx.x == 0) {      // what only the tail reads: into L2 now, so that its loads do not wait on DRAM there
        asm volatile("prefetch.global.L2 [%0];" ::"l"(b));
        asm volatile("prefetch.global.L2 [%0];" ::"l"(linkfnull));
    }
    const int i0 = blockIdx.x * ipb;
    if (STAGE) {
        // asynchronous copies (cp.async), all issued before any is waited on: the staging costs one DRAM round trip rather
        // than one per table
        auto cp8 = [](double* d, const double* s) { __pipeline_memcpy_async(d, s, sizeof(double)); };
        auto cp4 = [](int* d, const int* s) { __pipeline_memcpy_async(d, s, sizeof(int)); };
        const int rows = min(ipb, n - i0);
        const double* Xb = X + (size_t)i0 * D;
        for (int idx = threadIdx.x; idx < rows * D; idx += blockDim.x) cp8(sX + idx, Xb + idx);
        if (MAPS) {
            for (int idx = threadIdx.x; idx < cm.n_keys; idx += blockDim.x) cp8(sW + idx, cm.keys + idx);
            for (int idx = threadIdx.x; idx < cm.n_vals; idx += blockDim.x) cp8(sW + cm.n_keys + idx, cm.vals + idx);
            for (int idx = threadIdx.x; idx < 4 * D; idx += blockDim.x) cp4(sHdr + idx, cm.hdr + idx);
        } else {
            for (int idx = threadIdx.x; idx < R * D; idx += blockDim.x) cp8(sW + idx, W + idx);
        }
        for (int idx = threadIdx.x; idx < D; idx += blockDim.x) {
            cp8(sMin + idx, colmin + idx); cp8(sMax + idx, colmax + idx);
            cp4(sNan + idx, colnan + idx); cp4(sCols + idx, gcols + idx);
        }
        for (int idx = threadIdx.x; idx <= G; idx += blockDim.x) cp4(sOff + idx, goff + idx);
        __pipeline_commit();
        __pipeline_wait_prior(0);
        __syncthreads();
    }
    for (int idx = threadIdx.x; idx < ipb * G; idx += blockDim.x) {
        const int li = idx / G, g = idx - li * G, i = i0 + li;
        if (i >= n) continue;
        bool varies = false;
        double acc[RB];
#pragma unroll
        for (int r = 0; r < RB; ++r) acc[r] = 0;
        const int c0 = STAGE ? sOff[g] : goff[g], c1 = STAGE ? sOff[g + 1] : goff[g + 1];
        for (int c = c0; c < c1; ++c) {
            const int col = STAGE ? sCols[c] : gcols[c];
            const double xv = STAGE ? sX[(size_t)li * D + col] : X[(size_t)i * D + col];
            if (MAPS) {
                if (!cm_add<RB>(STAGE ? sHdr + 4 * col : cm.hdr + 4 * col, STAGE ? sW : cm.keys,
                                STAGE ? sW + cm.n_keys : cm.vals, xv, R, acc))
                    cm_report(status, i);
            } else {
#pragma unroll
                for (int r = 0; r < RB; ++r)
                    if (r < R) acc[r] += xv * (STAGE ? sW[(size_t)r * D + col] : W[(size_t)r * D + col]);
            }
            if ((STAGE ? sNan[col] : colnan[col]) || isnan(xv)) {
                if (!varies)
                    for (int j = 0; j < N && !varies; ++j) varies = !np_isclose(xv, bg[(size_t)j * D + col]);
            } else {
                // |x-b| - rtol|b| is decreasing for b <= x and increasing for b >= x: the extremes decide
                const double mn = STAGE ? sMin[col] : colmin[col], mx = STAGE ? sMax[col] : colmax[col];
                varies = varies || !np_isclose(xv, mn) || !np_isclose(xv, mx);
            }
        }
#pragma unroll
        for (int r = 0; r < RB; ++r) {
            if (r >= R) continue;
            sXW[(size_t)idx * R + r] = acc[r];
            XW[((size_t)i * G + g) * R + r] = acc[r];
        }
        sflag[idx] = varies ? 1 : 0;
    }
    __syncthreads();
    if (XT != nullptr) {
        // XT[i][r][t][x] = xt_scale * sum_{b<4} bit_b(x) (XW[i][4t+b][r] - xt_sub[4t+b][r]): the shared-plan kernels add
        // one table entry per nibble of a coalition row instead of one term per group (xt_sub: the identity head's Bbar)
        const int ntab = (G + 3) / 4;
        for (int idx = threadIdx.x; idx < ipb * R * ntab * 16; idx += blockDim.x) {
            const int li = idx / (R * ntab * 16), rem = idx - li * R * ntab * 16, r = rem / (ntab * 16);
            const int t = (rem >> 4) - r * ntab, x = rem & 15;
            const int i = i0 + li;
            if (i >= n) continue;
            double acc = 0.0;
#pragma unroll
            for (int b = 0; b < 4; ++b)
                if (((x >> b) & 1) && 4 * t + b < G) {
                    const int k = 4 * t + b;
                    acc += xt_sub != nullptr ? sXW[((size_t)li * G + k) * R + r] - xt_sub[(size_t)k * R + r]
                                             : sXW[((size_t)li * G + k) * R + r];
                }
            // MIX: member-major [K][n][R_m][ntab][16], so that a member's tables are the layout of the single-model head
            const size_t row = MIX ? ((size_t)(r / mix->Rm) * n + i) * mix->Rm + r % mix->Rm : (size_t)i * R + r;
            XT[(row * ntab + t) * 16 + x] = xt_scale * acc;
        }
    }
    // the per-instance tail, one thread per instance (ipb <= blockDim.x)
    const int li = threadIdx.x, i = i0 + li;
    const bool mine = li < ipb && i < n;
    int list = 0, rank = 0;
    if (mine) {
        uint64_t m = 0;                       // varying bit-mask (groups 0..63; wider problems only use the count)
        int M = 0;
        double z[RB], o[CB];
#pragma unroll
        for (int r = 0; r < RB; ++r) z[r] = r < R ? b[r] : 0.0;
        for (int g = 0; g < G; ++g) {
            if (sflag[li * G + g]) { if (g < 64) m |= (1ull << g); ++M; }
#pragma unroll
            for (int r = 0; r < RB; ++r) if (r < R) z[r] += sXW[((size_t)li * G + g) * R + r];
        }
        vmask[i] = m;
        Mcnt[i] = M;
        atomicAdd(&sHist[M], 1);
        // list: all groups vary (candidates for the shared-plan fast path) / everything else
        list = M == G && M >= 2 ? 0 : 1;
        rank = atomicAdd(&sCnt[list], 1);
        if constexpr (MIX) mix_head_f64(z, *mix, o);
        else head_f64<RB>(z, R, act, kappa, o);
#pragma unroll
        for (int c = 0; c < CB; ++c)
            if (c < C) dlink[(size_t)i * C + c] = link_f(o[c], link) - linkfnull[c];
        // exp head: f(x) = exp(z) overflows for z > 709.78; the explain kernels then never write this instance's phi
        if (act == DKS_ACT_EXP && !isfinite(o[0]) && atomicCAS(&status[0], 0, DKS_ERR_NUMERIC) == 0) status[1] = i;
    }
    __syncthreads();
    if (threadIdx.x < 2 && sCnt[threadIdx.x] > 0) sCnt[2 + threadIdx.x] = atomicAdd(&counts[threadIdx.x], sCnt[threadIdx.x]);
    for (int t = threadIdx.x; t <= G; t += blockDim.x)
        if (sHist[t] > 0) atomicAdd(&hist[t], sHist[t]);
    __syncthreads();
    if (mine) (list == 0 ? idx_full : idx_other)[sCnt[2 + list] + rank] = i;
}
// maps_doubles: the column maps' keys + values staged in place of W (0: the W path); their headers add 4 D ints.
// Every layout ends with the block's list counters and histogram (G + 5 ints) and the flags.
inline size_t prep_smem_bytes(bool stage, int ipb, int G, int R, int D, size_t maps_doubles = 0) {
    size_t b = sizeof(double) * (size_t)ipb * G * R + sizeof(int) * ((size_t)G + 5) + (size_t)ipb * G + 16;
    if (stage && maps_doubles)
        b += sizeof(double) * ((size_t)ipb * D + maps_doubles + 2 * (size_t)D) + sizeof(int) * (6 * (size_t)D + G + 1);
    else if (stage)
        b += sizeof(double) * ((size_t)ipb * D + (size_t)R * D + 2 * (size_t)D) + sizeof(int) * (2 * (size_t)D + G + 1);
    return b;
}

// ------------------------------------------------------------------------------------------------------
// Constrained WLS (KernelExplainer.solve without the l1 branch), float64, one CTA
// ------------------------------------------------------------------------------------------------------
// With L the last varying position and z' = (z_L ? ~z : z):  e_k e_l = z'_k & z'_l  and  e_k = (z_L ? -1 : 1) z'_k,
// where e_k = z_k - z_L is a column of upstream's `etmp`.

// A = E^T diag(w) E for k,l < M-1 (symmetric, row-major nA x nA), built warp-per-entry
__device__ inline void wls_build_normal(const uint64_t* __restrict__ zp, const double* __restrict__ wp, int S, int M,
                                        double* A, int warp, int nwarps) {
    const int nA = M - 1, L = M - 1;
    const int lane = threadIdx.x & 31;
    const int npairs = nA * (nA + 1) / 2;
    for (int pr = warp; pr < npairs; pr += nwarps) {
        int k = 0, rem = pr;
        while (rem > k) { rem -= (k + 1); ++k; }  // pr = k(k+1)/2 + l, l <= k
        int l = rem;
        double acc = 0;
        for (int s = lane; s < S; s += 32) {
            uint64_t z = zp[s];
            if ((z >> L) & 1ull) z = ~z;
            if (((z >> k) & (z >> l)) & 1ull) acc += wp[s];
        }
        acc = warp_sum(acc);
        if (lane == 0) { A[k * nA + l] = acc; A[l * nA + k] = acc; }
    }
}

// in-place lower Cholesky of the nA x nA matrix A (row-major) by warp 0; returns false if not positive definite
__device__ inline bool wls_cholesky_warp(double* A, int nA) {
    const int lane = threadIdx.x & 31;
    bool ok = true;
    for (int c = 0; c < nA; ++c) {
        double d = A[c * nA + c];
        if (!(d > 0.0)) ok = false;
        d = sqrt(d);
        __syncwarp();
        if (lane == 0) A[c * nA + c] = d;
        for (int r = c + 1 + lane; r < nA; r += 32) A[r * nA + c] /= d;
        __syncwarp();
        for (int r = c + 1 + lane; r < nA; r += 32) {
            double lrc = A[r * nA + c];
            for (int c2 = c + 1; c2 <= r; ++c2) A[r * nA + c2] -= lrc * A[c2 * nA + c];
        }
        __syncwarp();
    }
    return ok;
}

// rhs[k] = sum_s w_s e_sk (y_s - z_sL * delta), warp-per-k
__device__ inline void wls_build_rhs(const uint64_t* __restrict__ zp, const double* __restrict__ wp,
                                     const double* ys, int S, int M, double delta, double* rhs, int warp, int nwarps) {
    const int nA = M - 1, L = M - 1;
    const int lane = threadIdx.x & 31;
    for (int k = warp; k < nA; k += nwarps) {
        double acc = 0;
        for (int s = lane; s < S; s += 32) {
            uint64_t z = zp[s];
            int zl = (int)((z >> L) & 1ull), zk = (int)((z >> k) & 1ull);
            int e = zk - zl;
            if (e != 0) {
                double yy = ys[s] - (zl ? delta : 0.0);
                acc += wp[s] * (double)e * yy;
            }
        }
        acc = warp_sum(acc);
        if (lane == 0) rhs[k] = acc;
    }
}

// solve (L L^T) beta = rhs in place (thread 0), then write phi for output dim c of instance i
__device__ inline void wls_solve_write(const double* Lf, double* rhs, int M, double delta, const int* vi,
                                       double* __restrict__ phi_row, double sign) {
    const int nA = M - 1;
    for (int r = 0; r < nA; ++r) {
        double v = rhs[r];
        for (int c = 0; c < r; ++c) v -= Lf[r * nA + c] * rhs[c];
        rhs[r] = v / Lf[r * nA + r];
    }
    for (int r = nA - 1; r >= 0; --r) {
        double v = rhs[r];
        for (int c = r + 1; c < nA; ++c) v -= Lf[c * nA + r] * rhs[c];
        rhs[r] = v / Lf[r * nA + r];
    }
    double sum = 0;
    for (int k = 0; k < nA; ++k) {
        double v = rhs[k];
        sum += v;
        if (fabs(v) < 1e-10) v = 0;
        phi_row[vi[k]] = sign * v;
    }
    double last = delta - sum;
    if (fabs(last) < 1e-10) last = 0;
    phi_row[vi[nA]] = sign * last;
}

// ---- the edges of the per-instance CUDA-core kernels (one CTA per instance): plan lookup, the varying positions and the
// solve of the instance's outputs.  What the kernels compute between them is their own. ----
__device__ __forceinline__ void report_status(int* status, int code, int detail) {
    if (atomicCAS(&status[0], 0, code) == 0) status[1] = detail;
}

// the end of a family's predict kernel for row i with outputs o[C]: out [i][C] = o and dlink [i][C] = link(o) - linkfnull,
// each when not NULL.  A non-finite dlink is reported as DKS_ERR_NUMERIC with the instance unless the row was refused.
__device__ __forceinline__ void predict_epilogue(const double* o, int C, int i, int link, const double* __restrict__ linkfnull,
                                                 double* __restrict__ out, double* __restrict__ dlink, int* status,
                                                 bool refused) {
    bool bad = false;
    for (int c = 0; c < C; ++c) {
        if (out) out[(size_t)i * C + c] = o[c];
        if (dlink) {
            const double d = link_f(o[c], link) - linkfnull[c];
            dlink[(size_t)i * C + c] = d;
            bad |= !isfinite(d);
        }
    }
    if (bad && !refused) report_status(status, DKS_ERR_NUMERIC, i);
}

// instance i's phi rows of every output start at zero: only the varying groups are written
__device__ __forceinline__ void zero_phi_rows(const ExplainParams& p, int i) {
    const size_t slab = (size_t)p.n * p.G;
    for (int idx = threadIdx.x; idx < p.C * p.G; idx += blockDim.x)
        p.phi[(size_t)(idx / p.G) * slab + (size_t)i * p.G + idx % p.G] = 0.0;
}

// the coalition plan of instance i (M >= 2 varying groups)
struct InstPlan {
    const uint64_t* z;
    const double* w;
    const double* chol;   // its factored normal matrix, NULL if not factored
    int S;
};

// caller or sampler rows (ext_*), else the shared plan of M.  Returns false, the instance skipped, when the shared plan is
// missing (DKS_ERR_PLAN_MISSING, detail M) or S exceeds the kernel's staging (DKS_ERR_INVALID, detail i).
__device__ __forceinline__ bool inst_plan(const ExplainParams& p, int i, int M, InstPlan& pl) {
    pl.S = dks_effective_S(M, p.S_req);
    pl.chol = nullptr;
    if (p.ext_z != nullptr) {
        pl.z = p.ext_z + (size_t)i * p.ext_stride;
        pl.w = p.ext_w + (size_t)i * p.ext_stride;
        if (p.ext_chol != nullptr) pl.chol = p.ext_chol + (size_t)i * p.ext_fstride;   // factored with the plan
    } else {
        const PlanDev pd = p.plans[M];
        if (pd.z == nullptr || pd.S != pl.S) {
            if (threadIdx.x == 0) report_status(p.status, DKS_ERR_PLAN_MISSING, M);
            return false;
        }
        pl.z = pd.z; pl.w = pd.w; pl.chol = pd.chol;
    }
    if (pl.S > p.S_cap) {
        if (threadIdx.x == 0) report_status(p.status, DKS_ERR_INVALID, i);
        return false;
    }
    return true;
}

// vi[k] = group of varying position k (thread 0; the caller's barrier publishes it)
__device__ __forceinline__ void varying_positions(uint64_t vm, int G, int* vi) {
    if (threadIdx.x == 0) {
        int k = 0;
        for (int g = 0; g < G; ++g) if ((vm >> g) & 1ull) vi[k++] = g;
    }
}

// the plan's Cholesky factor into A: copied, or built and factored by warp 0 (not positive definite: DKS_ERR_NUMERIC,
// detail i).  No barrier after it: wls_build_rhs does not read A, and the solve follows a barrier.
__device__ __forceinline__ void block_normal(const InstPlan& pl, int M, double* A, int i, int* status) {
    const int tid = threadIdx.x;
    if (pl.chol != nullptr) {
        for (int idx = tid; idx < (M - 1) * (M - 1); idx += blockDim.x) A[idx] = pl.chol[idx];
    } else {
        wls_build_normal(pl.z, pl.w, pl.S, M, A, tid >> 5, blockDim.x >> 5);
        __syncthreads();
        if (tid < 32) {
            const bool ok = wls_cholesky_warp(A, M - 1);
            if (!ok && tid == 0) report_status(status, DKS_ERR_NUMERIC, i);
        }
    }
}

// two outputs: class 0 is the exact negation of class 1 (p0 = 1 - p1 row-wise); thread 0, after class 1's solve
__device__ __forceinline__ void write_class0_negation(double* phi0, const double* phi1, int M, const int* vi) {
    for (int k = 0; k < M; ++k) { const double v = phi1[vi[k]]; phi0[vi[k]] = (v == 0.0) ? 0.0 : -v; }
}

// one output: rhs from its y row, then thread 0 solves with the factor in A and writes phi_row
__device__ __forceinline__ void block_solve_one(const InstPlan& pl, int M, const double* ys, double delta, const double* A,
                                                double* rhs, const int* vi, double* phi_row) {
    wls_build_rhs(pl.z, pl.w, ys, pl.S, M, delta, rhs, threadIdx.x >> 5, blockDim.x >> 5);
    __syncthreads();
    if (threadIdx.x == 0) wls_solve_write(A, rhs, M, delta, vi, phi_row, 1.0);
}

// every solved output of instance i: output u's y row at ys + u * ystride, solved for class c = u, or (neg: two outputs,
// one solved) for class 1 with class 0 its negation.  A barrier before each output: the previous solve still reads rhs.
__device__ __forceinline__ void block_solve(const ExplainParams& p, int i, const InstPlan& pl, int M, const double* ys,
                                            size_t ystride, int nsolve, bool neg, const double* A, double* rhs,
                                            const int* vi) {
    const size_t slab = (size_t)p.n * p.G;
    for (int u = 0; u < nsolve; ++u) {
        const int c = neg ? 1 : u;
        __syncthreads();
        block_solve_one(pl, M, ys + (size_t)u * ystride, p.dlink[(size_t)i * p.C + c], A, rhs, vi,
                        p.phi + (size_t)c * slab + (size_t)i * p.G);
    }
    if (neg && threadIdx.x == 0) write_class0_negation(p.phi + (size_t)i * p.G, p.phi + slab + (size_t)i * p.G, M, vi);
}

// Block-level: Cholesky factor and inverse of the nA x nA matrix in A (shared memory, row-major; A must be followed by
// nA*nA doubles of scratch).  Needs blockDim.x >= max(32, nA).  Returns (in every thread) whether A was positive definite.
__device__ inline bool wls_factor_invert(double* A, int nA, double* __restrict__ chol, double* __restrict__ ainv) {
    __shared__ int s_ok;
    if (threadIdx.x == 0) s_ok = 1;
    __syncthreads();
    if (threadIdx.x < 32) {
        bool ok = wls_cholesky_warp(A, nA);
        if (!ok) s_ok = 0;
    }
    __syncthreads();
    if (chol != nullptr)
        for (int idx = threadIdx.x; idx < nA * nA; idx += blockDim.x) chol[idx] = A[idx];
    // inverse of E^T W E (what upstream's np.linalg.inv computes): column c of the inverse solves L L^T x = e_c
    if ((int)threadIdx.x < nA) {
        const int c = threadIdx.x;
        double* x = A + nA * nA + c * nA;   // scratch column in shared memory
        for (int r = 0; r < nA; ++r) {
            double v = (r == c) ? 1.0 : 0.0;
            for (int k = 0; k < r; ++k) v -= A[r * nA + k] * x[k];
            x[r] = v / A[r * nA + r];
        }
        for (int r = nA - 1; r >= 0; --r) {
            double v = x[r];
            for (int k = r + 1; k < nA; ++k) v -= A[k * nA + r] * x[k];
            x[r] = v / A[r * nA + r];
        }
        if (ainv != nullptr)
            for (int r = 0; r < nA; ++r) ainv[r * nA + c] = x[r];
    }
    __syncthreads();
    return s_ok != 0;
}

// factor the normal matrix of a shared plan once (dks_set_shared_plan): one CTA
__global__ void plan_factor_kernel(const uint64_t* __restrict__ z, const double* __restrict__ w, int S, int M,
                                   double* __restrict__ chol, double* __restrict__ ainv, int* __restrict__ status) {
    extern __shared__ double sm_d[];
    double* A = sm_d;
    const int nA = M - 1;
    wls_build_normal(z, w, S, M, A, threadIdx.x >> 5, blockDim.x >> 5);
    __syncthreads();
    const bool ok = wls_factor_invert(A, nA, chol, ainv);
    if (!ok && threadIdx.x == 0) { status[0] = DKS_ERR_NUMERIC; status[1] = M; }
}

// ---- plans of 65..128 groups (two words per row) -----------------------------------------------------------------
__device__ __forceinline__ bool zbit2(const uint64_t* __restrict__ row, int k) { return (row[k >> 6] >> (k & 63)) & 1ull; }

// E^T W E of the first S rows of a two-word plan, warp-per-entry (A in shared or global memory)
__device__ inline void wls_build_normal2(const uint64_t* __restrict__ z, const double* __restrict__ w, int S, int M, double* A) {
    const int nA = M - 1, L = M - 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int npairs = nA * (nA + 1) / 2;
    for (int pr = warp; pr < npairs; pr += nwarps) {
        int k = (int)((sqrtf(8.0f * (float)pr + 1.0f) - 1.0f) * 0.5f);
        while (k * (k + 1) / 2 > pr) --k;
        while ((k + 1) * (k + 2) / 2 <= pr) ++k;
        const int l = pr - k * (k + 1) / 2;
        double acc = 0;
        for (int s = lane; s < S; s += 32) {
            const uint64_t* row = z + (size_t)s * 2;
            const bool zl = zbit2(row, L);
            if ((zbit2(row, k) != zl) && (zbit2(row, l) != zl)) acc += w[s];
        }
        acc = warp_sum(acc);
        if (lane == 0) { A[k * nA + l] = acc; A[l * nA + k] = acc; }
    }
}

// Same factorisation for two-word plans: the matrix (up to 127 x 127) lives in shared memory, the columns of the inverse
// are solved in a global scratch buffer [nA][nA].
__global__ void plan_factor_wide_kernel(const uint64_t* __restrict__ z, const double* __restrict__ w, int S, int M,
                                        double* __restrict__ chol, double* __restrict__ ainv, double* __restrict__ scratch,
                                        int* __restrict__ status) {
    extern __shared__ double sm_d[];
    double* A = sm_d;
    const int nA = M - 1;
    wls_build_normal2(z, w, S, M, A);
    __syncthreads();
    __shared__ int s_ok;
    if (threadIdx.x == 0) s_ok = 1;
    __syncthreads();
    if (threadIdx.x < 32) { if (!wls_cholesky_warp(A, nA)) s_ok = 0; }
    __syncthreads();
    for (int idx = threadIdx.x; idx < nA * nA; idx += blockDim.x) chol[idx] = A[idx];
    for (int c = threadIdx.x; c < nA; c += blockDim.x) {
        double* x = scratch + (size_t)c * nA;
        for (int r = 0; r < nA; ++r) {
            double v = (r == c) ? 1.0 : 0.0;
            for (int k = 0; k < r; ++k) v -= A[r * nA + k] * x[k];
            x[r] = v / A[r * nA + r];
        }
        for (int r = nA - 1; r >= 0; --r) {
            double v = x[r];
            for (int k = r + 1; k < nA; ++k) v -= A[k * nA + r] * x[k];
            x[r] = v / A[r * nA + r];
        }
        for (int r = 0; r < nA; ++r) ainv[r * nA + c] = x[r];
    }
    if (threadIdx.x == 0 && !s_ok) { status[0] = DKS_ERR_NUMERIC; status[1] = M; }
}

// Push all-gather: every rank stores its block of phi into slab `rank` of each peer's gathered buffer through NVLink
// peer memory (128-bit stores; blockIdx.y = peer slot).  The caller follows up with a cross-GPU barrier.
struct PeerPush { double* dst[16]; int npeers; };
__global__ void push_phi_kernel(const double* __restrict__ src, PeerPush pp, long long n_doubles) {
    double* dst = pp.dst[blockIdx.y];
    const long long nvec = n_doubles >> 1;
    const double2* s2 = reinterpret_cast<const double2*>(src);
    double2* d2 = reinterpret_cast<double2*>(dst);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) d2[i] = s2[i];
    if ((n_doubles & 1) && blockIdx.x == 0 && threadIdx.x == 0) dst[n_doubles - 1] = src[n_doubles - 1];
}

// Same, for the rows of an instance list only (the fused route's finish kernel has already stored its instances into the
// peers' buffers; what the general kernels computed still has to travel).  phi is [C][n][G].
__global__ void push_rows_kernel(const double* __restrict__ src, PeerPush pp, const int* __restrict__ list,
                                 const int* __restrict__ count, int n, int G, int C) {
    const int cnt = *count;
    const long long per = (long long)C * G;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < cnt * per; idx += (long long)gridDim.x * blockDim.x) {
        const int q = (int)(idx / per), rem = (int)(idx - q * per), c = rem / G, g = rem - c * G;
        const size_t off = ((size_t)c * n + list[q]) * G + g;
        const double v = src[off];
        for (int r = 0; r < pp.npeers; ++r) pp.dst[r][off] = v;
    }
}

// ---- KernelShap.build_explanation post-processing off the resident phi (kernel_shap.py:36-109, :112-207, :952-956) ----------
// Segment sums over consecutive groups (sum_categories), |.| accumulated per (output, segment) in 2^-40 fixed point
// (shared-memory atomics per block, one global atomic per block and cell: order-independent), argmax of the raw prediction.
__global__ void phi_summary_kernel(const double* __restrict__ phi, int C, int n, int G, const int* __restrict__ seg, int Gp,
                                   double* __restrict__ phi_sum, unsigned long long* __restrict__ absacc,
                                   const double* __restrict__ dlink, const double* __restrict__ linkfnull,
                                   int* __restrict__ argmax) {
    extern __shared__ unsigned long long s_abs[];           // [C * Gp]
    for (int idx = threadIdx.x; idx < C * Gp; idx += blockDim.x) s_abs[idx] = 0ull;
    __syncthreads();
    const long long total = (long long)C * n * Gp;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int gp = (int)(idx % Gp);
        const long long ci = idx / Gp;
        const int i = (int)(ci % n), c = (int)(ci / n);
        const int g0 = seg ? seg[gp] : gp, g1 = seg ? seg[gp + 1] : gp + 1;
        double v = 0.0;
        for (int g = g0; g < g1; ++g) v += phi[((size_t)c * n + i) * G + g];
        if (phi_sum) phi_sum[idx] = v;
        atomicAdd(&s_abs[c * Gp + gp], (unsigned long long)to_fix(fabs(v)));
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < C * Gp; idx += blockDim.x)
        if (s_abs[idx]) atomicAdd(&absacc[idx], s_abs[idx]);
    if (argmax != nullptr) {
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
            int best = 0;
            double bv = dlink[(size_t)i * C] + linkfnull[0];
            for (int c = 1; c < C; ++c) {
                const double v = dlink[(size_t)i * C + c] + linkfnull[c];
                if (v > bv) { bv = v; best = c; }
            }
            argmax[i] = best;
        }
    }
}
// mean |phi| per output and aggregated over outputs ([C + 1][Gp]) and their descending order (ties: higher index first,
// what reversing a stable ascending argsort gives).  One block.
__global__ void phi_rank_kernel(const unsigned long long* __restrict__ absacc, int C, int n, int Gp, double* __restrict__ mean_abs,
                                int* __restrict__ order) {
    for (int idx = threadIdx.x; idx < (C + 1) * Gp; idx += blockDim.x) {
        const int r = idx / Gp, g = idx - r * Gp;
        double v = 0.0;
        if (r < C) v = from_fix((long long)absacc[r * Gp + g]) / (double)n;
        else for (int c = 0; c < C; ++c) v += from_fix((long long)absacc[c * Gp + g]) / (double)n;
        mean_abs[idx] = v;
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < (C + 1) * Gp; idx += blockDim.x) {
        const int r = idx / Gp, g = idx - r * Gp;
        const double v = mean_abs[idx];
        int rank = 0;
        for (int l = 0; l < Gp; ++l) {
            const double o = mean_abs[r * Gp + l];
            if (o > v || (o == v && l > g)) ++rank;
        }
        order[r * Gp + rank] = g;
    }
}

// Cross-GPU completion of the push all-gather without a library barrier: every rank keeps a flag word per peer in
// peer-mapped memory.  After the solve kernels (whose epilogues stored phi into the peers' buffers) one thread per peer
// publishes this rank's step count into the peer's flag array (system-scope release) and waits until the peer's count has
// reached the same step (acquire).  The step counter lives on the device, so a replayed CUDA graph keeps counting.
struct PeerFlags {
    unsigned long long* mine;            // [world] flags written by the peers
    unsigned long long* peer[16];        // peer[r]: rank r's flag array, mapped here
    unsigned long long* step;            // this rank's step counter (device memory)
    int world, rank;
};
__global__ void peer_sync_kernel(PeerFlags f, int* __restrict__ status) {
    __shared__ unsigned long long s_step;
    if (threadIdx.x == 0) { s_step = *f.step + 1ull; *f.step = s_step; }
    __syncthreads();
    const int t = threadIdx.x;
    if (t >= f.world || t == f.rank) return;
    const unsigned long long e = s_step;
    __threadfence_system();              // everything this GPU stored before (previous kernels included) is ordered first
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(f.peer[t] + f.rank), "l"(e) : "memory");
    unsigned long long seen = 0ull;
    for (long long spins = 0; spins < (1ll << 31); ++spins) {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(f.mine + t) : "memory");
        if (seen >= e) return;
    }
    if (atomicCAS(&status[0], 0, DKS_ERR_CUDA) == 0) status[1] = -78;     // a peer never arrived
}

// an instance list that must be empty (shapes no kernel covers): report instead of computing
__global__ void flag_unsupported_kernel(const int* __restrict__ count, int detail, int* __restrict__ status) {
    if (*count > 0 && atomicCAS(&status[0], 0, DKS_ERR_UNSUPPORTED) == 0) status[1] = detail;
}

// normal matrix of the first `rows` rows of a plan (its enumerated prefix), unfactored: the per-instance sampler adds
// the sampled rows' part to it
__global__ void plan_prefix_normal_kernel(const uint64_t* __restrict__ z, const double* __restrict__ w, int rows, int M,
                                          double* __restrict__ afix) {
    extern __shared__ double sm_d[];
    const int nA = M - 1;
    wls_build_normal(z, w, rows, M, sm_d, threadIdx.x >> 5, blockDim.x >> 5);
    __syncthreads();
    for (int idx = threadIdx.x; idx < nA * nA; idx += blockDim.x) afix[idx] = sm_d[idx];
}
// the same for two-word plans, written straight to global memory (a 127 x 127 float64 matrix is 126 KB)
__global__ void plan_prefix_normal_wide_kernel(const uint64_t* __restrict__ z, const double* __restrict__ w, int rows, int M,
                                               double* __restrict__ afix) {
    wls_build_normal2(z, w, rows, M, afix);
}

// ------------------------------------------------------------------------------------------------------
// Fused coalition kernel, CUDA-core (SIMT) version.  One CTA per instance (grid-stride), one thread per
// coalition row.  Handles the binary-logistic and identity heads; any plan source.
// ------------------------------------------------------------------------------------------------------
struct SimtSmem {
    double* ys;     // [S_cap] link(ey) - link(fnull) per coalition
    double* A;      // [63*63] normal matrix / its Cholesky factor
    double* rhs;    // [64]
    double* xw;     // [64] scaled grouped contributions of the instance (varying positions)
    int* vi;        // [64] varying position -> group index
    float* Bs;      // [M][N] scaled grouped background contributions of the varying groups, then bases[N], wb[N]
};

__device__ inline SimtSmem simt_carve(unsigned char* base, int S_cap, int R, int ny) {
    SimtSmem s;
    s.ys = reinterpret_cast<double*>(base);
    s.A = s.ys + (size_t)S_cap * ny;
    s.rhs = s.A + 63 * 63;
    s.xw = s.rhs + 64;
    s.vi = reinterpret_cast<int*>(s.xw + 64 * (size_t)R);
    s.Bs = reinterpret_cast<float*>(s.vi + 64);
    return s;
}

// ny = number of y buffers (1, or C for the softmax head), R = score rows staged per instance
__host__ __device__ inline size_t simt_smem_bytes(int S_cap, int N, int Mmax, int R = 1, int ny = 1) {
    return sizeof(double) * ((size_t)S_cap * ny + 63 * 63 + 64 + 64 * (size_t)R) + sizeof(int) * 64 +
           sizeof(float) * ((size_t)Mmax * N * R + (size_t)N * R + (size_t)N);
}

namespace l1 {   // dks_l1.cuh
constexpr int MOM_THREADS = 256;
template <int W, bool SCALED>
__device__ void block_moments(const double* ys, int S, int M, const uint64_t* __restrict__ z, const double* __restrict__ w,
                              const double* __restrict__ b, const double* __restrict__ sqab, double* mom,
                              long long (*part)[32], double (*bound)[2]);
}

// l1 feature selection on this kernel (instantiation L1): for the instances of its list it stores the moment vectors of y
// of every output instead of solving the WLS, and l1_lars_kernel selects and solves from them
struct SimtL1 {
    const l1::Tables* tabs;  // [DKS_L1_MAX_GROUPS + 1] tables of the shared plan of each M
    double* mom;             // [n][outputs][2G + 4]
};

// instead of the solve: the moments of y of nsolve outputs (output u's y row at ys + u * ystride) into moment rows
// row0 + u (instance i's outputs are rows i * outputs ...).  The reduction scratch lives where the solve keeps its
// normal matrix, A.
template <bool SCALED>
__device__ __forceinline__ void block_moments_all(const SimtL1& q, int G, const InstPlan& pl, int M, const double* ys,
                                                  size_t ystride, int nsolve, size_t row0, double* A) {
    const l1::Tables& t = q.tabs[M];
    const size_t mstride = 2 * (size_t)G + 4;
    for (int u = 0; u < nsolve; ++u)
        l1::block_moments<1, SCALED>(ys + (size_t)u * ystride, pl.S, M, pl.z, pl.w, t.b, t.sqab, q.mom + (row0 + u) * mstride,
                                     reinterpret_cast<long long (*)[32]>(A),
                                     reinterpret_cast<double (*)[2]>(A + l1::MOM_THREADS));
}

// moment rows row0 .. row0 + nsolve - 1 of an instance that is not solved: NaN at entry 2M, which l1_lars_kernel skips
__device__ __forceinline__ void moments_skip(const SimtL1& q, int G, int M, int nsolve, size_t row0) {
    if ((int)threadIdx.x < nsolve) q.mom[(row0 + threadIdx.x) * (2 * (size_t)G + 4) + 2 * M] = NAN;
}

// a member of a soft-voting ensemble (instantiation ACC of the family explain kernels, DESIGN.md §5.0.17): in place of the
// link and the solve, the member's background means of every output, times pi_k, are written (first member) or added to
// the ensemble's workspace ey [n][C][S_cap]; explain_ensemble_tail_kernel solves from it
struct EnsAcc {
    double* ey;              // NULL: not a member
    double pi;
    int first;
};

// instance i's sums acc [C][S_cap] of S coalitions into ey; each thread handles the coalitions s = tid (mod blockDim.x)
__device__ __forceinline__ void ens_accumulate(const EnsAcc& e, const ExplainParams& p, int i, int S, const double* acc) {
    double* ey = e.ey + (size_t)i * p.C * p.S_cap;
    for (int s = threadIdx.x; s < S; s += blockDim.x)
        for (int c = 0; c < p.C; ++c) {
            const size_t at = (size_t)c * p.S_cap + s;
            const double v = e.pi * acc[at];
            ey[at] = e.first ? v : ey[at] + v;
        }
}

// exp head: ey(s) of one coalition row in float64, for the rows outside the fp32 range rule (DKS_EXP_T_LO / _HI):
// exp(a + m + ln sum_j w_j e^(d_j - m)) with a = sum_{k in s} XW_i[k], d_j = score_j - sum_{k in s} BW[j][k] and m the
// running maximum of d_j (one pass, the sum rescaled when m grows), zero-weight rows skipped.  Row bit k (k < M) is
// varying position k, group vi[k] (vi NULL: group k); z1 holds bits 64..127.
__device__ inline double exp_row_f64(const ExplainParams& p, const ExpBackground& eb, int i, uint64_t z0, uint64_t z1, int M,
                                     const int* vi) {
    const int G = p.G;
    double a = 0.0;
    for (int k = 0; k < M; ++k)
        if (((k < 64 ? z0 : z1) >> (k & 63)) & 1ull) a += p.XW[(size_t)i * G + (vi ? vi[k] : k)];
    double m = -INFINITY, e = 0.0;
    for (int j = 0; j < p.N; ++j) {
        const double wj = p.wbg[j];
        if (!(wj > 0.0)) continue;
        double c = 0.0;
        for (int k = 0; k < M; ++k)
            if (((k < 64 ? z0 : z1) >> (k & 63)) & 1ull) c += eb.BW[(size_t)j * G + (vi ? vi[k] : k)];
        const double d = eb.scores[j] - c;
        if (d > m) { e = e * exp(m - d) + wj; m = d; }
        else e += wj * exp(d - m);
    }
    return exp(a + m + log(e));
}

// exp head: ey(s) from the fp32 sum of 2^t'_j (t'_j = log2 e d(s, j) + log2 w_j: bases carry log2 w_j) and its largest
// exponent thi, times 2^a with a = log2 e sum_{k in s} XW_i[k] in float64.  Inside the range rule no term overflows and a
// term that flushes to zero is below 2^-26 of the sum; other rows, and products that overflow, take exp_row_f64.
__device__ __forceinline__ double exp_row_ey(const ExplainParams& p, const ExpBackground& eb, int i, double a, float sum,
                                             float thi, uint64_t z0, uint64_t z1, int M, const int* vi) {
    if (thi >= DKS_EXP_T_LO && thi <= DKS_EXP_T_HI) {
        const double ey = exp2(a) * (double)sum;
        if (isfinite(ey)) return ey;
    }
    return exp_row_f64(p, eb, i, z0, z1, M, vi);
}

// EXP: the instantiation of the exp head, which compiles its branch only (the other heads' instantiations are unchanged)
template <bool L1, bool EXP = false>
__global__ void __launch_bounds__(256) explain_simt_kernel(ExplainParams p, SimtL1 q, ExpBackground eb) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const bool ovr = p.act == DKS_ACT_OVR;
    const bool softmax = p.act == DKS_ACT_SOFTMAX || ovr;     // C score rows and C y buffers
    SimtSmem sm = simt_carve(smem_raw, p.S_cap, softmax ? p.R : 1, softmax ? p.C : 1);
    const int tid = threadIdx.x;
    const int N = p.N, G = p.G, C = p.C;
    const size_t slab = (size_t)p.n * G;

    const int ninst = dks_inst_count(p);
    for (int qi = blockIdx.x; qi < ninst; qi += gridDim.x) {
        const int i = dks_inst_at(p, qi);
        const int M = p.Mcnt[i];
        const uint64_t vm = p.vmask[i];
        __syncthreads();  // previous instance done with shared memory
        zero_phi_rows(p, i);
        if (M == 0) continue;
        if (M == 1) {
            // (exp head: a non-finite f(x) was reported by prep_kernel and is not written)
            if (tid < C && (!EXP || isfinite(p.dlink[(size_t)i * C + tid]))) {
                int g = __ffsll((long long)vm) - 1;
                p.phi[(size_t)tid * slab + (size_t)i * G + g] = p.dlink[(size_t)i * C + tid];
            }
            continue;
        }
        InstPlan pl;
        if (!inst_plan(p, i, M, pl)) continue;
        const int S = pl.S;
        const uint64_t* zp = pl.z;
        varying_positions(vm, G, sm.vi);
        __syncthreads();

        float* Bs = sm.Bs;
        float* bases = Bs + (size_t)M * N;
        float* wb = bases + N;

        if constexpr (EXP) {
            // ---- exp head (DESIGN.md §5.0.8): ey(s) = 2^a(s) sum_j 2^t'_j, the instance part a(s) factored out in float64,
            // the background part t'_j = bases_j - sum_k z_sk BWs[k][j] summed in fp32; scale = log2(e) ----
            for (int idx = tid; idx < M * N; idx += blockDim.x) {
                int k = idx / N, j = idx - k * N;
                Bs[idx] = p.BWs[(size_t)sm.vi[k] * N + j];
            }
            for (int j = tid; j < N; j += blockDim.x) bases[j] = p.bases[j];
            if (tid < M) sm.xw[tid] = p.scale * p.XW[(size_t)i * G + sm.vi[tid]];
            __syncthreads();
            const double fn = p.fnull[0], delta = p.dlink[i];
            int bad = !isfinite(delta);
            for (int s = tid; s < S; s += blockDim.x) {
                const uint64_t z = zp[s];
                double a = 0;
                for (int k = 0; k < M; ++k) if ((z >> k) & 1ull) a += sm.xw[k];
                float sum = 0.f, thi = -INFINITY;
                for (int j = 0; j < N; ++j) {
                    float c = 0.f;
                    for (int k = 0; k < M; ++k) if ((z >> k) & 1ull) c += Bs[k * N + j];
                    const float t = bases[j] - c;
                    thi = fmaxf(thi, t);
                    sum += ex2_approx(t);
                }
                const double y = exp_row_ey(p, eb, i, a, sum, thi, z, 0ull, M, sm.vi) - fn;
                bad |= !isfinite(y);
                sm.ys[s] = y;
            }
            if (__syncthreads_or(bad)) {
                // a non-finite ey (or f(x)) is reported, never solved: nothing of this instance reaches phi or the moments
                if (tid == 0) report_status(p.status, DKS_ERR_NUMERIC, i);
                if constexpr (L1) moments_skip(q, G, M, 1, i);
                continue;
            }
            if constexpr (L1) {
                block_moments_all<true>(q, G, pl, M, sm.ys, 0, 1, i, sm.A);
                continue;
            }
            block_normal(pl, M, sm.A, i, p.status);
            block_solve_one(pl, M, sm.ys, delta, sm.A, sm.rhs, sm.vi, p.phi + (size_t)i * G);
        } else if (p.act == DKS_ACT_BINARY_LOGISTIC) {
            // stage this instance's varying columns of the background table
            for (int idx = tid; idx < M * N; idx += blockDim.x) {
                int k = idx / N, j = idx - k * N;
                Bs[idx] = p.BWs[(size_t)sm.vi[k] * N + j];
            }
            for (int j = tid; j < N; j += blockDim.x) { bases[j] = p.bases[j]; wb[j] = p.wbf[j]; }
            if (tid < M) sm.xw[tid] = p.scale * p.XW[(size_t)i * G + sm.vi[tid]];
            __syncthreads();

            const double lf1 = p.linkfnull[1], f1 = p.fnull[1];
            for (int s = tid; s < S; s += blockDim.x) {
                const uint64_t z = zp[s];
                double a = 0;
                for (int k = 0; k < M; ++k) if ((z >> k) & 1ull) a += sm.xw[k];
                const float af = (float)a;
                float acc1 = 0.f, acc0 = 0.f;
                for (int j = 0; j < N; ++j) {
                    float c = 0.f;
                    for (int k = 0; k < M; ++k) if ((z >> k) & 1ull) c += Bs[k * N + j];
                    float t = (bases[j] - c) + af;     // = -kappa*log2(e) * masked score
                    t = fminf(fmaxf(t, -120.f), 120.f);
                    float u = ex2_approx(t);           // exp(-kappa*score)
                    float r = rcp_approx(1.f + u);     // p1 = sigmoid(kappa*score)
                    acc1 = fmaf(wb[j], r, acc1);
                    acc0 = fmaf(wb[j], u * r, acc0);   // p0 = 1 - p1, accumulated without cancellation
                }
                double y;
                if (p.link == DKS_LINK_LOGIT) y = log((double)acc1 / (double)acc0) - lf1;
                else y = (double)acc1 - f1;
                sm.ys[s] = y;
            }
            __syncthreads();
            if constexpr (L1) {
                block_moments_all<false>(q, G, pl, M, sm.ys, 0, 1, i, sm.A);
                continue;
            }

            // WLS for output 1; output 0 is its exact negation (p0 = 1 - p1 row-wise)
            block_normal(pl, M, sm.A, i, p.status);
            block_solve_one(pl, M, sm.ys, p.dlink[(size_t)i * C + 1], sm.A, sm.rhs, sm.vi, p.phi + slab + (size_t)i * G);
            if (tid == 0) write_class0_negation(p.phi + (size_t)i * G, p.phi + slab + (size_t)i * G, M, sm.vi);
        } else if (softmax) {
            // ---- general softmax and one-vs-rest heads: R = C score rows, outputs softmax(scores) or the normalised
            // sigmoids of the scores; scale = log2(e) ----
            const int R = p.R;
            float* basesR = Bs + (size_t)R * M * N;      // [R][N]
            float* wbR = basesR + (size_t)R * N;         // [N]
            for (int idx = tid; idx < R * M * N; idx += blockDim.x) {
                const int r = idx / (M * N), rem = idx - r * (M * N), k = rem / N, j = rem - k * N;
                Bs[idx] = p.BWs[((size_t)r * G + sm.vi[k]) * N + j];
            }
            for (int idx = tid; idx < R * N; idx += blockDim.x) basesR[idx] = p.bases[idx];
            for (int j = tid; j < N; j += blockDim.x) wbR[j] = p.wbf[j];
            for (int idx = tid; idx < R * M; idx += blockDim.x) {
                const int r = idx / M, k = idx - r * M;
                sm.xw[r * 64 + k] = p.scale * p.XW[((size_t)i * G + sm.vi[k]) * R + r];
            }
            __syncthreads();
            for (int s = tid; s < S; s += blockDim.x) {
                const uint64_t z = zp[s];
                float af[8], acc[8];
                for (int r = 0; r < R; ++r) {
                    double a = 0;
                    for (int k = 0; k < M; ++k) if ((z >> k) & 1ull) a += sm.xw[r * 64 + k];
                    af[r] = (float)a;
                    acc[r] = 0.f;
                }
                for (int j = 0; j < N; ++j) {
                    float t[8], mx = -3.0e38f;
                    for (int r = 0; r < R; ++r) {
                        float c = 0.f;
                        const float* Br = Bs + (size_t)r * M * N;
                        for (int k = 0; k < M; ++k) if ((z >> k) & 1ull) c += Br[k * N + j];
                        t[r] = (basesR[r * N + j] - c) + af[r];
                        mx = fmaxf(mx, t[r]);
                    }
                    float den = 0.f;
                    if (ovr) {
                        // 2^-h sigmoid_r = 1 / (2^h + 2^(h - t_r)) with h = min(max_r t_r, 0): the leading class is at
                        // least 1/2, so den >= 1/2; classes 2^-128 below it overflow to 1 / inf = 0
                        const float h = fminf(mx, 0.f), eh = ex2_approx(h);
                        for (int r = 0; r < R; ++r) { t[r] = rcp_approx(eh + ex2_approx(h - t[r])); den += t[r]; }
                    } else {
                        for (int r = 0; r < R; ++r) { t[r] = ex2_approx(t[r] - mx); den += t[r]; }
                    }
                    const float inv = wbR[j] * rcp_approx(den);
                    for (int r = 0; r < R; ++r) acc[r] = fmaf(t[r], inv, acc[r]);
                }
                for (int c = 0; c < C; ++c) {
                    double y;
                    if (p.link == DKS_LINK_LOGIT) {
                        float rest = 0.f;                 // 1 - ey_c as the sum of the other classes: no cancellation
                        for (int c2 = 0; c2 < C; ++c2) if (c2 != c) rest += acc[c2];
                        y = log((double)acc[c] / (double)rest) - p.linkfnull[c];
                    } else {
                        y = (double)acc[c] - p.fnull[c];
                    }
                    sm.ys[(size_t)c * p.S_cap + s] = y;
                }
            }
            __syncthreads();
            if constexpr (L1) {
                block_moments_all<true>(q, G, pl, M, sm.ys, p.S_cap, C, (size_t)i * C, sm.A);
                continue;
            }
            block_normal(pl, M, sm.A, i, p.status);
            block_solve(p, i, pl, M, sm.ys, p.S_cap, C, false, sm.A, sm.rhs, sm.vi);
        } else if (p.act == DKS_ACT_IDENTITY) {
            // identity head: the background average commutes with the head, so
            // ey_r(s) = fnull_r + sum_k z_sk (XW_i[k][r] - Bbar[k][r])   -- float64 throughout
            if constexpr (!L1) block_normal(pl, M, sm.A, i, p.status);
            for (int r = 0; r < p.R; ++r) {
                __syncthreads();
                if (tid < M) {
                    int g = sm.vi[tid];
                    sm.xw[tid] = p.XW[((size_t)i * G + g) * p.R + r] - p.Bbar[(size_t)g * p.R + r];
                }
                __syncthreads();
                const double fn = p.fnull[r], lfn = p.linkfnull[r];
                for (int s = tid; s < S; s += blockDim.x) {
                    const uint64_t z = zp[s];
                    double a = fn;
                    for (int k = 0; k < M; ++k) if ((z >> k) & 1ull) a += sm.xw[k];
                    sm.ys[s] = link_f(a, p.link) - lfn;
                }
                __syncthreads();
                if constexpr (L1) {
                    block_moments_all<true>(q, G, pl, M, sm.ys, 0, 1, (size_t)i * C + r, sm.A);
                    continue;
                }
                block_solve_one(pl, M, sm.ys, p.dlink[(size_t)i * C + r], sm.A, sm.rhs, sm.vi,
                                p.phi + (size_t)r * slab + (size_t)i * G);
            }
        }
    }
}

}  // namespace dks
