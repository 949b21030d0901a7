// Shared-plan path of the softmax head (C = R classes, 2..8): per-class coalition sums for instances whose groups all vary.
//
// The masked score separates per class as on the binary path (DESIGN.md §5.0.6):
//     t_c(i, s, j) = a_c(i, s) + d_c(s, j),   a_c = log2 e sum_k z_sk XW_i[k][c],   d_c = log2 e (score_jc - sum_k z_sk BW[j][k][c])
// p_c = 2^t_c / sum_c' 2^t_c' is unchanged when a term that does not depend on c is subtracted from every t_c, so
//     Dm_c(s, j) = 2^(d_c(s, j) - max_c' d_c'(s, j))   (plan upload: every entry in (0, 1], one class exactly 1)
//     A_c(i, s)  = 2^(a_c(i, s) - max_c' a_c'(i, s))   (per instance and row: every factor in (0, 1], one exactly 1)
// and with u_c = A_c Dm_c (no product can overflow: all u_c <= 1)
//     p_c = u_c / den,   den = sum_c u_c >= u_ca = Dm_ca(s, j),   ca = argmax_c a_c(i, s).
// lo_c(s) = min_j log2 Dm_c(s, j) therefore bounds den from below for every column at once: rows with lo_ca(s) >= -60 keep
// den >= 2^-60, and a probability of 2^-60 is still u_c >= 2^-120, a normal fp32 number.  One reciprocal serves all C
// classes of an element: 3C fp32 ops + 1 MUFU.  Rows with lo_ca(s) < -60 (scores saturated far apart) take a clamped
// scalar path that evaluates the element's softmax in float64 from the grouped background scores.
// Output: per-class fp32 sums  sum_j w'_j p_c(s, j)  with w'_j = N w_j (1 for a uniform background) -- the solve divides by
// N (identity link) or forms the ratio of a class to the sum of the other classes (logit link).
//
// One-vs-rest head (DESIGN.md §5.0.7): p_c = s_c / sum_c' s_c' with s_c = sigmoid(t_c) = 1 / (1 + 2^-t_c).  A sigmoid sees
// the absolute level of t_c, so the plan normalises by an integer instead of the class maximum:
//     nd(s, j) = ceil(max_c d_c(s, j)),  Dm_c(s, j) = 2^(d_c - nd) in (0, 1]   (nd is the one extra per-element quantity)
//     na(i, s) = ceil(max_c a_c(i, s)),  A_c(i, s)  = 2^(a_c - na)  in (0, 1]
// so that u_c = A_c Dm_c = 2^(t_c - k) with k = na + nd an exact integer.  With h = min(k, 0) the common factor 2^-h gives
//     r_c = 2^-h s_c = u_c / (alpha + beta u_c),   alpha = 2^-max(k, 0),  beta = 2^min(k, 0)
// (both exact powers of two, built from k with integer ops) and p_c = r_c / sum_c r_c: C reciprocals for the sigmoids and
// one for the normalisation per element.  hi(s) = max_j nd(s, j) bounds k from above for every column: rows with
// lo_ca(s) >= -60 and na + hi(s) <= 64 keep alpha >= 2^-64 and den >= 2^-62, so every p_c >= 2^-60 has u_c >= 2^-125, a
// normal fp32 number.  Other rows take the clamped scalar path, which forms log2 s_c in float64.
#pragma once

#include "dks_shared.cuh"

namespace dks {
namespace multi {

constexpr int MC_WARPS = 8;           // warps per CTA; they share the CTA's 32 coalition rows and split the instances
constexpr int MC_MAXN = 128;          // background columns per launch
constexpr float MC_LO_MIN = -60.f;    // rows whose den could fall below 2^-60 take the clamped path
constexpr double OVR_K_MAX = 64.0;    // one-vs-rest: rows whose k = na + nd could exceed 64 take the clamped path
constexpr double OVR_ND_MAX = 1048576.0;   // |nd| clamp (rows beyond it are clamped rows): k never overflows an int

// word of a one- or two-word coalition row holding bit k / nibble t (no dynamic index: the row stays in registers)
template <int W>
__device__ __forceinline__ uint64_t zword(const uint64_t (&zz)[W], int k) { return (W == 1 || k < 64) ? zz[0] : zz[W - 1]; }
template <int W>
__device__ __forceinline__ int znib(const uint64_t (&zz)[W], int t) { return (int)((zword<W>(zz, 4 * t) >> (4 * (t & 15))) & 15ull); }

// d_c(s, j) for the classes c < C <= CM, float64 (BW [N][G][C], scores [N][C])
template <int W, int CM>
__device__ __forceinline__ void plan_dc(const uint64_t (&zz)[W], const double* __restrict__ BW, const double* __restrict__ scores,
                                        int j, int G, int C, double scale, double (&d)[CM]) {
#pragma unroll
    for (int c = 0; c < CM; ++c) d[c] = 0.0;
    for (int k = 0; k < G; ++k)
        if ((zword<W>(zz, k) >> (k & 63)) & 1ull) {
#pragma unroll
            for (int c = 0; c < CM; ++c) if (c < C) d[c] += BW[((size_t)j * G + k) * C + c];
        }
#pragma unroll
    for (int c = 0; c < CM; ++c) d[c] = c < C ? scale * (scores[(size_t)j * C + c] - d[c]) : -1.0e300;
}

// one thread per coalition row: Dm [C][N][S_pad] and lo [C][S_pad] (padding rows: Dm = 1, lo = 0).  OVR: Dm_c is taken
// relative to nd = ceil(max_c d_c), stored as int bits in Dm slot C, and lo slot C holds hi = max_j nd
template <int W, bool OVR>
__device__ __forceinline__ void plan_tables(const uint64_t* __restrict__ z, int S, int S_pad, const double* __restrict__ BW,
                                            const double* __restrict__ scores, int N, int G, int C, double scale,
                                            float* __restrict__ dm, float* __restrict__ lo) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S_pad) return;
    uint64_t zz[W];
#pragma unroll
    for (int w = 0; w < W; ++w) zz[w] = s < S ? z[(size_t)s * W + w] : 0ull;
    double lmin[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) lmin[c] = 0.0;
    double hi = -1.0e30;
    for (int j = 0; j < N; ++j) {
        double d[8];
        plan_dc<W, 8>(zz, BW, scores, j, G, C, scale, d);
        double mx = d[0];
#pragma unroll
        for (int c = 1; c < 8; ++c) mx = fmax(mx, d[c]);
        if (OVR) {
            const double nd = s < S ? fmin(fmax(ceil(mx), -OVR_ND_MAX), OVR_ND_MAX) : 0.0;
            hi = fmax(hi, mx > OVR_ND_MAX ? 1.0e30 : nd);
            dm[((size_t)C * N + j) * S_pad + s] = __int_as_float((int)nd);
            mx = nd;
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            if (c < C) {
                const double e = s < S ? d[c] - mx : 0.0;
                lmin[c] = fmin(lmin[c], e);
                dm[((size_t)c * N + j) * S_pad + s] = (float)exp2(e);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) if (c < C) lo[(size_t)c * S_pad + s] = (float)fmax(lmin[c], -1.0e30);
    if (OVR) lo[(size_t)C * S_pad + s] = (float)hi;
}

template <int W>
__global__ void plan_softmax_kernel(const uint64_t* __restrict__ z, int S, int S_pad, const double* __restrict__ BW,
                                    const double* __restrict__ scores, int N, int G, int C, double scale,
                                    float* __restrict__ dm, float* __restrict__ lo) {
    plan_tables<W, false>(z, S, S_pad, BW, scores, N, G, C, scale, dm, lo);
}

// one-vs-rest head: Dm [C + 1][N][S_pad] (slot C: nd as int bits), lo [C + 1][S_pad] (slot C: hi)
template <int W>
__global__ void plan_ovr_kernel(const uint64_t* __restrict__ z, int S, int S_pad, const double* __restrict__ BW,
                                const double* __restrict__ scores, int N, int G, int C, double scale,
                                float* __restrict__ dm, float* __restrict__ lo) {
    plan_tables<W, true>(z, S, S_pad, BW, scores, N, G, C, scale, dm, lo);
}

struct SoftmaxParams {
    int n, N, G, S, S_pad, ntab;
    int j0, nc;              // background columns j0 .. j0 + nc of this launch
    int accumulate;          // add to the sums (second and later launches)
    double scale;            // log2 e
    const float* dm;         // [C][N][S_pad] ([C + 1][N][S_pad] for the one-vs-rest head)
    const float* lo;         // [C][S_pad] ([C + 1][S_pad])
    const float* wn;         // [N] N w_j
    const uint64_t* z;       // [S][W]
    const double* XT;        // [n][C][ntab][16] nibble tables of log2 e XW
    const double* BW;        // [N][G][C] (clamped path)
    const double* scores;    // [N][C]
    const int* list;
    const int* count;
    float* sums;             // [n][C][S_pad]
};

// CS = table slots per column: C, or C + 1 for the one-vs-rest head (nd)
__host__ __device__ inline size_t softmax_smem(int CS, int nc) { return sizeof(float) * ((size_t)32 * nc * CS + nc); }

// CTA = 32 coalition rows (lane = row) x MC_WARPS warps, each warp one instance at a time; the rows' Dm entries for all
// classes and the launch's columns sit in shared memory as [column][class][lane] (conflict-free, the weights after them)
template <bool OVR, int C, int W>
__device__ __forceinline__ void class_sums(const SoftmaxParams& p) {
    constexpr int CS = OVR ? C + 1 : C;
    extern __shared__ float s_mc[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nc = p.nc, N = p.N, S_pad = p.S_pad;
    const int s = blockIdx.x * 32 + lane;
    float* s_w = s_mc + (size_t)32 * nc * CS;
    for (int idx = threadIdx.x; idx < 32 * nc * CS; idx += blockDim.x) {
        const int l = idx & 31, q = idx >> 5, c = q % CS, j = q / CS;
        s_mc[idx] = p.dm[((size_t)c * N + p.j0 + j) * S_pad + blockIdx.x * 32 + l];
    }
    for (int j = threadIdx.x; j < nc; j += blockDim.x) s_w[j] = p.wn[p.j0 + j];
    __syncthreads();
    const int cnt = *p.count;
    uint64_t zz[W];
#pragma unroll
    for (int w = 0; w < W; ++w) zz[w] = s < p.S ? p.z[(size_t)s * W + w] : 0ull;
    const int ntab = p.ntab;
    for (int m = blockIdx.y * MC_WARPS + warp; m < cnt; m += gridDim.y * MC_WARPS) {
        const int i = p.list[m];
        const double* xt = p.XT + (size_t)i * C * ntab * 16;
        double a[C];
#pragma unroll
        for (int c = 0; c < C; ++c) {
            double a0 = 0.0, a1 = 0.0;
            for (int t = 0; t < ntab; t += 2) {
                a0 += __ldg(xt + (c * ntab + t) * 16 + znib<W>(zz, t));
                if (t + 1 < ntab) a1 += __ldg(xt + (c * ntab + t + 1) * 16 + znib<W>(zz, t + 1));
            }
            a[c] = a0 + a1;
        }
        double amax = a[0];
        int ca = 0;
#pragma unroll
        for (int c = 1; c < C; ++c) if (a[c] > amax) { amax = a[c]; ca = c; }
        if (OVR) amax = ceil(amax);                          // na: A_c relative to an integer
        float acc[C];
#pragma unroll
        for (int c = 0; c < C; ++c) acc[c] = 0.f;
        const bool clamped = s < p.S && (p.lo[(size_t)ca * S_pad + s] < MC_LO_MIN ||
                                         (OVR && amax + (double)p.lo[(size_t)C * S_pad + s] > OVR_K_MAX));
        if (!clamped) {
            float A[C];
#pragma unroll
            for (int c = 0; c < C; ++c) {
                // 2^(a_c - amax) = 2^n 2^f, f exact in fp32 (|f| <= 1/2); factors below 2^-125 are negligible next to den
                const double e = a[c] - amax;
                const double en = rint(e);
                A[c] = e < -125.0 ? 0.f : ex2_approx((float)(e - en)) * __int_as_float((127 + (int)en) << 23);
            }
            const int ka = OVR ? (int)fmin(fmax(amax, -2.0 * OVR_ND_MAX), 2.0 * OVR_ND_MAX) : 0;
#pragma unroll 4
            for (int j = 0; j < nc; ++j) {
                const float* col = s_mc + (size_t)j * CS * 32 + lane;
                float u[C];
                float den = 0.f;
                if (OVR) {
                    // r_c = u_c / (alpha + beta u_c); k <= 64 on this path, k <= -127 makes beta exactly 0
                    const int k = ka + __float_as_int(col[C * 32]);
                    const float alpha = __int_as_float((127 - max(k, 0)) << 23);
                    const float beta = __int_as_float((127 + max(min(k, 0), -127)) << 23);
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        const float uc = A[c] * col[c * 32];
                        u[c] = uc * rcp_approx(fmaf(beta, uc, alpha));
                        den += u[c];
                    }
                } else {
#pragma unroll
                    for (int c = 0; c < C; ++c) { u[c] = A[c] * col[c * 32]; den += u[c]; }
                }
                const float rw = s_w[j] * rcp_approx(den);
#pragma unroll
                for (int c = 0; c < C; ++c) acc[c] = fmaf(u[c], rw, acc[c]);
            }
        } else {
            for (int j = 0; j < nc; ++j) {
                double d[C];
                plan_dc<W, C>(zz, p.BW, p.scores, p.j0 + j, p.G, C, p.scale, d);
                double mx = -1.0e300;
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    d[c] += a[c];
                    // one-vs-rest: log2 sigmoid(t) = min(t, 0) - log2(1 + 2^-|t|); the softmax of these is p_c
                    if (OVR) d[c] = fmin(d[c], 0.0) - 1.4426950408889634 * log1p(exp2(-fabs(d[c])));
                    mx = fmax(mx, d[c]);
                }
                double den = 0.0;
#pragma unroll
                for (int c = 0; c < C; ++c) { d[c] = exp2(d[c] - mx); den += d[c]; }
                const double rw = (double)s_w[j] / den;
#pragma unroll
                for (int c = 0; c < C; ++c) acc[c] += (float)(d[c] * rw);
            }
        }
        if (s < p.S) {
            float* dst = p.sums + (size_t)i * C * S_pad + s;
#pragma unroll
            for (int c = 0; c < C; ++c) dst[(size_t)c * S_pad] = p.accumulate ? dst[(size_t)c * S_pad] + acc[c] : acc[c];
        }
    }
}

template <int C, int W>
__global__ void __launch_bounds__(32 * MC_WARPS) explain_softmax_kernel(SoftmaxParams p) { class_sums<false, C, W>(p); }

// (two CTAs per SM stated explicitly: left to itself ptxas spills the C = 4, 5 instantiations at 64 registers)
template <int C, int W>
__global__ void __launch_bounds__(32 * MC_WARPS, 2) explain_ovr_kernel(SoftmaxParams p) { class_sums<true, C, W>(p); }

// Launches the softmax (ovr = false) or one-vs-rest class-sum kernel over background chunks of MC_MAXN columns (sums
// accumulated).  Returns the number of launches, 0 when one could not be configured; *grid_out reports the CTAs.
inline int launch_class_sums(SoftmaxParams p, bool ovr, int C, int words, int n, int sm_count, int max_smem,
                             cudaStream_t stream, int* grid_out) {
    const int N = p.N, n_rg = p.S_pad / 32, CS = ovr ? C + 1 : C;
    const int per_sm_fit = (int)((size_t)max_smem / (softmax_smem(CS, N < MC_MAXN ? N : MC_MAXN) + 1024));
    const int resident = sm_count * (per_sm_fit < 1 ? 1 : per_sm_fit);
    int gy = (2 * resident + n_rg - 1) / n_rg;               // two waves of CTAs over the row groups
    const int gy_max = (n + MC_WARPS - 1) / MC_WARPS;
    if (gy > gy_max) gy = gy_max;
    if (gy < 1) gy = 1;
    const dim3 grid(n_rg, gy);
    *grid_out = n_rg * gy;
    int launches = 0;
    for (int j0 = 0; j0 < N; j0 += MC_MAXN, ++launches) {
        p.j0 = j0;
        p.nc = N - j0 < MC_MAXN ? N - j0 : MC_MAXN;
        p.accumulate = j0 > 0;
        const size_t smem = softmax_smem(CS, p.nc);
        if (smem > (size_t)max_smem) return 0;
        cudaError_t err = cudaErrorInvalidValue;
#define DKS_MC(KERN, CC, WW)                                                                                              \
    if (C == CC && words == WW) {                                                                                        \
        err = cudaFuncSetAttribute(KERN<CC, WW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);                \
        if (err == cudaSuccess) KERN<CC, WW><<<grid, 32 * MC_WARPS, smem, stream>>>(p);                                  \
    }
        if (!ovr) {
            DKS_MC(explain_softmax_kernel, 2, 1) DKS_MC(explain_softmax_kernel, 3, 1) DKS_MC(explain_softmax_kernel, 4, 1)
            DKS_MC(explain_softmax_kernel, 5, 1) DKS_MC(explain_softmax_kernel, 6, 1) DKS_MC(explain_softmax_kernel, 7, 1)
            DKS_MC(explain_softmax_kernel, 8, 1) DKS_MC(explain_softmax_kernel, 2, 2) DKS_MC(explain_softmax_kernel, 3, 2)
            DKS_MC(explain_softmax_kernel, 4, 2) DKS_MC(explain_softmax_kernel, 5, 2) DKS_MC(explain_softmax_kernel, 6, 2)
            DKS_MC(explain_softmax_kernel, 7, 2) DKS_MC(explain_softmax_kernel, 8, 2)
        } else {
            DKS_MC(explain_ovr_kernel, 3, 1) DKS_MC(explain_ovr_kernel, 4, 1) DKS_MC(explain_ovr_kernel, 5, 1)
            DKS_MC(explain_ovr_kernel, 6, 1) DKS_MC(explain_ovr_kernel, 7, 1) DKS_MC(explain_ovr_kernel, 8, 1)
            DKS_MC(explain_ovr_kernel, 3, 2) DKS_MC(explain_ovr_kernel, 4, 2) DKS_MC(explain_ovr_kernel, 5, 2)
            DKS_MC(explain_ovr_kernel, 6, 2) DKS_MC(explain_ovr_kernel, 7, 2) DKS_MC(explain_ovr_kernel, 8, 2)
        }
#undef DKS_MC
        if (err != cudaSuccess) return 0;
    }
    return launches;
}

}  // namespace multi
}  // namespace dks
