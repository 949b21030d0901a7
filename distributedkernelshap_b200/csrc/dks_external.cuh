// Models the engine cannot evaluate itself (DESIGN.md §5.0.19): a torch.nn.Module on the device, which the caller runs between
// the engine's launches.  A black box has no tables to fold a coalition into, so every coalition row s of instance i is
// materialised against every background row j: external_mask_kernel writes z_s(group(d)) ? x_i[d] : bg_j[d] in the module's
// dtype, the caller runs the module on those rows, and external_reduce_kernel forms ey[i][c][s] = sum_j w_j y(i, s, j)_c in
// the [n][C][S_cap] layout explain_ensemble_tail_kernel reads.  Rows are numbered flat: instances in index order (those with
// M >= 2), then coalition s of the instance's plan, then background row j.
#pragma once

#include "dks_kernels.cuh"

namespace dks {
namespace ext {

constexpr int SCAN_THREADS = 1024;
constexpr int MASK_THREADS = 256;
constexpr int MASK_COALITIONS = 8;    // coalitions per CTA of the mask kernel
constexpr int REDUCE_THREADS = 256;   // one warp per coalition

// dks_external_* dtypes of the module's inputs and outputs
__device__ __forceinline__ double load_out(const void* y, int f64, size_t k) {
    return f64 ? static_cast<const double*>(y)[k] : (double)static_cast<const float*>(y)[k];
}

// out [n][C] = the module's outputs y (float32 or float64) in float64 and, with dlink, link(y) - linkfnull (predict_epilogue:
// a non-finite dlink is DKS_ERR_NUMERIC with the row)
__global__ void external_load_kernel(const void* __restrict__ y, int f64, int n, int C, int link,
                                     const double* __restrict__ linkfnull, double* __restrict__ out,
                                     double* __restrict__ dlink, int* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double o[DKS_ENS_MAX_OUT];
    for (int c = 0; c < C; ++c) o[c] = load_out(y, f64, (size_t)i * C + c);
    predict_epilogue(o, C, i, link, linkfnull, out, dlink, status, false);
}

// soff [n + 1]: exclusive prefix sum over instances of their coalitions S_i (0 for M < 2), one CTA.  An instance whose
// shared plan is missing is DKS_ERR_PLAN_MISSING with its M, one whose S exceeds S_cap DKS_ERR_INVALID, each with S_i = 0.
__global__ void __launch_bounds__(SCAN_THREADS) external_offsets_kernel(ExplainParams p, long long* __restrict__ soff) {
    __shared__ long long warp_tot[SCAN_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int per = (p.n + SCAN_THREADS - 1) / SCAN_THREADS;
    const int lo = min(p.n, tid * per), hi = min(p.n, lo + per);
    long long mine = 0;
    for (int i = lo; i < hi; ++i) {
        const int M = p.Mcnt[i];
        if (M < 2) continue;
        const int S = dks_effective_S(M, p.S_req);
        if (p.ext_z == nullptr && (p.plans[M].z == nullptr || p.plans[M].S != S)) {
            report_status(p.status, DKS_ERR_PLAN_MISSING, M);
            continue;
        }
        if (S > p.S_cap) {
            report_status(p.status, DKS_ERR_INVALID, i);
            continue;
        }
        mine += S;
    }
    long long incl = mine;                                      // inclusive scan over the block, warp by warp
    for (int o = 1; o < 32; o <<= 1) {
        const long long v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        long long t = warp_tot[lane];
        for (int o = 1; o < 32; o <<= 1) {
            const long long v = __shfl_up_sync(0xffffffffu, t, o);
            if (lane >= o) t += v;
        }
        warp_tot[lane] = t;
    }
    __syncthreads();
    long long run = incl - mine + (wid > 0 ? warp_tot[wid - 1] : 0);
    for (int i = lo; i < hi; ++i) {
        soff[i] = run;
        const int M = p.Mcnt[i];
        if (M < 2) continue;
        const int S = dks_effective_S(M, p.S_req);
        if ((p.ext_z == nullptr && (p.plans[M].z == nullptr || p.plans[M].S != S)) || S > p.S_cap) continue;
        run += S;
    }
    if (tid == SCAN_THREADS - 1) soff[p.n] = run;
}

// the instance whose coalitions hold global coalition q: soff[i] <= q < soff[i + 1]
__device__ __forceinline__ int instance_of(const long long* __restrict__ soff, int n, long long q) {
    int lo = 0, hi = n;                                         // last i with soff[i] <= q
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (soff[mid] <= q) lo = mid; else hi = mid;
    }
    return lo;
}

// masked rows out [(q1 - q0) N][D] of coalitions q0 .. q1 - 1: MASK_COALITIONS coalitions per CTA, their on-groups (the
// coalition's bits deposited on the instance's varying groups) resolved once, then the CTA's rows stored flat
template <typename T>
__global__ void __launch_bounds__(MASK_THREADS) external_mask_kernel(ExplainParams p, const long long* __restrict__ soff,
                                                                     long long q0, long long q1,
                                                                     const double* __restrict__ X,
                                                                     const double* __restrict__ bg, int D,
                                                                     const int* __restrict__ colgrp, T* __restrict__ out) {
    __shared__ uint64_t on[MASK_COALITIONS];
    __shared__ int inst[MASK_COALITIONS];
    const long long c0 = q0 + (long long)blockIdx.x * MASK_COALITIONS;
    const int nc = (int)min((long long)MASK_COALITIONS, q1 - c0);
    if (threadIdx.x < nc) {
        const long long q = c0 + threadIdx.x;
        const int i = instance_of(soff, p.n, q);
        const int s = (int)(q - soff[i]);
        const int M = p.Mcnt[i];
        const uint64_t* z = p.ext_z ? p.ext_z + (size_t)i * p.ext_stride : p.plans[M].z;
        const uint64_t zs = z[s];
        uint64_t vm = p.vmask[i], g_on = 0;
        for (int k = 0; vm; ++k, vm &= vm - 1)                 // bit k of z_s -> the k-th varying group
            if ((zs >> k) & 1ull) g_on |= vm & (~vm + 1);
        on[threadIdx.x] = g_on;
        inst[threadIdx.x] = i;
    }
    __syncthreads();
    const long long row_base = (c0 - q0) * p.N;                 // first row of this CTA in out
    const int total = nc * p.N * D;
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
        const int r = e / D, d = e - r * D;                     // row within the CTA, column
        const int k = r / p.N, j = r - k * p.N;
        const bool x_on = (on[k] >> colgrp[d]) & 1ull;
        const double v = x_on ? X[(size_t)inst[k] * D + d] : bg[(size_t)j * D + d];
        out[(size_t)row_base * D + e] = (T)v;                   // float64 -> float32: round to nearest
    }
}

// ey[i][c][s] = sum_j w_j y(i, s, j)_c for coalitions q0 .. q1 - 1 from the module's outputs y [(q1 - q0) N][C]: one warp per
// coalition, lane l summing j = l, l + 32, ... in order, then a fixed shuffle tree (the same sums whatever the block split)
template <typename T>
__global__ void __launch_bounds__(REDUCE_THREADS) external_reduce_kernel(const long long* __restrict__ soff, int n, int N,
                                                                         int C, int S_cap, long long q0, long long q1,
                                                                         const T* __restrict__ y,
                                                                         const double* __restrict__ wbg,
                                                                         double* __restrict__ ey) {
    const int lane = threadIdx.x & 31;
    const long long nwarps = (long long)gridDim.x * (REDUCE_THREADS / 32);
    for (long long q = q0 + (long long)blockIdx.x * (REDUCE_THREADS / 32) + (threadIdx.x >> 5); q < q1; q += nwarps) {
        const T* yq = y + (size_t)(q - q0) * N * C;
        double acc[DKS_ENS_MAX_OUT];
#pragma unroll
        for (int c = 0; c < DKS_ENS_MAX_OUT; ++c) acc[c] = 0.0;
        for (int j = lane; j < N; j += 32) {
            const double w = wbg[j];
#pragma unroll
            for (int c = 0; c < DKS_ENS_MAX_OUT; ++c)
                if (c < C) acc[c] = fma(w, (double)yq[(size_t)j * C + c], acc[c]);
        }
#pragma unroll
        for (int c = 0; c < DKS_ENS_MAX_OUT; ++c)
            for (int o = 16; o > 0; o >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
        if (lane == 0) {
            const int i = instance_of(soff, n, q);
            const int s = (int)(q - soff[i]);
#pragma unroll
            for (int c = 0; c < DKS_ENS_MAX_OUT; ++c)
                if (c < C) ey[((size_t)i * C + c) * S_cap + s] = acc[c];
        }
    }
}

}  // namespace ext
}  // namespace dks
