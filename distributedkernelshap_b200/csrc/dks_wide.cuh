// Solve stage of the shared-plan path for plans of more than 128 groups (sixteen 64-bit words per coalition row; configs[3]
// of BASELINE.json read as 1024 singleton groups).
//
// The coalition stage is the shared-plan kernel of dks_shared.cuh (explain_shared_smem_kernel<NTAIL, 16>): it leaves
// (sum p1, sum p0) per (instance, coalition).  The (M-1) x (M-1) normal matrix -- 8 MB at M = 1024 -- no longer fits shared
// memory, and it does not have to: the plan is shared, so the projection P = inv(E^T W E) E^T W is formed ONCE on the host
// in float64 (plan.py: projection(), np.linalg.inv like upstream's solve) and uploaded transposed, PT [S_pad][KP], with
// dks_set_plan_projection.  Per batch of instances the solve is then
//     Y  [cnt x S]  = link(ey) - link(fnull)                     wide_link_kernel
//     B  [cnt x KP] = Y PT                                       wide_beta2_kernel  (float64 GEMM, CUDA cores)
//     phi_k = B_k - delta d_k,  phi_last = delta - sum_k phi_k   wide_finish_kernel
// All of it float64; every sum has a fixed order (no atomics), so results are reproducible run to run.
// Work per instance at M = 1024, S = 8192: 8.4 M float64 multiply-adds, about the cost of the coalition stage.
#pragma once

#ifdef DKS_HOST_EMULATION          // tests/emu: the kernels below run on host threads (no GPU in the build container)
#include "emu_shim.h"
#include "dks.h"
#include "dks_linkmath.cuh"
#else
#include "dks_kernels.cuh"
#endif

namespace dks {
namespace wide {

constexpr int BN = 64, BK = 16;              // tile of the Y PT product: 64 coefficients, 16 coalitions a step
constexpr int THREADS = 256;                 // 16 x 16 threads

inline int kpad(int M) { return (M - 1 + BN - 1) / BN * BN; }

struct WideParams {
    int n, N, G, C, S, S_pad, KP, link;
    const float2* sums;      // [n][S_pad] (sum p1, sum p0) of the coalition stage
    const double* PT;        // [S_pad][KP] projection, transposed, zero padded
    const double* dvec;      // [KP] P z_L
    const double* dlink;     // [n][C]
    const double* linkfnull;
    const double* fnull;
    const int* list;         // instances on this path
    const int* count;        // their number (device)
    double* y;               // [n][S_pad] workspace
    double* beta;            // [n][KP] workspace
    double* phi;             // [C][n][G]
};

// y[i][s] = link(ey_s) - link(fnull) for the listed instances; padding coalitions get 0
__global__ void __launch_bounds__(256) wide_link_kernel(WideParams p) {
    __shared__ LogTabEntry s_logtab[DKS_LOGTAB_SIZE];
    if (threadIdx.x < DKS_LOGTAB_SIZE) logtab_fill(s_logtab, threadIdx.x);
    __syncthreads();
    const int cnt = *p.count;
    const double lf1 = p.linkfnull[1], f1 = p.fnull[1], inv_n = 1.0 / (double)p.N;
    for (int m = blockIdx.y; m < cnt; m += gridDim.y) {
        const int i = p.list[m];
        const float2* sums = p.sums + (size_t)i * p.S_pad;
        double* y = p.y + (size_t)i * p.S_pad;
        for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < p.S_pad; s += gridDim.x * blockDim.x) {
            double v = 0.0;
            if (s < p.S) {
                const float2 a = sums[s];
                if (p.link == DKS_LINK_LOGIT) v = fast_log_ratio(a.x, a.y, s_logtab) - lf1;
                else v = (double)a.x * inv_n - f1;
            }
            y[s] = v;
        }
    }
}

// beta[i][k] = sum_s y[i][s] PT[s][k], coalition index ascending (fixed order).  A plain 64 x 64 tiling is bound by
// shared-memory loads (bank conflicts; FP64 pipe under a third active), so: 128 instances x 64 coefficients per CTA, 8 x 4
// outputs per thread, every shared-memory operand a 128-bit load: a thread's rows are 4 ty .. +3 and 64 + 4 ty .. +3 (a
// warp holds two values of ty: broadcasts), its columns 2 tx, 2 tx + 1 and 32 + 2 tx, 32 + 2 tx + 1 (sixteen consecutive
// 16-byte pieces per load: no conflicts).  Per coalition step 6 LDS.128 feed 32 DFMA.
constexpr int BM2 = 128;
__global__ void __launch_bounds__(THREADS) wide_beta2_kernel(WideParams p) {
    __shared__ __align__(16) double As[BK][BM2];     // y tile, transposed: [coalition][instance]
    __shared__ __align__(16) double Bs[BK][BN];      // PT tile: [coalition][coefficient]
    __shared__ int s_inst[BM2];
    const int cnt = *p.count;
    const int m0 = blockIdx.y * BM2, k0 = blockIdx.x * BN;
    if (m0 >= cnt) return;
    const int t = threadIdx.x;
    if (t < BM2) s_inst[t] = m0 + t < cnt ? p.list[m0 + t] : -1;
    __syncthreads();
    // loader roles: y tile -- instance t & 127, eight consecutive coalitions from 8 (t >> 7); PT tile -- coalition t >> 4,
    // four coefficients from 4 (t & 15)
    const int la_m = t & (BM2 - 1), la_k = (t >> 7) * 8;
    const int lb_k = t >> 4, lb_c = (t & 15) * 4;
    const int inst = s_inst[la_m];
    const double* yrow = inst >= 0 ? p.y + (size_t)inst * p.S_pad : nullptr;       // rows are 256-byte aligned (S_pad % 32 == 0)
    const int ty = t >> 4, tx = t & 15;
    double acc[8][4];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
    for (int s0 = 0; s0 < p.S_pad; s0 += BK) {
        if (yrow) {
            const double2* src = reinterpret_cast<const double2*>(yrow + s0 + la_k);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const double2 v = src[q];
                As[la_k + 2 * q][la_m] = v.x;
                As[la_k + 2 * q + 1][la_m] = v.y;
            }
        } else {
#pragma unroll
            for (int q = 0; q < 8; ++q) As[la_k + q][la_m] = 0.0;
        }
        const double2* prow = reinterpret_cast<const double2*>(p.PT + (size_t)(s0 + lb_k) * p.KP + k0 + lb_c);   // KP % 64 == 0
        *reinterpret_cast<double2*>(&Bs[lb_k][lb_c]) = prow[0];
        *reinterpret_cast<double2*>(&Bs[lb_k][lb_c + 2]) = prow[1];
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const double2 a0 = *reinterpret_cast<const double2*>(&As[kk][4 * ty]);
            const double2 a1 = *reinterpret_cast<const double2*>(&As[kk][4 * ty + 2]);
            const double2 a2 = *reinterpret_cast<const double2*>(&As[kk][64 + 4 * ty]);
            const double2 a3 = *reinterpret_cast<const double2*>(&As[kk][64 + 4 * ty + 2]);
            const double2 b0 = *reinterpret_cast<const double2*>(&Bs[kk][2 * tx]);
            const double2 b1 = *reinterpret_cast<const double2*>(&Bs[kk][32 + 2 * tx]);
            const double a[8] = {a0.x, a0.y, a1.x, a1.y, a2.x, a2.y, a3.x, a3.y};
            const double b[4] = {b0.x, b0.y, b1.x, b1.y};
#pragma unroll
            for (int r = 0; r < 8; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[r][c] = fma(a[r], b[c], acc[r][c]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const int i = s_inst[(r < 4 ? 0 : 64) + 4 * ty + (r & 3)];
        if (i < 0) continue;
        double* out = p.beta + (size_t)i * p.KP + k0;
        double2 lo, hi;
        lo.x = acc[r][0]; lo.y = acc[r][1]; hi.x = acc[r][2]; hi.y = acc[r][3];
        *reinterpret_cast<double2*>(out + 2 * tx) = lo;
        *reinterpret_cast<double2*>(out + 32 + 2 * tx) = hi;
    }
}

// one CTA per listed instance: phi_k = beta_k - delta d_k, the eliminated (last) group takes the remainder
__global__ void __launch_bounds__(256) wide_finish_kernel(WideParams p) {
    __shared__ double s_part[8];
    __shared__ double s_sum;
    const int cnt = *p.count;
    const int G = p.G, nA = G - 1;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const size_t slab = (size_t)p.n * G;
    for (int m = blockIdx.x; m < cnt; m += gridDim.x) {
        const int i = p.list[m];
        const double delta = p.dlink[(size_t)i * p.C + 1];
        const double* beta = p.beta + (size_t)i * p.KP;
        double part = 0.0;
        for (int k = threadIdx.x; k < nA; k += blockDim.x) part += beta[k] - delta * p.dvec[k];
        part = warp_sum(part);
        if (lane == 0) s_part[wib] = part;
        __syncthreads();
        if (threadIdx.x == 0) {
            double sum = 0.0;
            for (int w = 0; w < 8; ++w) sum += s_part[w];          // fixed order
            s_sum = sum;
        }
        __syncthreads();
        const double sum = s_sum;
        for (int k = threadIdx.x; k < G; k += blockDim.x) {
            double val = k < nA ? beta[k] - delta * p.dvec[k] : delta - sum;
            if (fabs(val) < 1e-10) val = 0.0;
            p.phi[slab + (size_t)i * G + k] = val;
            p.phi[(size_t)i * G + k] = (val == 0.0) ? 0.0 : -val;
        }
        __syncthreads();                                           // s_part / s_sum are reused by the next instance
    }
}

// launch geometry (shared with the host emulation)
inline dim3 link_grid(int S_pad, int n, int sm_count) {
    const int gx = (S_pad + 255) / 256 < 8 ? (S_pad + 255) / 256 : 8;
    return dim3(gx, n < 4 * sm_count ? n : 4 * sm_count);
}
inline dim3 beta2_grid(int KP, int n) { return dim3(KP / BN, (n + BM2 - 1) / BM2); }
inline int finish_grid(int n, int sm_count) { return n < 8 * sm_count ? n : 8 * sm_count; }

#ifndef DKS_HOST_EMULATION
// three launches on `stream`; n = instances of the call (upper bound of the device-side count)
inline cudaError_t launch_wide_solve(const WideParams& p, int n, int sm_count, cudaStream_t stream) {
    wide_link_kernel<<<link_grid(p.S_pad, n, sm_count), 256, 0, stream>>>(p);
    wide_beta2_kernel<<<beta2_grid(p.KP, n), THREADS, 0, stream>>>(p);
    wide_finish_kernel<<<finish_grid(n, sm_count), 256, 0, stream>>>(p);
    return cudaGetLastError();
}
#endif

}  // namespace wide
}  // namespace dks
