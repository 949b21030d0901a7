// Soft-voting ensembles on the device (DESIGN.md §5.0.17): f = sum_k pi_k f_k over K members, each a tree ensemble, a kernel
// machine, an MLP or a neighbour model (dks_set_ensemble).  Soft voting is linear in the members, so the background mean of
// every coalition row is ey(s) = sum_k pi_k ey_k(s): each member's explain kernel, in its ACC instantiation, forms its
// ey_k(s) as it always does and adds it, times pi_k, into one workspace ey [n][C][S_cap] (members in order, on one stream);
// explain_ensemble_tail_kernel then takes the link and the solve once.
#pragma once

#include "dks_kernels.cuh"

namespace dks {
namespace ens {

constexpr int THREADS = 256;      // = l1::MOM_THREADS: the l1 instantiation forms the moments with block_moments

// f(x) [n][C] = sum_k pi_k out_k [K][n][C] (members in order) and, with dlink, link(f(x)) - link(fnull) for stage 1.  A row a
// member refused is already reported (DKS_ERR_DOMAIN) by that member's predict kernel, which runs first.
__global__ void ensemble_predict_kernel(const double* __restrict__ outk, int K, const double* __restrict__ pi, int n, int C,
                                        int link, const double* __restrict__ linkfnull, double* __restrict__ out,
                                        double* __restrict__ dlink, int* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double o[DKS_ENS_MAX_OUT];
    for (int c = 0; c < C; ++c) {
        double f = 0.0;
        for (int k = 0; k < K; ++k) f += pi[k] * outk[((size_t)k * n + i) * C + c];
        o[c] = f;
    }
    predict_epilogue(o, C, i, link, linkfnull, out, dlink, status, false);
}

// shared memory of explain_ensemble_tail_kernel: y [C][S_cap], the normal matrix [63 * 63], rhs [64] and the varying groups
__host__ __device__ inline size_t tail_smem_bytes(int S_cap, int C) {
    return sizeof(double) * ((size_t)C * S_cap + 63 * 63 + 64) + sizeof(int) * 64;
}

// One CTA per instance (grid-stride) over the list the members ran on.  M = 0 and M = 1 from the ensemble's dlink; else
// y = link(ey) - link(fnull) for every output (each solved on its own, as shap does), then the CUDA-core kernel's
// constrained WLS, or (L1) the moments of y for l1_lars_kernel.  Under the logit 1 - ey_c is, for a soft-voting ensemble
// of probabilities that sum to one, the sum of the other outputs' ey (no cancellation); with `complement` (a model whose
// outputs need not sum to one, dks_external.cuh) it is 1 - ey_c itself, the elementwise logit stage 1 and fnull take.  A
// non-finite y or f(x) is reported as DKS_ERR_NUMERIC and nothing of the instance is written.
template <bool L1>
__global__ void __launch_bounds__(THREADS) explain_ensemble_tail_kernel(ExplainParams p, SimtL1 q,
                                                                        const double* __restrict__ ey, int complement) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x;
    const int G = p.G, C = p.C;
    double* y = reinterpret_cast<double*>(smem_raw);            // [C][S_cap]
    double* A = y + (size_t)C * p.S_cap;                        // [63 * 63]
    double* rhs = A + 63 * 63;                                  // [64]
    int* vi = reinterpret_cast<int*>(rhs + 64);                 // [64]
    const size_t slab = (size_t)p.n * G;

    const int ninst = dks_inst_count(p);
    for (int qi = blockIdx.x; qi < ninst; qi += gridDim.x) {
        const int i = dks_inst_at(p, qi);
        const int M = p.Mcnt[i];
        const uint64_t vm = p.vmask[i];
        __syncthreads();  // previous instance done with shared memory
        zero_phi_rows(p, i);
        bool fx_bad = false;                                    // a member refused the row, or link(f(x)) is not finite
        for (int c = 0; c < C; ++c) fx_bad |= !isfinite(p.dlink[(size_t)i * C + c]);
        if (M == 0) continue;
        if (M == 1) {
            // the one varying group takes link(f(x)) - link(fnull) of every output
            if (tid < C && !fx_bad)
                p.phi[(size_t)tid * slab + (size_t)i * G + (__ffsll((long long)vm) - 1)] = p.dlink[(size_t)i * C + tid];
            continue;
        }
        InstPlan pl;
        if (!inst_plan(p, i, M, pl)) continue;
        if (fx_bad) {
            if (L1) moments_skip(q, G, M, C, (size_t)i * C);
            continue;
        }
        const int S = pl.S;
        varying_positions(vm, G, vi);
        const double* e = ey + (size_t)i * C * p.S_cap;
        int bad = 0;
        for (int s = tid; s < S; s += blockDim.x)
            for (int c = 0; c < C; ++c) {
                const double ec = e[(size_t)c * p.S_cap + s];
                double v;
                if (p.link == DKS_LINK_LOGIT) {
                    double rest = 0.0;
                    if (C == 1 || complement) rest = 1.0 - ec;
                    else for (int c2 = 0; c2 < C; ++c2) if (c2 != c) rest += e[(size_t)c2 * p.S_cap + s];
                    v = log(ec / rest) - p.linkfnull[c];
                } else {
                    v = ec - p.fnull[c];
                }
                bad |= !isfinite(v);
                y[(size_t)c * p.S_cap + s] = v;
            }
        if (__syncthreads_or(bad)) {
            if (tid == 0) report_status(p.status, DKS_ERR_NUMERIC, i);
            if (L1) moments_skip(q, G, M, C, (size_t)i * C);
            continue;
        }
        if constexpr (L1) {
            block_moments_all<true>(q, G, pl, M, y, p.S_cap, C, (size_t)i * C, A);
            continue;
        }
        block_normal(pl, M, A, i, p.status);
        block_solve(p, i, pl, M, y, p.S_cap, C, false, A, rhs, vi);
    }
}

}  // namespace ens
}  // namespace dks
