// Mixture head on the CUDA-core kernel (DESIGN.md §5.0.10): outputs p(x) = sum_k pi_k h(z_k(x)) over K members that share
// one member head h -- binary-logistic, softmax or one-vs-rest.  The background mean and the member mean are both weighted
// sums, so they commute: ey(s) = sum_k pi_k [sum_j w_j h(t_k(s, j))], and each bracket is what the single-model kernel sums.
// This kernel evaluates every member's head per (coalition, background row) and adds pi_k w_j h(.) into one fp32 sum per
// output; everything after the sums (link, constrained WLS or the l1 moments) is the CUDA-core kernel's.
#pragma once

#include "dks_kernels.cuh"

namespace dks {
namespace mix {

// fit: the background contributions and scores split per member, BWm [K][N][G][R_m] and scm [K][N][R_m], so that each
// member's plan tables come from the single-model plan kernels
__global__ void mix_split_kernel(const double* __restrict__ BW, const double* __restrict__ scores, int N, int G, int K, int Rm,
                                 double* __restrict__ BWm, double* __restrict__ scm) {
    const int R = K * Rm;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * G * R) return;
    const int q = (int)(idx % Rm), g = (int)((idx / Rm) % G), j = (int)((idx / ((long long)Rm * G)) % N);
    const int k = (int)(idx / ((long long)Rm * G * N));
    BWm[idx] = BW[((size_t)j * G + g) * R + k * Rm + q];
    if (g == 0) scm[((size_t)k * N + j) * Rm + q] = scores[(size_t)j * R + k * Rm + q];
}

// shared-plan route: dst (+)= pi_k src over the listed instances' rows of `stride` floats (a member's sums into the
// mixture's; first: store instead of add)
__global__ void mix_axpy_kernel(const float* __restrict__ src, float* __restrict__ dst, float pi, int first,
                                const int* __restrict__ list, const int* __restrict__ count, int stride) {
    const long long total = (long long)*count * stride;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int q = (int)(idx / stride);
        const size_t off = (size_t)list[q] * stride + (size_t)(idx - (long long)q * stride);
        dst[off] = first ? pi * src[off] : fmaf(pi, src[off], dst[off]);
    }
}

// shared memory: the CUDA-core kernel's layout with all R = K R_m score rows staged and one y buffer per solved output
inline size_t smem_bytes(int S_cap, int N, int Mmax, const MixHead& mh, int C) {
    const bool binary = mh.mact == DKS_ACT_BINARY_LOGISTIC;
    return simt_smem_bytes(S_cap, N, Mmax, mh.K * mh.Rm, binary ? 1 : C);
}

// One CTA per instance (grid-stride), one thread per coalition row, any plan source (shared, per-instance, caller-supplied).
// Scores are staged scaled by log2(e) (the head's scale), so the exponent of member row r is t_r = log2(e) z_r(s, j).
//   binary members (R_m = 1): u = 2^-t (t clamped to +-120), p1 = 1 / (1 + u), p0 = u p1 -- the binary head's pair, so
//     that sum p0 carries no cancellation and the logit link reads log(sum p1 / sum p0);
//   softmax members: 2^(t_q - max) / sum;  one-vs-rest members: the normalised sigmoids formed as in the one-vs-rest head.
// pi_k w_j multiplies the member's normalised outputs once per element.  L1: stores the moments of y for l1_lars_kernel.
template <bool L1>
__global__ void __launch_bounds__(256, L1 ? 1 : 2) explain_simt_mix_kernel(ExplainParams p, SimtL1 q, MixHead mh) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const bool binary = mh.mact == DKS_ACT_BINARY_LOGISTIC, ovr = mh.mact == DKS_ACT_OVR;
    const int R = p.R, Rm = mh.Rm, K = mh.K;
    SimtSmem sm = simt_carve(smem_raw, p.S_cap, R, binary ? 1 : p.C);
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
            if (tid < C) {
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

        float* Bs = sm.Bs;                              // [R][M][N] scaled background contributions of the varying groups
        float* basesR = Bs + (size_t)R * M * N;         // [R][N]    scaled background scores
        float* wbR = basesR + (size_t)R * N;            // [N]       background weights
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
            float af[DKS_MIX_MAX_R], acc[8];
            for (int r = 0; r < R; ++r) {
                double a = 0;
                for (int k = 0; k < M; ++k) if ((z >> k) & 1ull) a += sm.xw[r * 64 + k];
                af[r] = (float)a;
            }
            for (int c = 0; c < 8; ++c) acc[c] = 0.f;
            for (int j = 0; j < N; ++j) {
                const float wj = wbR[j];
                for (int m = 0; m < K; ++m) {
                    const float pw = mh.pif[m] * wj;
                    float t[8], mx = -3.0e38f;
                    for (int u = 0; u < Rm; ++u) {
                        const int r = m * Rm + u;
                        const float* Br = Bs + (size_t)r * M * N;
                        float c = 0.f;
                        for (int k = 0; k < M; ++k) if ((z >> k) & 1ull) c += Br[k * N + j];
                        t[u] = (basesR[r * N + j] - c) + af[r];
                        mx = fmaxf(mx, t[u]);
                    }
                    if (binary) {
                        const float tt = fminf(fmaxf(t[0], -120.f), 120.f);
                        const float e = ex2_approx(-tt);          // exp(-z)
                        const float r1 = rcp_approx(1.f + e);     // p1 = sigmoid(z)
                        acc[1] = fmaf(pw, r1, acc[1]);
                        acc[0] = fmaf(pw, e * r1, acc[0]);        // p0 = 1 - p1 without cancellation
                    } else {
                        float den = 0.f;
                        if (ovr) {
                            const float h = fminf(mx, 0.f), eh = ex2_approx(h);
                            for (int u = 0; u < Rm; ++u) { t[u] = rcp_approx(eh + ex2_approx(h - t[u])); den += t[u]; }
                        } else {
                            for (int u = 0; u < Rm; ++u) { t[u] = ex2_approx(t[u] - mx); den += t[u]; }
                        }
                        const float inv = pw * rcp_approx(den);
                        for (int u = 0; u < Rm; ++u) acc[u] = fmaf(t[u], inv, acc[u]);
                    }
                }
            }
            if (binary) {
                sm.ys[s] = p.link == DKS_LINK_LOGIT ? log((double)acc[1] / (double)acc[0]) - p.linkfnull[1]
                                                    : (double)acc[1] - p.fnull[1];
            } else {
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
        }
        __syncthreads();
        const int nsolve = binary ? 1 : C;             // binary members: class 0 is the negation of class 1
        if constexpr (L1) {
            if (binary) block_moments_all<false>(q, G, pl, M, sm.ys, p.S_cap, 1, i, sm.A);
            else block_moments_all<true>(q, G, pl, M, sm.ys, p.S_cap, C, (size_t)i * C, sm.A);
            continue;
        }
        block_normal(pl, M, sm.A, i, p.status);
        for (int u = 0; u < nsolve; ++u) {
            const int c = binary ? 1 : u;
            __syncthreads();
            const double delta = p.dlink[(size_t)i * C + c];
            wls_build_rhs(pl.z, pl.w, sm.ys + (size_t)u * p.S_cap, S, M, delta, sm.rhs, threadIdx.x >> 5, blockDim.x >> 5);
            __syncthreads();
            if (tid == 0) wls_solve_write(sm.A, sm.rhs, M, delta, sm.vi, p.phi + (size_t)c * slab + (size_t)i * G, 1.0);
        }
        if (binary && tid == 0) write_class0_negation(p.phi + (size_t)i * G, p.phi + slab + (size_t)i * G, M, sm.vi);
    }
}

}  // namespace mix
}  // namespace dks
