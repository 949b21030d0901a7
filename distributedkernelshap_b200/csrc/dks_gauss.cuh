// Gaussian generative models on the device (DESIGN.md §5.0.23): QuadraticDiscriminantAnalysis, GaussianNB,
// GaussianMixture, BayesianGaussianMixture and EllipticEnvelope, read into K <= 8 component scores (GaussDev,
// dks_set_gaussian_model)
//   l_k(m) = c_k - gamma_k ||L_k^T (m - mu_k)||^2,   L_k: D x r_k,
// and a fixed head over them (DKS_GAUSS_HEAD_*: softmax, logsumexp, identity, the difference l_1 - l_0).
//
// For instance x, background row b_j and coalition z the masked row is m = b_j + sum_{g in z} (x - b_j)|_g.  With
// a = L_k^T (b_j - mu_k) and B_g = L_k^T x|_g - L_k^T b_j|_g,
//   q_kj(z) = ||a + sum_{g in z} B_g||^2 = alpha + sum_{g in z} beta_g + 2 sum_{g < h in z} Q_gh,
//   alpha = ||a||^2,  beta_g = 2 a^T B_g + ||B_g||^2,  Q_gh = B_g^T B_h.
// The fit step forms a, alpha and L_k^T b_j|_g (gauss_fit_tables_kernel); per instance the explain kernel forms L_k^T x|_g
// once, and per (j, k) the M x M table T[p][p] = beta_p, T[p][h] = 2 Q_ph (h < p).  A coalition then costs about |z|^2 / 2
// table reads per component, whatever the number of columns D or the rank r_k.
#pragma once

#include "dks_kernels.cuh"

namespace dks {
namespace gauss {

constexpr int THREADS = 256;      // = l1::MOM_THREADS: the l1 instantiation forms the moments with block_moments

// the head over the component scores l [K] into the outputs o
__device__ __forceinline__ void gauss_head(const GaussDev& gm, const double* l, double* o) {
    const int K = gm.K;
    if (gm.head == DKS_GAUSS_HEAD_IDENTITY) {
#pragma unroll
        for (int k = 0; k < DKS_GAUSS_MAX_K; ++k)
            if (k < K) o[k] = l[k];
        return;
    }
    if (gm.head == DKS_GAUSS_HEAD_DIFF) {
        o[0] = l[1] - l[0];
        return;
    }
    double mx = l[0];
#pragma unroll
    for (int k = 1; k < DKS_GAUSS_MAX_K; ++k)
        if (k < K) mx = fmax(mx, l[k]);
    double e[DKS_GAUSS_MAX_K], s = 0.0;
#pragma unroll
    for (int k = 0; k < DKS_GAUSS_MAX_K; ++k)
        if (k < K) {
            e[k] = exp(l[k] - mx);
            s += e[k];
        }
    if (gm.head == DKS_GAUSS_HEAD_LOGSUMEXP) {
        o[0] = mx + log(s);
        return;
    }
#pragma unroll
    for (int k = 0; k < DKS_GAUSS_MAX_K; ++k)
        if (k < K) o[k] = e[k] / s;
}

// f(X) [n][C] (dks_predict_host, the background at fit time) and, with dlink, link(f(x)) - link(fnull) for stage 1.  A row
// holding NaN or an infinity is reported as DKS_ERR_DOMAIN with the row (scikit-learn refuses it) and its outputs are NaN;
// a non-finite link(f(x)) is reported as DKS_ERR_NUMERIC with the instance.
__global__ void gauss_predict_kernel(const double* __restrict__ X, int n, int D, GaussDev gm, int C, int link,
                                     const double* __restrict__ linkfnull, double* __restrict__ out,
                                     double* __restrict__ dlink, int* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* x = X + (size_t)i * D;
    bool refused = false;
    for (int c = 0; c < D; ++c) refused |= !isfinite(x[c]);
    double o[DKS_GAUSS_MAX_K];
    if (refused) {
        for (int c = 0; c < C; ++c) o[c] = NAN;
        if (status) report_status(status, DKS_ERR_DOMAIN, i);
    } else {
        double l[DKS_GAUSS_MAX_K];
#pragma unroll
        for (int k = 0; k < DKS_GAUSS_MAX_K; ++k) {
            if (k >= gm.K) break;
            const double* mu = gm.mu + (size_t)k * D;
            double q = 0.0;
            for (int t = gm.r_off[k]; t < gm.r_off[k + 1]; ++t) {
                const double* Lt = gm.L + (size_t)t * D;
                double u = 0.0;
                for (int c = 0; c < D; ++c) u = fma(Lt[c], x[c] - mu[c], u);
                q = fma(u, u, q);
            }
            l[k] = fma(-gm.gamma[k], q, gm.c[k]);
        }
        gauss_head(gm, l, o);
    }
    predict_epilogue(o, C, i, link, linkfnull, out, dlink, status, refused);
}

// fit, threads over (j, k): a = L_k^T (bg_j - mu_k) into Abg[j][r_off[k] ..], alpha[j][k] = ||a||^2 and, per group g,
// Pbg[j][g][r_off[k] ..] = L_k^T bg_j|_g summed over the group's columns in CSR order (the explain kernel forms
// L_k^T x|_g in the same order, so B_g is exactly 0 where x equals bg_j on g)
__global__ void gauss_fit_tables_kernel(const double* __restrict__ bg, int N, int D, int G, const int* __restrict__ goff,
                                        const int* __restrict__ gcols, GaussDev gm, double* __restrict__ Abg,
                                        double* __restrict__ alpha, double* __restrict__ Pbg) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * gm.K) return;
    const int j = idx / gm.K, k = idx - j * gm.K, RT = gm.RT;
    const double* b = bg + (size_t)j * D;
    const double* mu = gm.mu + (size_t)k * D;
    double al = 0.0;
    for (int t = gm.r_off[k]; t < gm.r_off[k + 1]; ++t) {
        const double* Lt = gm.L + (size_t)t * D;
        double a = 0.0;
        for (int c = 0; c < D; ++c) a = fma(Lt[c], b[c] - mu[c], a);
        Abg[(size_t)j * RT + t] = a;
        al = fma(a, a, al);
        for (int g = 0; g < G; ++g) {
            double s = 0.0;
            for (int e = goff[g]; e < goff[g + 1]; ++e) s = fma(Lt[gcols[e]], b[gcols[e]], s);
            Pbg[((size_t)j * G + g) * RT + t] = s;
        }
    }
    alpha[(size_t)j * gm.K + k] = al;
}

// shared memory of explain_gauss_kernel: [C][S_cap] float64 sums / y, one region the background loop holds the tables of
// every component in ([K] alpha, then [K][G][G] T) and the solve the normal matrix [63 * 63] and rhs [64], and the varying
// groups [64]
__host__ __device__ inline size_t smem_bytes(int S_cap, int C, int G, int K) {
    const size_t tab = (size_t)K * (1 + (size_t)G * G), solve = 63 * 63 + 64;
    return sizeof(double) * ((size_t)C * S_cap + (tab > solve ? tab : solve)) + sizeof(int) * 64;
}

// One CTA per instance (grid-stride), any plan source (shared, per-instance, caller-supplied), up to 64 groups.  Per
// instance the CTA writes L_k^T x|_g of every varying group into its scratch gm.xp; per background row j (zero-weight rows
// skipped):
//   1. threads over (k, p, h <= p) form T_k[p][h] from B_p = xp[p] - Pbg[j][vi[p]] over the rank of component k;
//   2. threads over coalitions evaluate q_k = alpha_k + sum_{p in z} sum_{h in z, h <= p} T_k[p][h] (set bits in increasing
//      order), l_k = c_k - gamma_k q_k, the head, and add w_j times the outputs into the coalition's sums.
// Each coalition belongs to one thread throughout and every sum runs in a fixed order: the result does not depend on the
// grid.  Then y = link(ey) - link(fnull) for every output (each solved on its own) and the CUDA-core kernel's constrained
// WLS, or (L1) the moments of y for l1_lars_kernel.  A non-finite y or f(x) is reported as DKS_ERR_NUMERIC and nothing of
// the instance is written.
template <bool L1>
__global__ void __launch_bounds__(THREADS) explain_gauss_kernel(ExplainParams p, SimtL1 q, GaussDev gm,
                                                                const double* __restrict__ X, int D,
                                                                const int* __restrict__ goff,
                                                                const int* __restrict__ gcols) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x;
    const int N = p.N, G = p.G, C = p.C, K = gm.K, RT = gm.RT;
    double* acc = reinterpret_cast<double*>(smem_raw);          // [C][S_cap]
    double* region = acc + (size_t)C * p.S_cap;
    const size_t tab = (size_t)K * (1 + (size_t)G * G), solve = 63 * 63 + 64;
    double* A = region;                                         // [63 * 63] (solve)
    double* rhs = A + 63 * 63;                                  // [64]
    double* al = region;                                        // [K] (background loop)
    double* T = al + K;                                         // [K][M][M]
    int* vi = reinterpret_cast<int*>(region + (tab > solve ? tab : solve));   // [64]
    double* xp = gm.xp + (size_t)blockIdx.x * G * RT;           // [M][RT] this CTA's scratch
    const size_t slab = (size_t)p.n * G;

    const int ninst = dks_inst_count(p);
    for (int qi = blockIdx.x; qi < ninst; qi += gridDim.x) {
        const int i = dks_inst_at(p, qi);
        const int M = p.Mcnt[i];
        const uint64_t vm = p.vmask[i];
        __syncthreads();  // previous instance done with shared memory and the scratch
        zero_phi_rows(p, i);
        bool fx_bad = false;                                    // stage 1 reported a refused row or a non-finite link(f(x))
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
        const uint64_t* zp = pl.z;
        varying_positions(vm, G, vi);
        for (int idx = tid; idx < C * S; idx += blockDim.x) acc[(size_t)(idx / S) * p.S_cap + idx % S] = 0.0;
        __syncthreads();

        // L_k^T x|_g of every varying group, in the group's CSR order
        const double* x = X + (size_t)i * D;
        for (int idx = tid; idx < M * RT; idx += blockDim.x) {
            const int pp = idx / RT, t = idx - pp * RT, g = vi[pp];
            const double* Lt = gm.L + (size_t)t * D;
            double s = 0.0;
            for (int e = goff[g]; e < goff[g + 1]; ++e) s = fma(Lt[gcols[e]], x[gcols[e]], s);
            xp[idx] = s;
        }
        __syncthreads();

        for (int j = 0; j < N; ++j) {
            const double wj = p.wbg[j];
            if (wj == 0.0) continue;                            // block-uniform
            const double* aj = gm.Abg + (size_t)j * RT;
            const double* pj = gm.Pbg + (size_t)j * G * RT;
            for (int k = tid; k < K; k += blockDim.x) al[k] = gm.alpha[(size_t)j * K + k];
            for (int idx = tid; idx < K * M * M; idx += blockDim.x) {
                const int k = idx / (M * M), rem = idx - k * M * M, pp = rem / M, h = rem - pp * M;
                if (h > pp) continue;
                const double* xa = xp + (size_t)pp * RT;
                const double* pa = pj + (size_t)vi[pp] * RT;
                double s = 0.0;
                if (h == pp) {
                    for (int t = gm.r_off[k]; t < gm.r_off[k + 1]; ++t) {
                        const double B = xa[t] - pa[t];
                        s = fma(B, fma(2.0, aj[t], B), s);
                    }
                } else {
                    const double* xb = xp + (size_t)h * RT;
                    const double* pb = pj + (size_t)vi[h] * RT;
                    for (int t = gm.r_off[k]; t < gm.r_off[k + 1]; ++t) s = fma(xa[t] - pa[t], xb[t] - pb[t], s);
                    s *= 2.0;
                }
                T[idx] = s;
            }
            __syncthreads();
            for (int s = tid; s < S; s += blockDim.x) {
                const uint64_t z = zp[s];
                double l[DKS_GAUSS_MAX_K], o[DKS_GAUSS_MAX_K];
#pragma unroll
                for (int k = 0; k < DKS_GAUSS_MAX_K; ++k) {
                    if (k >= K) break;
                    const double* Tk = T + (size_t)k * M * M;
                    double qk = al[k];
                    for (uint64_t zz = z; zz; zz &= zz - 1) {
                        const int pp = __ffsll((long long)zz) - 1;
                        const double* row = Tk + (size_t)pp * M;
                        double r = 0.0;
                        for (uint64_t w = z & ((2ull << pp) - 1); w; w &= w - 1) r += row[__ffsll((long long)w) - 1];
                        qk += r;
                    }
                    l[k] = fma(-gm.gamma[k], qk, gm.c[k]);
                }
                gauss_head(gm, l, o);
                for (int c = 0; c < C; ++c) acc[(size_t)c * p.S_cap + s] = fma(wj, o[c], acc[(size_t)c * p.S_cap + s]);
            }
            __syncthreads();
        }

        // y = link(ey) - link(fnull) of every output, written over the sums
        int bad = 0;
        for (int s = tid; s < S; s += blockDim.x)
            for (int c = 0; c < C; ++c) {
                const double e = acc[(size_t)c * p.S_cap + s];
                const double y = p.link == DKS_LINK_LOGIT ? log(e / (1.0 - e)) - p.linkfnull[c] : e - p.fnull[c];
                bad |= !isfinite(y);
                acc[(size_t)c * p.S_cap + s] = y;
            }
        if (__syncthreads_or(bad)) {
            if (tid == 0) report_status(p.status, DKS_ERR_NUMERIC, i);
            if (L1) moments_skip(q, G, M, C, (size_t)i * C);
            continue;
        }
        if constexpr (L1) {
            block_moments_all<true>(q, G, pl, M, acc, p.S_cap, C, (size_t)i * C, A);
            continue;
        }
        block_normal(pl, M, A, i, p.status);
        block_solve(p, i, pl, M, acc, p.S_cap, C, false, A, rhs, vi);
    }
}

}  // namespace gauss
}  // namespace dks
