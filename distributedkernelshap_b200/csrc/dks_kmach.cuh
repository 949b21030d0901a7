// Kernel machines on the device (DESIGN.md §5.0.12): scikit-learn SVC / NuSVC decision functions, SVR / NuSVR, KernelRidge and
// sigmoid-calibrated SVCs, read into support vectors in raw feature space (KmDev, dks_set_kernel_machine).  KernelSHAP on a
// kernel machine needs the real masked forward pass of every (coalition s, background row j): x's value for the groups of s
// that vary, bg_j's for the rest.
//
// The reduction that makes it cheap: every kernel is phi(t) of a statistic that adds up over columns, so for support vector v
//   t(s, j, v) = T[j][v] + sum_{p in s} Delta_j[p][v],   T[j][v] = sum_c h(bg_j,c, v_c)  (fit time),
//   Delta_j[p][v] = sum_{c in group p} h(x_c, v_c) - h(bg_j,c, v_c)                  (per instance and row).
// Per (j, tile of support vectors) the Delta go into nibble tables (16 partial sums per 4 varying groups), so one masked
// forward pass costs ceil(M / 4) table reads and one phi per support vector, whatever the number of columns.
#pragma once

#include "dks_kernels.cuh"

namespace dks {
namespace kmach {

constexpr int THREADS = 256;      // = l1::MOM_THREADS: the l1 instantiation forms the moments with block_moments
constexpr int TILE = 32;          // support vectors per shared-memory tile

// per-column term h(m, v) of the kernel's statistic t, for column weight w and origin o
__device__ __forceinline__ double km_term(int kernel, double m, double v, double w, double o) {
    if (kernel == DKS_KM_KERNEL_RBF) { const double d = m - v; return w * d * d; }
    if (kernel == DKS_KM_KERNEL_LAPLACIAN) return w * fabs(m - v);
    return w * (m - o) * (v - o);
}

// K = phi(t): additive statistic first, then one phi (no product of exponentials: nothing overflows while the kernel
// value stays in [0, 1]; a t whose exp underflows gives 0, as scikit-learn's kernel does)
__device__ __forceinline__ double km_phi(const KmDev& k, double t, double gamma) {
    if (k.kernel == DKS_KM_KERNEL_RBF || k.kernel == DKS_KM_KERNEL_LAPLACIAN) return exp(-gamma * t);
    const double u = fma(gamma, t, k.coef0);
    return k.kernel == DKS_KM_KERNEL_POLY ? pow(u, k.degree) : tanh(u);
}

// [p0, p1] contributions of one calibrated member, p1 = expit(-(a f + b)), neither half formed by cancellation
__device__ __forceinline__ void cal_member(double z, double* p0, double* p1) {
    const double e = exp(-fabs(z));
    const double big = 1.0 / (1.0 + e), small = e / (1.0 + e);
    *p1 = z >= 0 ? small : big;
    *p0 = z >= 0 ? big : small;
}

// outputs o[C] of one row: member scores summed over support vectors in order, then the head
__device__ inline void km_outputs(const KmDev& k, const double* __restrict__ x, int D, double* o) {
    if (k.head == DKS_KM_HEAD_CALIBRATED) { o[0] = 0.0; o[1] = 0.0; }
    for (int m = 0; m < k.K; ++m) {
        double f[DKS_KM_MAX_R];
        for (int q = 0; q < k.R; ++q) f[q] = 0.0;
        const double* w = k.colw + (size_t)m * D;
        const double* org = k.colo + (size_t)m * D;
        for (int v = k.sv_off[m]; v < k.sv_off[m + 1]; ++v) {
            const double* sv = k.sv + (size_t)v * D;
            double t = 0.0;
            for (int c = 0; c < D; ++c) t += km_term(k.kernel, x[c], sv[c], w[c], org[c]);
            const double kv = km_phi(k, t, k.gamma[m]);
            for (int q = 0; q < k.R; ++q) f[q] = fma(k.dual[(size_t)v * k.R + q], kv, f[q]);
        }
        if (k.head == DKS_KM_HEAD_CALIBRATED) {
            double p0, p1;
            cal_member(fma(k.cal_a[m], f[0] + k.icpt[m], k.cal_b[m]), &p0, &p1);
            o[0] = fma(k.pi[m], p0, o[0]);
            o[1] = fma(k.pi[m], p1, o[1]);
        } else {
            for (int q = 0; q < k.R; ++q) o[q] = f[q] + k.icpt[q];
        }
    }
}

// f(X) [n][C] (dks_predict_host, the background at fit time) and, with dlink, link(f(x)) - link(fnull) for stage 1.  A row
// holding NaN is reported as DKS_ERR_DOMAIN with the row (scikit-learn refuses it) and its outputs are NaN; a non-finite
// link(f(x)) is reported as DKS_ERR_NUMERIC with the instance.
__global__ void km_predict_kernel(const double* __restrict__ X, int n, int D, KmDev k, int C, int link,
                                  const double* __restrict__ linkfnull, double* __restrict__ out, double* __restrict__ dlink,
                                  int* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* x = X + (size_t)i * D;
    bool nan = false;
    for (int c = 0; c < D; ++c) nan |= isnan(x[c]);
    double o[DKS_KM_MAX_R];
    if (nan) {
        for (int c = 0; c < C; ++c) o[c] = NAN;
        if (status) report_status(status, DKS_ERR_DOMAIN, i);
    } else {
        km_outputs(k, x, D, o);
    }
    predict_epilogue(o, C, i, link, linkfnull, out, dlink, status, nan);
}

// fit: T[j][v] = sum_c h(bg_j,c, v_c) with the weights and origins of v's member, columns in order
__global__ void km_fit_table_kernel(const double* __restrict__ bg, int N, int D, KmDev k, double* __restrict__ Tbg) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * k.n_sv) return;
    const int j = (int)(idx / k.n_sv), v = (int)(idx - (long long)j * k.n_sv);
    int m = 0;
    while (v >= k.sv_off[m + 1]) ++m;
    const double* w = k.colw + (size_t)m * D;
    const double* org = k.colo + (size_t)m * D;
    const double* sv = k.sv + (size_t)v * D;
    const double* b = bg + (size_t)j * D;
    double t = 0.0;
    for (int c = 0; c < D; ++c) t += km_term(k.kernel, b[c], sv[c], w[c], org[c]);
    Tbg[idx] = t;
}

// doubles of the per-tile tables: T_j [TILE], dual [TILE][R], Delta [G][TILE], nibble tables [ceil(G/4)][TILE][16]
__host__ __device__ inline size_t tile_doubles(int R, int G) {
    return (size_t)TILE * (1 + R + G + 16 * ((G + 3) / 4));
}

// shared memory of explain_kmach_kernel: [C][S_cap] float64 sums / y, one member's scores [S_cap] (calibrated head), then
// one region the background loop holds a tile's tables in and the solve the normal matrix [63 * 63] and rhs [64], and the
// varying groups [64]
__host__ __device__ inline size_t smem_bytes(int S_cap, int C, int R, int G, bool cal) {
    const size_t tab = tile_doubles(R, G), solve = 63 * 63 + 64;
    return sizeof(double) * ((size_t)(C + (cal ? 1 : 0)) * S_cap + (tab > solve ? tab : solve)) + sizeof(int) * 64;
}

// One CTA per instance (grid-stride), any plan source (shared, per-instance, caller-supplied), up to 64 groups.  Background
// rows are the outer loop (zero-weight rows skipped); per row j, member and tile of TILE support vectors:
//   1. threads over (varying position p, v) form Delta_j[p][v] from the group's columns, then the nibble tables
//      tb[q][v][pat] = sum of Delta over the set bits of pat (positions 4q .. 4q + 3, in order);
//   2. threads over coalitions read t = T[j][v] + sum_q tb[q][v][z's nibble q] per support vector and add dual[v] phi(t)
//      to the coalition's score: identity head straight into the sums (times w_j), calibrated head into the member's score,
//      whose expit goes into the sums times w_j pi_k once the member's support vectors are done.
// Each coalition belongs to one thread throughout and every sum runs in a fixed order: the result does not depend on the
// grid.  Then y = link(ey) - link(fnull) per solved output (calibrated head: class 1, class 0 its negation), and the CUDA-core
// kernel's constrained WLS, or (L1) the moments of y for l1_lars_kernel.  A non-finite y or f(x) is reported as
// DKS_ERR_NUMERIC and nothing of the instance is written.
// ACC (a soft-voting ensemble's member): the sums of every output go into ea.ey instead (ens_accumulate); instances
// with M <= 1 or a refused f(x) are left to explain_ensemble_tail_kernel.
// ROWS (a stacking ensemble's member, with ACC): per background row of the chunk the sums are formed at unit weight from
// zero -- each coalition's outputs -- and go to er.ws (rows_store), each thread storing the coalitions it owns; nothing is
// summed over the background.
template <bool L1, bool ACC = false, bool ROWS = false>
__global__ void __launch_bounds__(THREADS) explain_kmach_kernel(ExplainParams p, SimtL1 q, KmDev k,
                                                                const double* __restrict__ X, const double* __restrict__ bg,
                                                                int D, const int* __restrict__ goff,
                                                                const int* __restrict__ gcols, EnsAcc ea, EnsRows er) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x;
    const int N = p.N, G = p.G, C = p.C, R = k.R;
    const bool cal = k.head == DKS_KM_HEAD_CALIBRATED;
    double* acc = reinterpret_cast<double*>(smem_raw);          // [C][S_cap]
    double* fsc = acc + (size_t)C * p.S_cap;                    // [S_cap] one member's scores (calibrated head)
    double* region = fsc + (cal ? p.S_cap : 0);
    const size_t tab = tile_doubles(R, G), solve = 63 * 63 + 64;
    double* A = region;                                         // [63 * 63] (solve)
    double* rhs = A + 63 * 63;                                  // [64]
    double* tj = region;                                        // [TILE] (background loop)
    double* du = tj + TILE;                                     // [TILE][R]
    double* dl = du + TILE * R;                                 // [G][TILE]
    double* tb = dl + (size_t)G * TILE;                         // [ceil(G/4)][TILE][16]
    int* vi = reinterpret_cast<int*>(region + (tab > solve ? tab : solve));   // [64]
    const size_t slab = (size_t)p.n * G;
    const int nsolve = cal ? 1 : C;                             // calibrated: class 0 is the negation of class 1

    const int ninst = dks_inst_count(p);
    for (int qi = blockIdx.x; qi < ninst; qi += gridDim.x) {
        const int i = dks_inst_at(p, qi);
        const int M = p.Mcnt[i];
        const uint64_t vm = p.vmask[i];
        __syncthreads();  // previous instance done with shared memory
        if constexpr (!ACC) zero_phi_rows(p, i);
        bool fx_bad = false;                                    // stage 1 reported a NaN row or a non-finite link(f(x))
        if constexpr (ROWS) fx_bad = rows_fx_bad(er, i);
        else for (int c = 0; c < C; ++c) fx_bad |= !isfinite(p.dlink[(size_t)i * C + c]);
        if (M == 0) continue;
        if (M == 1) {
            // the one varying group takes link(f(x)) - link(fnull); calibrated: class 0 is the negation of class 1, as below
            if (!ACC && tid < C && !fx_bad) {
                const double v = p.dlink[(size_t)i * C + (cal ? 1 : tid)];
                p.phi[(size_t)tid * slab + (size_t)i * G + (__ffsll((long long)vm) - 1)] =
                    (cal && tid == 0) ? ((v == 0.0) ? 0.0 : -v) : v;
            }
            continue;
        }
        InstPlan pl;
        if (!inst_plan(p, i, M, pl)) continue;
        if (fx_bad) {
            if (L1) moments_skip(q, G, M, nsolve, (size_t)i * nsolve);
            continue;
        }
        const int S = pl.S;
        const uint64_t* zp = pl.z;
        varying_positions(vm, G, vi);
        for (int idx = tid; idx < C * S; idx += blockDim.x) acc[(size_t)(idx / S) * p.S_cap + idx % S] = 0.0;
        if (cal) for (int s = tid; s < S; s += blockDim.x) fsc[s] = 0.0;
        __syncthreads();

        const double* x = X + (size_t)i * D;
        const int nib = (M + 3) >> 2;
        for (int j = ROWS ? er.j0 : 0; j < (ROWS ? er.j1 : N); ++j) {
            const double wb = p.wbg[j];
            if (wb == 0.0) continue;                            // block-uniform
            const double wj = ROWS ? 1.0 : wb;
            const double* b = bg + (size_t)j * D;
            if constexpr (ROWS)
                for (int s = tid; s < S; s += blockDim.x)
                    for (int c = 0; c < C; ++c) acc[(size_t)c * p.S_cap + s] = 0.0;
            if (!cal)
                for (int s = tid; s < S; s += blockDim.x)
                    for (int c = 0; c < C; ++c) acc[(size_t)c * p.S_cap + s] = fma(wj, k.icpt[c], acc[(size_t)c * p.S_cap + s]);
            for (int m = 0; m < k.K; ++m) {
                const double gm = k.gamma[m];
                const double* w = k.colw + (size_t)m * D;
                const double* org = k.colo + (size_t)m * D;
                for (int v0 = k.sv_off[m]; v0 < k.sv_off[m + 1]; v0 += TILE) {
                    const int nv = min(TILE, k.sv_off[m + 1] - v0);
                    for (int idx = tid; idx < nv; idx += blockDim.x) tj[idx] = k.Tbg[(size_t)j * k.n_sv + v0 + idx];
                    for (int idx = tid; idx < nv * R; idx += blockDim.x) du[idx] = k.dual[(size_t)v0 * R + idx];
                    for (int idx = tid; idx < M * nv; idx += blockDim.x) {
                        const int pp = idx / nv, v = idx - pp * nv, g = vi[pp];
                        const double* sv = k.sv + (size_t)(v0 + v) * D;
                        double d = 0.0;
                        for (int e = goff[g]; e < goff[g + 1]; ++e) {
                            const int c = gcols[e];
                            d += km_term(k.kernel, x[c], sv[c], w[c], org[c]) - km_term(k.kernel, b[c], sv[c], w[c], org[c]);
                        }
                        dl[(size_t)pp * TILE + v] = d;
                    }
                    __syncthreads();
                    for (int idx = tid; idx < nib * nv * 16; idx += blockDim.x) {
                        const int qn = idx / (nv * 16), rem = idx - qn * nv * 16, v = rem >> 4, pat = rem & 15;
                        double t = 0.0;
                        for (int bit = 0; bit < 4; ++bit)
                            if (((pat >> bit) & 1) && 4 * qn + bit < M) t += dl[(size_t)(4 * qn + bit) * TILE + v];
                        tb[((size_t)qn * TILE + v) * 16 + pat] = t;
                    }
                    __syncthreads();
                    for (int s = tid; s < S; s += blockDim.x) {
                        const uint64_t z = zp[s];
                        double f[DKS_KM_MAX_R];
#pragma unroll
                        for (int r = 0; r < DKS_KM_MAX_R; ++r) f[r] = 0.0;
                        for (int v = 0; v < nv; ++v) {
                            double t = tj[v];
                            for (int qn = 0; qn < nib; ++qn) t += tb[((size_t)qn * TILE + v) * 16 + ((z >> (4 * qn)) & 15)];
                            const double kv = km_phi(k, t, gm);
#pragma unroll
                            for (int r = 0; r < DKS_KM_MAX_R; ++r)
                                if (r < R) f[r] = fma(du[v * R + r], kv, f[r]);
                        }
                        if (cal) {
                            fsc[s] += f[0];
                        } else {
#pragma unroll
                            for (int r = 0; r < DKS_KM_MAX_R; ++r)
                                if (r < C) acc[(size_t)r * p.S_cap + s] = fma(wj, f[r], acc[(size_t)r * p.S_cap + s]);
                        }
                    }
                    __syncthreads();
                }
                if (cal) {
                    // the member is complete: its calibrated probabilities, times w_j pi_k, into the sums
                    const double wk = wj * k.pi[m];
                    for (int s = tid; s < S; s += blockDim.x) {
                        double p0, p1;
                        cal_member(fma(k.cal_a[m], fsc[s] + k.icpt[m], k.cal_b[m]), &p0, &p1);
                        acc[s] = fma(wk, p0, acc[s]);
                        acc[(size_t)p.S_cap + s] = fma(wk, p1, acc[(size_t)p.S_cap + s]);
                        fsc[s] = 0.0;
                    }
                }
            }
            if constexpr (ROWS)
                for (int s = tid; s < S; s += blockDim.x) {
                    double o[DKS_KM_MAX_R];
                    for (int c = 0; c < C; ++c) o[c] = acc[(size_t)c * p.S_cap + s];
                    rows_store<0>(er, p.S_cap, i, j, s, o);
                }
        }
        __syncthreads();
        if constexpr (ROWS) continue;
        if constexpr (ACC) {
            ens_accumulate(ea, p, i, S, acc);
            continue;
        }

        // y = link(ey) - link(fnull) per solved output, written over the sums (row u of acc); calibrated head: the logit's
        // 1 - ey is the sum of class 0 (no cancellation)
        int bad = 0;
        for (int s = tid; s < S; s += blockDim.x) {
            double y[DKS_KM_MAX_R];
            for (int u = 0; u < nsolve; ++u) {
                const int c = cal ? 1 : u;
                const double e = acc[(size_t)c * p.S_cap + s];
                if (p.link == DKS_LINK_LOGIT) {
                    const double rest = cal ? acc[s] : 1.0 - e;
                    y[u] = log(e / rest) - p.linkfnull[c];
                } else {
                    y[u] = e - p.fnull[c];
                }
                bad |= !isfinite(y[u]);
            }
            for (int u = 0; u < nsolve; ++u) acc[(size_t)u * p.S_cap + s] = y[u];
        }
        if (__syncthreads_or(bad)) {
            if (tid == 0) report_status(p.status, DKS_ERR_NUMERIC, i);
            if (L1) moments_skip(q, G, M, nsolve, (size_t)i * nsolve);
            continue;
        }
        if constexpr (L1) {
            block_moments_all<true>(q, G, pl, M, acc, p.S_cap, nsolve, (size_t)i * nsolve, A);
            continue;
        }
        block_normal(pl, M, A, i, p.status);
        block_solve(p, i, pl, M, acc, p.S_cap, nsolve, cal, A, rhs, vi);
    }
}

}  // namespace kmach
}  // namespace dks
