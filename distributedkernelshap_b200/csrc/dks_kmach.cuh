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
// The program kernel (DKS_KM_KERNEL_PROGRAM, KmProg, DESIGN.md §5.0.21) carries L <= 4 such statistics, each with its own
// column weights and origins, and evaluates a postfix expression of them per support vector: L ceil(M / 4) table reads.
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

// per-column term of a program statistic (DKS_KM_STAT_*): the rbf and dot-product terms above
__device__ __forceinline__ double km_stat_term(int kind, double m, double v, double w, double o) {
    return km_term(kind == DKS_KM_STAT_SQDIST ? DKS_KM_KERNEL_RBF : DKS_KM_KERNEL_POLY, m, v, w, o);
}

// K(x, v) of the program kernel from the statistics t[L].  The operand stack is four registers shifted on every push and
// pop (indices known at compile time: nothing goes to local memory); t is read through unrolled selects for the same reason.
// A squared distance formed from tables can come out a rounding below zero: the square roots clamp it.
__device__ __forceinline__ double km_program(const KmProg& g, const double* t) {
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    for (int pc = 0; pc < g.n; ++pc) {
        const int op = g.op[pc];
        const double a = g.a[pc];
        if (op == DKS_KM_OP_ADD || op == DKS_KM_OP_MUL) {
            s0 = op == DKS_KM_OP_ADD ? s1 + s0 : s1 * s0;
            s1 = s2; s2 = s3;
            continue;
        }
        if (op == DKS_KM_OP_POW) { s0 = pow(s0, a); continue; }
        if (op == DKS_KM_OP_ADDC) { s0 = s0 + a; continue; }
        if (op == DKS_KM_OP_MULC) { s0 = s0 * a; continue; }
        const int l = g.arg[pc];
        double tl = t[0];
#pragma unroll
        for (int q = 1; q < DKS_KM_MAX_STATS; ++q)
            if (l == q) tl = t[q];
        double v;
        if (op == DKS_KM_OP_CONST) {
            v = a;
        } else if (op == DKS_KM_OP_STAT) {
            v = tl;
        } else if (op == DKS_KM_OP_EXP) {
            v = exp(-a * tl);
        } else if (op == DKS_KM_OP_RQ) {
            v = pow(1.0 + tl, a);
        } else {
            const double r = sqrt(fmax(tl, 0.0));
            if (op == DKS_KM_OP_MATERN05) {
                v = exp(-r);
            } else if (op == DKS_KM_OP_MATERN15) {
                const double k = r * 1.7320508075688772;
                v = (1.0 + k) * exp(-k);
            } else if (op == DKS_KM_OP_MATERN25) {
                const double k = r * 2.23606797749979;
                v = (1.0 + k + k * k / 3.0) * exp(-k);
            } else {
                const double sn = sin(3.141592653589793 * r / a) / g.b[pc];
                v = exp(-2.0 * (sn * sn));
            }
        }
        s3 = s2; s2 = s1; s1 = s0; s0 = v;
    }
    return s0;
}

// outputs o[R] of one row under the program kernel (identity head, one member): t_l per statistic, columns in order
__device__ inline void km_prog_outputs(const KmDev& k, const KmProg& g, const double* __restrict__ x, int D, double* o) {
    double f[DKS_KM_MAX_R];
    for (int q = 0; q < k.R; ++q) f[q] = 0.0;
    for (int v = 0; v < k.n_sv; ++v) {
        const double* sv = k.sv + (size_t)v * D;
        double t[DKS_KM_MAX_STATS];
#pragma unroll
        for (int l = 0; l < DKS_KM_MAX_STATS; ++l) {
            t[l] = 0.0;
            if (l < g.L) {
                const double* w = k.colw + (size_t)l * D;
                const double* org = k.colo + (size_t)l * D;
                for (int c = 0; c < D; ++c) t[l] += km_stat_term(g.kind[l], x[c], sv[c], w[c], org[c]);
            }
        }
        const double kv = km_program(g, t);
        for (int q = 0; q < k.R; ++q) f[q] = fma(k.dual[(size_t)v * k.R + q], kv, f[q]);
    }
    for (int q = 0; q < k.R; ++q) o[q] = f[q] + k.icpt[q];
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

// km_predict_kernel under the program kernel
__global__ void km_prog_predict_kernel(const double* __restrict__ X, int n, int D, KmDev k, KmProg g, int C, int link,
                                       const double* __restrict__ linkfnull, double* __restrict__ out,
                                       double* __restrict__ dlink, int* __restrict__ status) {
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
        km_prog_outputs(k, g, x, D, o);
    }
    predict_epilogue(o, C, i, link, linkfnull, out, dlink, status, nan);
}

// fit under the program kernel: T[j][v][l] = sum_c h_l(bg_j,c, v_c), columns in order
__global__ void km_prog_fit_table_kernel(const double* __restrict__ bg, int N, int D, KmDev k, KmProg g,
                                         double* __restrict__ Tbg) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * k.n_sv * g.L) return;
    const long long jv = idx / g.L;
    const int l = (int)(idx - jv * g.L);
    const int j = (int)(jv / k.n_sv), v = (int)(jv - (long long)j * k.n_sv);
    const double* w = k.colw + (size_t)l * D;
    const double* org = k.colo + (size_t)l * D;
    const double* sv = k.sv + (size_t)v * D;
    const double* b = bg + (size_t)j * D;
    double t = 0.0;
    for (int c = 0; c < D; ++c) t += km_stat_term(g.kind[l], b[c], sv[c], w[c], org[c]);
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
// PROG (the program kernel, identity head): a tile holds TILE / L support vectors, and its T, Delta and nibble-table columns
// are (statistic l, support vector v) at l nv + v, so the tables of L statistics fill the shared memory of one; per
// coalition and support vector the L statistics are read from the tables and the expression gives the kernel value.
template <bool L1, bool ACC = false, bool ROWS = false, bool PROG = false>
__global__ void __launch_bounds__(THREADS) explain_kmach_kernel(ExplainParams p, SimtL1 q, KmDev k,
                                                                const double* __restrict__ X, const double* __restrict__ bg,
                                                                int D, const int* __restrict__ goff,
                                                                const int* __restrict__ gcols, EnsAcc ea, EnsRows er,
                                                                KmProg g) {
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
                const int tw = PROG ? TILE / g.L : TILE;        // support vectors per tile
                for (int v0 = k.sv_off[m]; v0 < k.sv_off[m + 1]; v0 += tw) {
                    const int nv = min(tw, k.sv_off[m + 1] - v0);
                    const int ncol = PROG ? g.L * nv : nv;      // table columns
                    if constexpr (PROG) {
                        for (int idx = tid; idx < ncol; idx += blockDim.x) {
                            const int l = idx / nv, v = idx - l * nv;
                            tj[idx] = k.Tbg[((size_t)j * k.n_sv + v0 + v) * g.L + l];
                        }
                    } else {
                        for (int idx = tid; idx < nv; idx += blockDim.x) tj[idx] = k.Tbg[(size_t)j * k.n_sv + v0 + idx];
                    }
                    for (int idx = tid; idx < nv * R; idx += blockDim.x) du[idx] = k.dual[(size_t)v0 * R + idx];
                    if constexpr (PROG) {
                        for (int idx = tid; idx < M * ncol; idx += blockDim.x) {
                            const int pp = idx / ncol, col = idx - pp * ncol, l = col / nv, v = col - l * nv, g0 = vi[pp];
                            const double* sv = k.sv + (size_t)(v0 + v) * D;
                            const double* wl = k.colw + (size_t)l * D;
                            const double* ol = k.colo + (size_t)l * D;
                            const int kind = g.kind[l];
                            double d = 0.0;
                            for (int e = goff[g0]; e < goff[g0 + 1]; ++e) {
                                const int c = gcols[e];
                                d += km_stat_term(kind, x[c], sv[c], wl[c], ol[c]) - km_stat_term(kind, b[c], sv[c], wl[c], ol[c]);
                            }
                            dl[(size_t)pp * TILE + col] = d;
                        }
                    } else
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
                    for (int idx = tid; idx < nib * ncol * 16; idx += blockDim.x) {
                        const int qn = idx / (ncol * 16), rem = idx - qn * ncol * 16, v = rem >> 4, pat = rem & 15;
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
                        if constexpr (PROG) {
                            for (int v = 0; v < nv; ++v) {
                                double t[DKS_KM_MAX_STATS];
#pragma unroll
                                for (int l = 0; l < DKS_KM_MAX_STATS; ++l) {
                                    t[l] = 0.0;
                                    if (l < g.L) {
                                        const int col = l * nv + v;
                                        t[l] = tj[col];
                                        for (int qn = 0; qn < nib; ++qn)
                                            t[l] += tb[((size_t)qn * TILE + col) * 16 + ((z >> (4 * qn)) & 15)];
                                    }
                                }
                                const double kv = km_program(g, t);
#pragma unroll
                                for (int r = 0; r < DKS_KM_MAX_R; ++r)
                                    if (r < R) f[r] = fma(du[v * R + r], kv, f[r]);
                            }
                        } else
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

// ---- multi-class SVMs: the one-vs-one head (DKS_KM_HEAD_OVO, KmOvo, DESIGN.md §5.0.22) ----------------------------------
// A member's pair scores live in 28 registers d[] laid out for 8 classes (slot of pair (a, b) below); a multi-class SVM
// with fewer classes leaves the slots of b >= classes at zero.  Every index into d, and into the per-class partials pt, is a
// compile-time constant of an unrolled loop: nothing goes to local memory.

constexpr int OVO_C = DKS_KM_OVO_MAX_CLASSES;
constexpr int OVO_SLOTS = OVO_C * (OVO_C - 1) / 2;

__host__ __device__ constexpr int ovo_slot(int a, int b) { return a * (2 * OVO_C - a - 1) / 2 + (b - a - 1); }

// the partials pt[r] = sum_v dual[v][r] K(x, v) over support vectors of class c into the pair scores: dual row r of class c
// belongs to pair (c, r + 1) for r >= c and to pair (r, c) for r < c (scikit-learn's dual_coef_ layout)
__device__ __forceinline__ void ovo_scatter(int c, const double* pt, double* d) {
#pragma unroll
    for (int a = 0; a < OVO_C; ++a)
#pragma unroll
        for (int b = a + 1; b < OVO_C; ++b) {
            if (c == a) d[ovo_slot(a, b)] += pt[b - 1];
            else if (c == b) d[ovo_slot(a, b)] += pt[a];
        }
}

// member m's head on its pair scores d (intercepts not yet added), handing each output to emit(row, value):
// DKS_KM_OVO_DECISION dec_k = d + intercept for row k = 0 .. P - 1 in scikit-learn's pair order; DKS_KM_OVO_PROBA the
// calibrated probabilities of the ovr-vote decision function f_c = votes_c + conf_c / (3 (|conf_c| + 1)) for row c (dec >= 0
// votes for the first class of the pair, as libsvm decides it; conf summed in the pair order, as scikit-learn sums it),
// e_c = expit(-(a_c f_c + b_c)), normalised by their sum (uniform 1 / classes for a zero sum), (1, 1 + 1e-5] clipped to 1
template <typename Emit>
__device__ __forceinline__ void ovo_head(const KmOvo& ov, int m, const double* d, Emit&& emit) {
    const int nc = ov.classes;
    const double* ic = ov.icpt + (size_t)m * ov.P;
    double votes[OVO_C], conf[OVO_C];
#pragma unroll
    for (int c = 0; c < OVO_C; ++c) { votes[c] = 0.0; conf[c] = 0.0; }
    int k = 0;
#pragma unroll
    for (int a = 0; a < OVO_C; ++a)
#pragma unroll
        for (int b = a + 1; b < OVO_C; ++b)
            if (b < nc) {
                const double dec = d[ovo_slot(a, b)] + ic[k];
                if (ov.mode == DKS_KM_OVO_DECISION) {
                    emit(k, dec);
                } else {
                    if (dec >= 0.0) votes[a] += 1.0; else votes[b] += 1.0;
                    conf[a] += dec;
                    conf[b] -= dec;
                }
                ++k;
            }
    if (ov.mode == DKS_KM_OVO_DECISION) return;
    const double* ca = ov.cal_a + (size_t)m * nc;
    const double* cb = ov.cal_b + (size_t)m * nc;
    double e[OVO_C], sum = 0.0;
#pragma unroll
    for (int c = 0; c < OVO_C; ++c) {
        e[c] = 0.0;
        if (c < nc) {
            const double f = votes[c] + conf[c] / (3.0 * (fabs(conf[c]) + 1.0));
            double p0;
            cal_member(fma(ca[c], f, cb[c]), &p0, &e[c]);
            sum += e[c];
        }
    }
#pragma unroll
    for (int c = 0; c < OVO_C; ++c)
        if (c < nc) {
            double pc = sum != 0.0 ? e[c] / sum : 1.0 / nc;
            if (pc > 1.0 && pc <= 1.0 + 1e-5) pc = 1.0;
            emit(c, pc);
        }
}

// outputs o[C] of one row under the one-vs-one head: per member and class the partials over the class's support vectors
// in order, then the head; members weighted by pi
__device__ inline void km_ovo_outputs(const KmDev& k, const KmOvo& ov, const double* __restrict__ x, int D, double* o) {
    const int C = ov.mode == DKS_KM_OVO_DECISION ? ov.P : ov.classes;
    for (int c = 0; c < C; ++c) o[c] = 0.0;
    for (int m = 0; m < k.K; ++m) {
        double d[OVO_SLOTS];
#pragma unroll
        for (int e = 0; e < OVO_SLOTS; ++e) d[e] = 0.0;
        const double* w = k.colw + (size_t)m * D;
        const double* org = k.colo + (size_t)m * D;
        const int* co = ov.cls_off + (size_t)m * (ov.classes + 1);
        for (int c = 0; c < ov.classes; ++c) {
            double pt[DKS_KM_MAX_R];
#pragma unroll
            for (int r = 0; r < DKS_KM_MAX_R; ++r) pt[r] = 0.0;
            for (int v = co[c]; v < co[c + 1]; ++v) {
                const double* sv = k.sv + (size_t)v * D;
                double t = 0.0;
                for (int cc = 0; cc < D; ++cc) t += km_term(k.kernel, x[cc], sv[cc], w[cc], org[cc]);
                const double kv = km_phi(k, t, k.gamma[m]);
#pragma unroll
                for (int r = 0; r < DKS_KM_MAX_R; ++r)
                    if (r < k.R) pt[r] = fma(k.dual[(size_t)v * k.R + r], kv, pt[r]);
            }
            ovo_scatter(c, pt, d);
        }
        const double pm = k.pi[m];
        ovo_head(ov, m, d, [&](int r, double val) { o[r] = ov.mode == DKS_KM_OVO_DECISION ? val : fma(pm, val, o[r]); });
    }
}

// km_predict_kernel under the one-vs-one head
__global__ void km_ovo_predict_kernel(const double* __restrict__ X, int n, int D, KmDev k, KmOvo ov, int C, int link,
                                      const double* __restrict__ linkfnull, double* __restrict__ out,
                                      double* __restrict__ dlink, int* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* x = X + (size_t)i * D;
    bool nan = false;
    for (int c = 0; c < D; ++c) nan |= isnan(x[c]);
    double o[OVO_C];
    if (nan) {
        for (int c = 0; c < C; ++c) o[c] = NAN;
        if (status) report_status(status, DKS_ERR_DOMAIN, i);
    } else {
        km_ovo_outputs(k, ov, x, D, o);
    }
    predict_epilogue(o, C, i, link, linkfnull, out, dlink, status, nan);
}

// shared memory of explain_kmach_ovo_kernel: [C][S_cap] float64 sums / y, then the tile-table / solve region and the varying
// groups [64] as in explain_kmach_kernel (the pair scores live in registers)
__host__ __device__ inline size_t ovo_smem_bytes(int S_cap, int C, int R, int G) {
    const size_t tab = tile_doubles(R, G), solve = 63 * 63 + 64;
    return sizeof(double) * ((size_t)C * S_cap + (tab > solve ? tab : solve)) + sizeof(int) * 64;
}

// explain_kmach_kernel for the one-vs-one head (one CTA per SM's worth of registers: the 28 pair scores stay in registers
// without spilling): the same plans, tables, instantiations (L1, ACC, ROWS) and solve, in the
// loop order the head needs.  Per background row j, coalitions go in chunks of blockDim.x, each thread owning one
// coalition of the chunk; per member the thread keeps that coalition's pair scores in registers across the member's tiles.
// Tiles follow the class blocks (class c is uniform within a tile): a support vector adds dual[v][r] K into the tile's
// partials pt[r], which go into the pair scores when the tile is done (ovo_scatter).  When the member's classes are done,
// its head adds w_j pi_m p_c (or w_j dec_k) into the sums.  The Delta and nibble tables are rebuilt per chunk; threads
// without a coalition in the last chunk still build tables and reach every barrier.  Every sum runs in a fixed order: the
// result does not depend on the grid.  Then y = link(ey) - link(fnull) for every output (logit: 1 - e_c is the sum of
// the other classes), and the solve.
template <bool L1, bool ACC = false, bool ROWS = false>
__global__ void __launch_bounds__(THREADS, 1) explain_kmach_ovo_kernel(ExplainParams p, SimtL1 q, KmDev k, KmOvo ov,
                                                                       const double* __restrict__ X,
                                                                       const double* __restrict__ bg, int D,
                                                                       const int* __restrict__ goff,
                                                                       const int* __restrict__ gcols, EnsAcc ea,
                                                                       EnsRows er) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x;
    const int N = p.N, G = p.G, C = p.C, R = k.R;
    const bool proba = ov.mode == DKS_KM_OVO_PROBA;
    double* acc = reinterpret_cast<double*>(smem_raw);          // [C][S_cap]
    double* region = acc + (size_t)C * p.S_cap;
    const size_t tab = tile_doubles(R, G), solve = 63 * 63 + 64;
    double* A = region;                                         // [63 * 63] (solve)
    double* rhs = A + 63 * 63;                                  // [64]
    double* tj = region;                                        // [TILE] (background loop)
    double* du = tj + TILE;                                     // [TILE][R]
    double* dl = du + TILE * R;                                 // [G][TILE]
    double* tb = dl + (size_t)G * TILE;                         // [ceil(G/4)][TILE][16]
    int* vi = reinterpret_cast<int*>(region + (tab > solve ? tab : solve));   // [64]
    const size_t slab = (size_t)p.n * G;

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
            if (!ACC && tid < C && !fx_bad)
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

        const double* x = X + (size_t)i * D;
        const int nib = (M + 3) >> 2;
        for (int j = ROWS ? er.j0 : 0; j < (ROWS ? er.j1 : N); ++j) {
            const double wb = p.wbg[j];
            if (wb == 0.0) continue;                            // block-uniform
            const double wj = ROWS ? 1.0 : wb;
            const double* b = bg + (size_t)j * D;
            for (int s0 = 0; s0 < S; s0 += blockDim.x) {
                const int s = s0 + tid;
                const bool live = s < S;
                const uint64_t z = live ? zp[s] : 0;
                if (ROWS && live)
                    for (int c = 0; c < C; ++c) acc[(size_t)c * p.S_cap + s] = 0.0;
                for (int m = 0; m < k.K; ++m) {
                    const double gm = k.gamma[m];
                    const double* w = k.colw + (size_t)m * D;
                    const double* org = k.colo + (size_t)m * D;
                    const int* co = ov.cls_off + (size_t)m * (ov.classes + 1);
                    double d[OVO_SLOTS];
#pragma unroll
                    for (int e = 0; e < OVO_SLOTS; ++e) d[e] = 0.0;
                    for (int c = 0; c < ov.classes; ++c) {
                        const int c1 = co[c + 1];
                        for (int v0 = co[c]; v0 < c1; v0 += TILE) {
                            const int nv = min(TILE, c1 - v0);
                            for (int idx = tid; idx < nv; idx += blockDim.x) tj[idx] = k.Tbg[(size_t)j * k.n_sv + v0 + idx];
                            for (int idx = tid; idx < nv * R; idx += blockDim.x) du[idx] = k.dual[(size_t)v0 * R + idx];
                            for (int idx = tid; idx < M * nv; idx += blockDim.x) {
                                const int pp = idx / nv, v = idx - pp * nv, g = vi[pp];
                                const double* sv = k.sv + (size_t)(v0 + v) * D;
                                double dd = 0.0;
                                for (int e = goff[g]; e < goff[g + 1]; ++e) {
                                    const int cc = gcols[e];
                                    dd += km_term(k.kernel, x[cc], sv[cc], w[cc], org[cc]) -
                                          km_term(k.kernel, b[cc], sv[cc], w[cc], org[cc]);
                                }
                                dl[(size_t)pp * TILE + v] = dd;
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
                            if (live) {
                                double pt[DKS_KM_MAX_R];
#pragma unroll
                                for (int r = 0; r < DKS_KM_MAX_R; ++r) pt[r] = 0.0;
                                for (int v = 0; v < nv; ++v) {
                                    double t = tj[v];
                                    for (int qn = 0; qn < nib; ++qn)
                                        t += tb[((size_t)qn * TILE + v) * 16 + ((z >> (4 * qn)) & 15)];
                                    const double kv = km_phi(k, t, gm);
#pragma unroll
                                    for (int r = 0; r < DKS_KM_MAX_R; ++r)
                                        if (r < R) pt[r] = fma(du[v * R + r], kv, pt[r]);
                                }
                                ovo_scatter(c, pt, d);
                            }
                            __syncthreads();
                        }
                    }
                    if (live) {
                        const double wk = proba ? wj * k.pi[m] : wj;
                        ovo_head(ov, m, d, [&](int r, double val) {
                            double* a = acc + (size_t)r * p.S_cap + s;
                            *a = fma(wk, val, *a);
                        });
                    }
                }
                if (ROWS && live) {
                    double o[OVO_C];
                    for (int c = 0; c < C; ++c) o[c] = acc[(size_t)c * p.S_cap + s];
                    rows_store<0>(er, p.S_cap, i, j, s, o);
                }
            }
        }
        __syncthreads();
        if constexpr (ROWS) continue;
        if constexpr (ACC) {
            ens_accumulate(ea, p, i, S, acc);
            continue;
        }

        // y = link(ey) - link(fnull) per output, written over the sums: the probabilities' 1 - e_c is the sum of the other
        // classes (no cancellation), the pair values' 1 - e as written.  Each thread reads and writes only the coalitions it
        // owns.
        int bad = 0;
        for (int s = tid; s < S; s += blockDim.x) {
            double y[OVO_C];
            for (int c = 0; c < C; ++c) {
                const double e = acc[(size_t)c * p.S_cap + s];
                if (p.link == DKS_LINK_LOGIT) {
                    double rest = 0.0;
                    if (proba) {
                        for (int c2 = 0; c2 < C; ++c2)
                            if (c2 != c) rest += acc[(size_t)c2 * p.S_cap + s];
                    } else {
                        rest = 1.0 - e;
                    }
                    y[c] = log(e / rest) - p.linkfnull[c];
                } else {
                    y[c] = e - p.fnull[c];
                }
                bad |= !isfinite(y[c]);
            }
            for (int c = 0; c < C; ++c) acc[(size_t)c * p.S_cap + s] = y[c];
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

}  // namespace kmach
}  // namespace dks
