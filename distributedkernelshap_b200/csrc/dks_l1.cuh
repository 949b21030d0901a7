// l1 feature selection of KernelExplainer.solve on the device (shared-plan path).
//
// Upstream (shap 0.35.0 solve, reached from explainers/kernel_shap.py:250/253 with the kwargs of :836-845, :880): when
// l1_reg is 'aic' / 'bic' / 'num_features(k)', or 'auto' with under 20% of the coalition space sampled, the regression is
// first run on the AUGMENTED system  X = [sqrt(a) z ; sqrt(b) (z - 1)],  y = [sqrt(a) ey ; sqrt(b) (ey - delta)],
// a = w (M - |z|), b = w |z|,  through scikit-learn 0.23.2 -- LassoLarsIC (centre, scale the columns to unit norm, lasso
// path by least-angle regression, information criterion n MSE / var(y) + K df per path step) or lars_path(max_iter = k) --
// and the constrained WLS is then solved on the selected features only.
//
// With a shared plan everything that depends on the plan -- the Gram matrix of the augmented columns (raw, and centred +
// normalised), column sums, norms, the weighted Gram of the plain rows -- is formed once on the host (plan.py: l1_tables).
// Per instance only MOMENT vectors of y are needed:  c_k = sum_s w_s z_sk y_s,  u_k = sum_s b_s z_sk y_s  and three scalars,
//   X^T y_k = (M c_k - u_k) - ((T1 - u_k) - delta (sum_b - bz_k)),   y^T y = M Qw - 2 delta T1 + delta^2 sum_b, ...
// l1_moments_kernel forms them from the (sum p1, sum p0) buffer of the coalition kernel (fixed-point accumulation: exact,
// order-independent); l1_lars_kernel runs the path, the criterion (residual sums of squares as quadratic forms in the Gram
// matrix), and the restricted WLS, one warp per instance, float64, the Cholesky factor of the active block in shared memory.
//
// Instances with a partial varying set (M < G, up to 64 groups) select on the shared plan of their own M: the CUDA-core
// kernel (explain_simt_kernel<true>) forms their moments with the same block_moments, and l1_lars_kernel reads each task's
// M, its tables and its varying groups.
#pragma once

#include "dks_shared.cuh"

namespace dks {
namespace l1 {

constexpr int MODE_AIC = 1, MODE_BIC = 2, MODE_NUM_FEATURES = 3;
constexpr double TINY32 = 1.17549435082228750797e-38;     // np.finfo(np.float32).tiny
constexpr double EQ_TOL = 1.1920928955078125e-07;         // np.finfo(np.float32).eps
constexpr double EPS64 = 2.220446049250313e-16;

struct Params {
    int n, N, G, C, S, S_pad, link, mode, kfeat;
    int nout;                // outputs solved per instance: 1 (binary head: class 1, class 0 its negation) or C
    int binary;              // the binary head (nout 1 is also the identity head with one output, which has no class 0)
    int Mmax;                // largest M of the tasks (sizes each warp's shared-memory area)
    shared_path::HeadSource src;   // softmax / identity heads (nout == C)
    const float2* sums;      // [n][S_pad]
    const uint64_t* z;       // [S][W]
    const double* w;         // [S]
    const Tables* tabs;      // [DKS_L1_MAX_GROUPS + 1] tables of the shared plan of each M
    const int* Mcnt;         // [n] M per instance; NULL: every task has M = G (the shared-plan path)
    const uint64_t* vmask;   // [n] varying groups per instance (with Mcnt; M <= 64)
    const double* dlink;     // [n][C]
    const double* linkfnull;
    const double* fnull;
    const int* list;
    const int* count;
    double* mom;             // [n][nout][2G + 4]: c [M], u [M], T1, Qw, R
    double* phi;             // [C][n][G]
    int* status;
};

// ---- moments of y over the rows of a plan of M groups: c_k = sum_s w_s z_sk y_s and u_k = sum_s b_s z_sk y_s (k < M) into
// mom[k] and mom[M + k]; T1 = sum b y, Qw = sum w y^2, R = sum (sqrt a + sqrt b) y into mom[2M .. 2M + 2].  By a block of
// MOM_THREADS threads; y (ys[s], s < S) is in shared memory, written before a __syncthreads.  2^-40 fixed point: exact and
// order-independent.  SCALED (the multi-output heads): the fixed point is scaled per task by an exact power of two
// (shared_path::fix_exponent; Qw, quadratic in y, by its own even exponent) and the moments are stored unscaled, so the LARS
// path compares them with its absolute thresholds in the units of y.  part / bound: shared scratch.
template <int W, bool SCALED>
__device__ void block_moments(const double* ys, int S, int M, const uint64_t* __restrict__ z, const double* __restrict__ w,
                              const double* __restrict__ b, const double* __restrict__ sqab, double* mom,
                              long long (*part)[32], double (*bound)[2]) {
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    long long t1 = 0, qw = 0, rr = 0;
    double sc = 1.0, isc = 1.0, sq = 1.0, isq = 1.0;
    if constexpr (SCALED) {
        double b1 = 0.0, b2 = 0.0;        // bounds of the linear moments and of Qw
        for (int s = threadIdx.x; s < S; s += MOM_THREADS) {
            const double y = ys[s];
            b1 += (w[s] + b[s] + sqab[s]) * fabs(y);
            b2 += w[s] * y * y;
        }
        b1 = warp_sum(b1); b2 = warp_sum(b2);
        if (lane == 0) { bound[wib][0] = b1; bound[wib][1] = b2; }
        __syncthreads();
        double t1b = 0.0, t2b = 0.0;
#pragma unroll
        for (int wq = 0; wq < MOM_THREADS / 32; ++wq) { t1b += bound[wq][0]; t2b += bound[wq][1]; }
        const int e1 = shared_path::fix_exponent(t1b), e2 = shared_path::fix_exponent(t2b) >> 1;
        sc = ldexp(1.0, e1); isc = ldexp(1.0, -e1);
        sq = ldexp(1.0, e2); isq = ldexp(1.0, -2 * e2);
        for (int s = threadIdx.x; s < S; s += MOM_THREADS) {
            const double y = ys[s];
            t1 += to_fix(b[s] * y * sc);
            qw += to_fix(w[s] * (y * sq) * (y * sq));
            rr += to_fix(sqab[s] * y * sc);
        }
    } else {
        for (int s = threadIdx.x; s < S; s += MOM_THREADS) {
            const double y = ys[s];
            t1 += to_fix(b[s] * y);
            qw += to_fix(w[s] * y * y);
            rr += to_fix(sqab[s] * y);
        }
    }
    t1 = warp_sum_ll(t1); qw = warp_sum_ll(qw); rr = warp_sum_ll(rr);
    if (lane == 0) { part[wib][0] = t1; part[wib][1] = qw; part[wib][2] = rr; }
    __syncthreads();
    if (threadIdx.x < 3) {
        long long acc = 0;
        for (int wq = 0; wq < MOM_THREADS / 32; ++wq) acc += part[wq][threadIdx.x];
        mom[2 * M + threadIdx.x] = SCALED ? from_fix(acc) * (threadIdx.x == 1 ? isq : isc) : from_fix(acc);
    }
    __syncthreads();
    // sixteen coefficients of c and u per pass over the rows
    for (int k0 = 0; k0 < M; k0 += 16) {
        long long Ck[16], Uk[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) { Ck[k] = 0; Uk[k] = 0; }
#pragma unroll 2
        for (int s = threadIdx.x; s < S; s += MOM_THREADS) {
            const double y = SCALED ? ys[s] * sc : ys[s];
            const long long vc = to_fix(w[s] * y), vu = to_fix(b[s] * y);
            const uint32_t zb = (uint32_t)(z[(size_t)s * W + (k0 >> 6)] >> (k0 & 63));
#pragma unroll
            for (int k = 0; k < 16; ++k)
                if ((zb >> k) & 1u) { Ck[k] += vc; Uk[k] += vu; }
        }
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const long long rc = warp_sum_ll(Ck[k]), ru = warp_sum_ll(Uk[k]);
            if (lane == 0) { part[wib][k] = rc; part[wib][16 + k] = ru; }
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            long long acc = 0;
            for (int wq = 0; wq < MOM_THREADS / 32; ++wq) acc += part[wq][threadIdx.x];
            const int k = k0 + (threadIdx.x & 15);
            if (k < M) mom[(threadIdx.x < 16 ? 0 : M) + k] = SCALED ? from_fix(acc) * isc : from_fix(acc);
        }
        __syncthreads();
    }
}

// ---- moments of the shared-plan path's instances (M = G): y from the (sum p1, sum p0) buffer, or (MULTI: the softmax,
// one-vs-rest and identity heads, one task per (instance, output)) from p.src
template <int W, bool MULTI = false>
__global__ void __launch_bounds__(MOM_THREADS) l1_moments_kernel(Params p) {
    extern __shared__ double s_y[];                       // [S]
    __shared__ long long s_part[MOM_THREADS / 32][32];
    __shared__ LogTabEntry s_logtab[DKS_LOGTAB_SIZE];
    __shared__ double s_bound[MOM_THREADS / 32][2];
    const int G = p.G;
    const int nout = MULTI ? p.nout : 1;
    const int cnt = *p.count * nout;
    if ((int)blockIdx.x >= cnt) return;
    if (threadIdx.x < DKS_LOGTAB_SIZE) logtab_fill(s_logtab, threadIdx.x);
    __syncthreads();
    const Tables& t = p.tabs[G];
    const double lf1 = p.linkfnull[1], f1 = p.fnull[1], inv_n = 1.0 / (double)p.N;
    for (int m = blockIdx.x; m < cnt; m += gridDim.x) {
        const int i = p.list[MULTI ? m / nout : m];
        const int cls = MULTI ? m % nout : 1;
        const float2* sums = p.sums + (size_t)i * p.S_pad;
        double* mom = p.mom + ((size_t)i * nout + (MULTI ? cls : 0)) * (2 * G + 4);
        if constexpr (MULTI) {
            const double fnc = p.fnull[cls], lfc = p.linkfnull[cls];
            int bad = 0;
            for (int s = threadIdx.x; s < p.S; s += MOM_THREADS) {
                const double y = shared_path::head_y<W>(p.src, i, cls, p.C, s, p.S_pad, p.z + (size_t)s * W, p.link, inv_n,
                                                        fnc, lfc);
                bad |= !isfinite(y);
                s_y[s] = y;
            }
            // exp head: a non-finite y is reported and kept out of the fixed point; NaN moments make the LARS skip the task
            if (__syncthreads_or(p.src.act == DKS_ACT_EXP && bad)) {
                if (threadIdx.x == 0) {
                    if (atomicCAS(&p.status[0], 0, DKS_ERR_NUMERIC) == 0) p.status[1] = i;
                    mom[2 * G] = NAN;
                }
                continue;
            }
        } else {
            for (int s = threadIdx.x; s < p.S; s += MOM_THREADS) {
                const float2 a = sums[s];
                double y;
                if (p.link == DKS_LINK_LOGIT) y = fast_log_ratio(a.x, a.y, s_logtab) - lf1;
                else y = (double)a.x * inv_n - f1;
                s_y[s] = y;
            }
        }
        __syncthreads();
        block_moments<W, MULTI>(s_y, p.S, G, p.z, p.w, t.b, t.sqab, mom, s_part, s_bound);
    }
}

// splits the general kernels' instance list (all n instances when list is NULL) into those whose M selects (bit M - 1 of
// sel) and the rest; counts [2] are zero on entry
__global__ void l1_partition_kernel(const int* __restrict__ list, const int* __restrict__ count, int n,
                                    const int* __restrict__ Mcnt, uint64_t sel_lo, uint64_t sel_hi, int* __restrict__ out_sel,
                                    int* __restrict__ out_plain, int* __restrict__ counts) {
    const int cnt = list != nullptr ? *count : n;
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < cnt; q += gridDim.x * blockDim.x) {
        const int i = list != nullptr ? list[q] : q;
        const int M = Mcnt[i];
        const bool sel = M >= 1 && M <= 128 && (((M <= 64 ? sel_lo >> (M - 1) : sel_hi >> (M - 65)) & 1ull) != 0);
        if (sel) out_sel[atomicAdd(&counts[0], 1)] = i;
        else out_plain[atomicAdd(&counts[1], 1)] = i;
    }
}

// ---- warp helpers ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double wsum(double v) { return warp_sum(v); }
__device__ __forceinline__ double wmin(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ int tri(int r) { return r * (r + 1) / 2; }        // packed lower-triangular row offset

// Cholesky factor (packed, row-major lower) of gram[perm[a]][perm[b]], a, b < k: by the whole warp, column by column
__device__ inline void chol_rebuild(double* L, const double* __restrict__ gram, const int* perm, int k, int M, int lane) {
    for (int r = lane; r < k; r += 32)
        for (int c = 0; c <= r; ++c) L[tri(r) + c] = gram[(size_t)perm[r] * M + perm[c]];
    __syncwarp();
    for (int c = 0; c < k; ++c) {
        const double d = sqrt(fmax(L[tri(c) + c], EPS64 * EPS64));
        __syncwarp();
        if (lane == 0) L[tri(c) + c] = d;
        for (int r = c + 1 + lane; r < k; r += 32) L[tri(r) + c] /= d;
        __syncwarp();
        for (int r = c + 1 + lane; r < k; r += 32) {
            const double lrc = L[tri(r) + c];
            for (int c2 = c + 1; c2 <= r; ++c2) L[tri(r) + c2] -= lrc * L[tri(c2) + c];
        }
        __syncwarp();
    }
}

// x <- (L L^T)^-1 x for the leading k x k block (column-oriented substitutions: no reductions)
__device__ inline void chol_solve(const double* L, double* x, int k, int lane) {
    for (int c = 0; c < k; ++c) {
        __syncwarp();
        const double xc = x[c] / L[tri(c) + c];
        __syncwarp();
        if (lane == 0) x[c] = xc;
        for (int r = c + 1 + lane; r < k; r += 32) x[r] -= L[tri(r) + c] * xc;
    }
    for (int c = k - 1; c >= 0; --c) {
        __syncwarp();
        const double xc = x[c] / L[tri(c) + c];
        __syncwarp();
        if (lane == 0) x[c] = xc;
        for (int r = lane; r < c; r += 32) x[r] -= L[tri(c) + r] * xc;
    }
    __syncwarp();
}

// a warp's area ends with M ints: rounded up to whole doubles, so that the next warp's area (and the staged Gram matrix
// behind the last one) stays 8-byte aligned for odd M
__host__ __device__ inline size_t lars_smem_per_warp(int M) {
    const size_t bytes = sizeof(double) * ((size_t)M * (M + 1) / 2 + 8 * (size_t)M) + sizeof(int) * (size_t)M;
    return (bytes + sizeof(double) - 1) / sizeof(double) * sizeof(double);
}

// group of the v-th varying position (the v-th set bit of vm)
__device__ __forceinline__ int nth_set_bit(uint64_t vm, int v) {
    for (int r = 0; r < v; ++r) vm &= vm - 1;
    return __ffsll((long long)vm) - 1;
}

// one warp per (instance, output).  stage_gram: every task has M = p.Mmax (the shared-plan path's launch), whose Gram matrix
// the CTA stages in shared memory; tasks of mixed M (the general list) read theirs through L2.
__global__ void l1_lars_kernel(Params p, int warps_per_cta, int stage_gram) {
    extern __shared__ __align__(16) unsigned char l1_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int G = p.G, C = p.C;
    const int cnt = *p.count;
    const size_t per_warp = lars_smem_per_warp(p.Mmax);
    const bool lasso = p.mode != MODE_NUM_FEATURES;
    double* sg = reinterpret_cast<double*>(l1_smem + (size_t)warps_per_cta * per_warp);
    if (stage_gram) {
        // the Gram matrix of the path (read k (M - k) times per step) shared by the warps of the CTA, behind their private areas
        const Tables& t = p.tabs[p.Mmax];
        const double* src = lasso ? t.gram_norm : t.gram_raw;
        for (int idx = threadIdx.x; idx < p.Mmax * p.Mmax; idx += blockDim.x) sg[idx] = src[idx];
        __syncthreads();
    }
    unsigned char* warea = l1_smem + (size_t)wib * per_warp;
    const int max_iter = lasso ? 500 : p.kfeat;
    const size_t slab = (size_t)p.n * G;

    const int nout = p.nout;
    for (int m = blockIdx.x * warps_per_cta + wib; m < cnt * nout; m += gridDim.x * warps_per_cta) {
        // one warp per (instance, output): upstream's solve runs the selection for each output on its own
        const int i = p.list[m / nout];
        const int cls = p.binary ? 1 : m % nout;
        const int M = p.Mcnt != nullptr ? p.Mcnt[i] : G;
        const Tables* t = p.tabs + M;
        double* L = reinterpret_cast<double*>(warea);  // packed lower triangle
        double* cov = L + (size_t)M * (M + 1) / 2;      // by variable
        double* cov0 = cov + M;
        double* coef = cov0 + M;                        // by variable
        double* ls = coef + M;                          // by active position
        double* corr = ls + M;                          // by variable
        double* sgn = corr + M;                         // by active position
        double* xrow = sgn + M;                         // scratch
        double* cm = xrow + M;                          // c moments (by variable)
        int* perm = reinterpret_cast<int*>(cm + M);     // position -> variable
        const double* gram = stage_gram ? sg : (lasso ? t->gram_norm : t->gram_raw);
        const double nsamp = (double)t->n_aug;
        const double sum_b = t->sum_b;
        const double* mom = p.mom + ((size_t)i * nout + (p.binary ? 0 : cls)) * (2 * G + 4);
        const double delta = p.dlink[(size_t)i * C + cls];
        const double T1 = mom[2 * M], Qw = mom[2 * M + 1], R = mom[2 * M + 2];
        if (p.src.act == DKS_ACT_EXP && !isfinite(T1 + delta)) {
            // a task the moments kernel reported (non-finite y: NaN T1) or a non-finite f(x): nothing is written to phi
            if (lane == 0 && atomicCAS(&p.status[0], 0, DKS_ERR_NUMERIC) == 0) p.status[1] = i;
            continue;
        }
        const double ybar = lasso ? (R - delta * t->sum_sqb) / nsamp : 0.0;
        const double yy = (double)M * Qw - 2.0 * delta * T1 + delta * delta * sum_b - nsamp * ybar * ybar;
        for (int v = lane; v < M; v += 32) {
            const double c = mom[v], u = mom[M + v];
            double xty = ((double)M * c - u) - ((T1 - u) - delta * (sum_b - t->bz[v]));
            if (lasso) xty = (xty - t->colsum[v] * ybar) / t->scale[v];
            cov[v] = xty; cov0[v] = xty; coef[v] = 0.0; corr[v] = 0.0; cm[v] = c; perm[v] = v;
        }
        __syncwarp();
        int k = 0, n_iter = 0;
        bool drop = false;
        double prev_alpha = 0.0;
        const double K = p.mode == MODE_BIC ? log(nsamp) : 2.0;
        double best_crit = nsamp * (yy / nsamp) / (yy / nsamp + EPS64);       // path step 0: all coefficients zero
        unsigned long long best_lo = 0ull, best_hi = 0ull;
        double rss = yy;                         // residual sum of squares along the path (centred y at step 0)

        while (true) {
            // most correlated inactive variable, first maximum in position order
            double bv = -1.0; int bp = M;
            for (int pos = k + lane; pos < M; pos += 32) {
                const double a = fabs(cov[perm[pos]]);
                if (a > bv) { bv = a; bp = pos; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int op = __shfl_xor_sync(0xffffffffu, bp, o);
                if (ov > bv || (ov == bv && op < bp)) { bv = ov; bp = op; }
            }
            const double Cabs = k < M ? bv : 0.0;
            const double C_ = k < M ? cov[perm[bp]] : 0.0;
            const double alpha = Cabs / nsamp;
            if (alpha <= EQ_TOL) break;                       // alpha_min = 0: the path is complete
            if (n_iter >= max_iter || k >= M) break;
            if (!drop) {
                // the variable joins the active set: one more row of the Cholesky factor
                __syncwarp();
                if (lane == 0) { const int t = perm[k]; perm[k] = perm[bp]; perm[bp] = t; }
                __syncwarp();
                const int v = perm[k];
                for (int j = lane; j < k; j += 32) xrow[j] = gram[(size_t)v * M + perm[j]];
                __syncwarp();
                for (int c = 0; c < k; ++c) {                 // forward substitution, column-oriented
                    const double xc = xrow[c] / L[tri(c) + c];
                    __syncwarp();
                    if (lane == 0) xrow[c] = xc;
                    for (int r = c + 1 + lane; r < k; r += 32) xrow[r] -= L[tri(r) + c] * xc;
                    __syncwarp();
                }
                double v2 = 0.0;
                for (int j = lane; j < k; j += 32) v2 += xrow[j] * xrow[j];
                v2 = wsum(v2);
                const double diag = fmax(sqrt(fabs(gram[(size_t)v * M + v] - v2)), EPS64);
                if (diag < 1e-7) {
                    // degenerate regressor: its correlation is zeroed and it goes back among the inactive ones
                    __syncwarp();
                    if (lane == 0) { cov[v] = 0.0; const int t = perm[k]; perm[k] = perm[bp]; perm[bp] = t; }
                    __syncwarp();
                    continue;
                }
                for (int j = lane; j < k; j += 32) L[tri(k) + j] = xrow[j];
                if (lane == 0) { L[tri(k) + k] = diag; sgn[k] = C_ > 0.0 ? 1.0 : (C_ < 0.0 ? -1.0 : 0.0); }
                ++k;
                __syncwarp();
            }
            if (lasso && n_iter > 0 && prev_alpha < alpha) break;            // alpha increasing: numerical noise, stop
            // equiangular direction: (L L^T) ls = sign
            for (int a = lane; a < k; a += 32) ls[a] = sgn[a];
            __syncwarp();
            chol_solve(L, ls, k, lane);
            double AA;
            if (k == 1 && ls[0] == 0.0) {
                __syncwarp();
                if (lane == 0) ls[0] = 1.0;
                AA = 1.0;
                __syncwarp();
            } else {
                double dot = 0.0;
                for (int a = lane; a < k; a += 32) dot += ls[a] * sgn[a];
                dot = wsum(dot);
                AA = 1.0 / sqrt(dot);
                if (!isfinite(AA)) {
                    if (lane == 0 && atomicCAS(&p.status[0], 0, DKS_ERR_NUMERIC) == 0) p.status[1] = i;
                    break;
                }
                __syncwarp();
                for (int a = lane; a < k; a += 32) ls[a] *= AA;
                __syncwarp();
            }
            // correlation of every inactive variable with the equiangular direction, step length
            double g = 1.7976931348623157e308;
            for (int pos = k + lane; pos < M; pos += 32) {
                const int v = perm[pos];
                double acc = 0.0;
                for (int a = 0; a < k; ++a) acc += gram[(size_t)perm[a] * M + v] * ls[a];
                corr[v] = acc;
                const double g1 = (Cabs - cov[v]) / (AA - acc + TINY32), g2 = (Cabs + cov[v]) / (AA + acc + TINY32);
                if (g1 > 0.0) g = fmin(g, g1);
                if (g2 > 0.0) g = fmin(g, g2);
            }
            g = wmin(g);
            double gamma = fmin(g, Cabs / AA);
            // a coefficient about to cross zero?
            double zp = 1.7976931348623157e308;
            for (int a = lane; a < k; a += 32) {
                const double z = -coef[perm[a]] / (ls[a] + TINY32);
                xrow[a] = z;
                if (z > 0.0) zp = fmin(zp, z);
            }
            zp = wmin(zp);
            __syncwarp();
            drop = false;
            if (zp < gamma) {
                for (int a = lane; a < k; a += 32) if (xrow[a] == zp) sgn[a] = -sgn[a];
                if (lasso) gamma = zp;
                drop = true;
            }
            ++n_iter;
            __syncwarp();
            for (int a = lane; a < k; a += 32) coef[perm[a]] += gamma * ls[a];
            for (int pos = k + lane; pos < M; pos += 32) cov[perm[pos]] -= gamma * corr[perm[pos]];
            __syncwarp();
            if (lasso) {
                // information criterion of this path step.  The residual moves along the unit equiangular vector u by gamma
                // and r'u = C / AA (every active variable has correlation +-C with r), so
                //     RSS_new = RSS - 2 gamma C / AA + gamma^2
                // -- O(1) per step instead of the quadratic form b'Gb (which re-read k^2 Gram entries through L2).
                rss += gamma * gamma - 2.0 * gamma * Cabs / AA;
                int df = 0;
                unsigned long long nz_lo = 0ull, nz_hi = 0ull;
                for (int a = lane; a < k; a += 32) {
                    const int va = perm[a];
                    if (fabs(coef[va]) > EPS64) ++df;
                    if (coef[va] != 0.0) { if (va < 64) nz_lo |= 1ull << va; else nz_hi |= 1ull << (va - 64); }
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    df += __shfl_xor_sync(0xffffffffu, df, o);
                    nz_lo |= __shfl_xor_sync(0xffffffffu, nz_lo, o);
                    nz_hi |= __shfl_xor_sync(0xffffffffu, nz_hi, o);
                }
                const double crit = nsamp * (rss / nsamp) / (yy / nsamp + EPS64) + K * (double)df;
                if (crit < best_crit) { best_crit = crit; best_lo = nz_lo; best_hi = nz_hi; }
            }
            if (drop && lasso) {
                // the variable(s) whose coefficient reached zero leave the active set (highest position first)
                for (int a = k - 1; a >= 0; --a) {
                    if (xrow[a] != zp) continue;
                    __syncwarp();
                    const int d = perm[a];
                    double acc = 0.0;                          // its correlation is recomputed from the copies
                    for (int v = lane; v < M; v += 32) acc += gram[(size_t)d * M + v] * coef[v];
                    acc = wsum(acc);
                    __syncwarp();
                    if (lane == 0) {
                        for (int q = a; q < k - 1; ++q) { perm[q] = perm[q + 1]; sgn[q] = sgn[q + 1]; xrow[q] = xrow[q + 1]; }
                        perm[k - 1] = d; sgn[k - 1] = 0.0; xrow[k - 1] = -1.0;
                        cov[d] = cov0[d] - acc;
                        coef[d] = 0.0;
                    }
                    --k;
                    __syncwarp();
                }
                chol_rebuild(L, gram, perm, k, M, lane);
            }
            prev_alpha = alpha;
        }

        // ---- selected features -> restricted constrained WLS (the last selected feature is eliminated)
        unsigned long long sel_lo = best_lo, sel_hi = best_hi;
        if (!lasso) {
            sel_lo = 0ull; sel_hi = 0ull;
            for (int a = 0; a < k; ++a) { const int v = perm[a]; if (v < 64) sel_lo |= 1ull << v; else sel_hi |= 1ull << (v - 64); }
        }
        __syncwarp();
        int q = 0;
        for (int v = 0; v < M; ++v) {
            const bool on = v < 64 ? ((sel_lo >> v) & 1ull) : ((sel_hi >> (v - 64)) & 1ull);
            if (on) { if (lane == 0) perm[q] = v; ++q; }
        }
        __syncwarp();
        double* phi1 = p.phi + (size_t)cls * slab + (size_t)i * G;
        double* phi0 = p.phi + (size_t)i * G;       // binary head only: class 0 is the negation of class 1
        const bool anti = p.binary != 0;
        // variable v is the group of the v-th varying position; the groups that do not vary keep zeros
        const uint64_t vm = p.Mcnt != nullptr ? p.vmask[i] : 0ull;
        auto grp = [&](int v) { return p.Mcnt != nullptr ? nth_set_bit(vm, v) : v; };
        for (int g = lane; g < G; g += 32) { phi1[g] = 0.0; if (anti) phi0[g] = 0.0; }
        __syncwarp();
        if (q == 1) {
            if (lane == 0) { double val = fabs(delta) < 1e-10 ? 0.0 : delta; const int g = grp(perm[0]); phi1[g] = val; if (anti) phi0[g] = val == 0.0 ? 0.0 : -val; }
        } else if (q >= 2) {
            const int nA = q - 1, Lv = perm[q - 1];
            const double* gw = t->gram_w;
            const double gLL = gw[(size_t)Lv * M + Lv];
            for (int r = lane; r < nA; r += 32) {
                const int vr = perm[r];
                for (int c = 0; c <= r; ++c) {
                    const int vc = perm[c];
                    L[tri(r) + c] = gw[(size_t)vr * M + vc] - gw[(size_t)vr * M + Lv] - gw[(size_t)vc * M + Lv] + gLL;
                }
                xrow[r] = (cm[vr] - cm[Lv]) - delta * (gw[(size_t)vr * M + Lv] - gLL);
            }
            __syncwarp();
            // in-place Cholesky of the nA x nA normal matrix
            bool ok = true;
            for (int c = 0; c < nA; ++c) {
                const double dd = L[tri(c) + c];
                if (!(dd > 0.0)) ok = false;
                const double d = sqrt(dd);
                __syncwarp();
                if (lane == 0) L[tri(c) + c] = d;
                for (int r = c + 1 + lane; r < nA; r += 32) L[tri(r) + c] /= d;
                __syncwarp();
                for (int r = c + 1 + lane; r < nA; r += 32) {
                    const double lrc = L[tri(r) + c];
                    for (int c2 = c + 1; c2 <= r; ++c2) L[tri(r) + c2] -= lrc * L[tri(c2) + c];
                }
                __syncwarp();
            }
            if (!ok && lane == 0 && atomicCAS(&p.status[0], 0, DKS_ERR_NUMERIC) == 0) p.status[1] = i;
            chol_solve(L, xrow, nA, lane);
            double sum = 0.0;
            for (int r = lane; r < nA; r += 32) {
                double val = xrow[r];
                sum += val;
                if (fabs(val) < 1e-10) val = 0.0;
                const int g = grp(perm[r]);
                phi1[g] = val;
                if (anti) phi0[g] = val == 0.0 ? 0.0 : -val;
            }
            sum = wsum(sum);
            if (lane == 0) {
                double last = delta - sum;
                if (fabs(last) < 1e-10) last = 0.0;
                const int g = grp(Lv);
                phi1[g] = last;
                if (anti) phi0[g] = last == 0.0 ? 0.0 : -last;
            }
        }
        __syncwarp();
    }
}

}  // namespace l1
}  // namespace dks
