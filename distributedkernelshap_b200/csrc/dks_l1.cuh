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
#pragma once

#include "dks_shared.cuh"

namespace dks {
namespace l1 {

constexpr int MODE_AIC = 1, MODE_BIC = 2, MODE_NUM_FEATURES = 3;
constexpr double TINY32 = 1.17549435082228750797e-38;     // np.finfo(np.float32).tiny
constexpr double EQ_TOL = 1.1920928955078125e-07;         // np.finfo(np.float32).eps
constexpr double EPS64 = 2.220446049250313e-16;

struct Tables {              // per plan (M == G), device pointers
    const double* gram_raw;  // [M][M]
    const double* gram_norm; // [M][M]
    const double* colsum;    // [M]
    const double* scale;     // [M]
    const double* bz;        // [M]
    const double* gram_w;    // [M][M] sum_s w_s z_sk z_sl
    const double* b;         // [S] w_s |z_s|
    const double* sqab;      // [S] sqrt(a_s) + sqrt(b_s)
    double sum_b, sum_sqb;
    int n_aug;
};

struct Params {
    int n, N, G, C, S, S_pad, link, mode, kfeat;
    int nout;                // outputs solved per instance: 1 (binary head: class 1, class 0 its negation) or C
    shared_path::HeadSource src;   // softmax / identity heads (nout == C)
    const float2* sums;      // [n][S_pad]
    const uint64_t* z;       // [S][W]
    const double* w;         // [S]
    Tables t;
    const double* dlink;     // [n][C]
    const double* linkfnull;
    const double* fnull;
    const int* list;
    const int* count;
    double* mom;             // [n][nout][2G + 4]: c, u, T1, Qw, R
    double* phi;             // [C][n][G]
    int* status;
};

// ---- moments of y over the plan rows: c_k, u_k (k < G) and T1 = sum b y, Qw = sum w y^2, R = sum (sqrt a + sqrt b) y
// MULTI: the softmax and identity heads, one task per (instance, output) with y from p.src; the fixed point is scaled per
// task (shared_path::fix_exponent; Qw, quadratic in y, by its own even exponent) and the moments are stored unscaled, so the
// LARS path compares them with its absolute thresholds in the units of y.
constexpr int MOM_THREADS = 256;
template <int W, bool MULTI = false>
__global__ void __launch_bounds__(MOM_THREADS) l1_moments_kernel(Params p) {
    extern __shared__ double s_y[];                       // [S]
    __shared__ long long s_part[MOM_THREADS / 32][32];
    __shared__ LogTabEntry s_logtab[DKS_LOGTAB_SIZE];
    __shared__ double s_bound[MOM_THREADS / 32][2];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int G = p.G;
    const int nout = MULTI ? p.nout : 1;
    const int cnt = *p.count * nout;
    if ((int)blockIdx.x >= cnt) return;
    if (threadIdx.x < DKS_LOGTAB_SIZE) logtab_fill(s_logtab, threadIdx.x);
    __syncthreads();
    const double lf1 = p.linkfnull[1], f1 = p.fnull[1], inv_n = 1.0 / (double)p.N;
    for (int m = blockIdx.x; m < cnt; m += gridDim.x) {
        const int i = p.list[MULTI ? m / nout : m];
        const int cls = MULTI ? m % nout : 1;
        const float2* sums = p.sums + (size_t)i * p.S_pad;
        double* mom = p.mom + ((size_t)i * nout + (MULTI ? cls : 0)) * (2 * G + 4);
        // pass 0: y into shared memory + the three scalars
        long long t1 = 0, qw = 0, rr = 0;
        double sc = 1.0, isc = 1.0, sq = 1.0, isq = 1.0;
        if constexpr (MULTI) {
            const double fnc = p.fnull[cls], lfc = p.linkfnull[cls];
            double b1 = 0.0, b2 = 0.0;        // bounds of the linear moments and of Qw
            for (int s = threadIdx.x; s < p.S; s += MOM_THREADS) {
                const double y = shared_path::head_y<W>(p.src, i, cls, p.C, s, p.S_pad, p.z + (size_t)s * W, p.link, inv_n,
                                                        fnc, lfc);
                s_y[s] = y;
                b1 += (p.w[s] + p.t.b[s] + p.t.sqab[s]) * fabs(y);
                b2 += p.w[s] * y * y;
            }
            b1 = warp_sum(b1); b2 = warp_sum(b2);
            if (lane == 0) { s_bound[wib][0] = b1; s_bound[wib][1] = b2; }
            __syncthreads();
            double t1b = 0.0, t2b = 0.0;
#pragma unroll
            for (int wq = 0; wq < MOM_THREADS / 32; ++wq) { t1b += s_bound[wq][0]; t2b += s_bound[wq][1]; }
            const int e1 = shared_path::fix_exponent(t1b), e2 = shared_path::fix_exponent(t2b) >> 1;
            sc = ldexp(1.0, e1); isc = ldexp(1.0, -e1);
            sq = ldexp(1.0, e2); isq = ldexp(1.0, -2 * e2);
            for (int s = threadIdx.x; s < p.S; s += MOM_THREADS) {
                const double y = s_y[s];
                t1 += to_fix(p.t.b[s] * y * sc);
                qw += to_fix(p.w[s] * (y * sq) * (y * sq));
                rr += to_fix(p.t.sqab[s] * y * sc);
            }
        } else {
            for (int s = threadIdx.x; s < p.S; s += MOM_THREADS) {
                const float2 a = sums[s];
                double y;
                if (p.link == DKS_LINK_LOGIT) y = fast_log_ratio(a.x, a.y, s_logtab) - lf1;
                else y = (double)a.x * inv_n - f1;
                s_y[s] = y;
                t1 += to_fix(p.t.b[s] * y);
                qw += to_fix(p.w[s] * y * y);
                rr += to_fix(p.t.sqab[s] * y);
            }
        }
        t1 = warp_sum_ll(t1); qw = warp_sum_ll(qw); rr = warp_sum_ll(rr);
        if (lane == 0) { s_part[wib][0] = t1; s_part[wib][1] = qw; s_part[wib][2] = rr; }
        __syncthreads();
        if (threadIdx.x < 3) {
            long long acc = 0;
            for (int wq = 0; wq < MOM_THREADS / 32; ++wq) acc += s_part[wq][threadIdx.x];
            mom[2 * G + threadIdx.x] = MULTI ? from_fix(acc) * (threadIdx.x == 1 ? isq : isc) : from_fix(acc);
        }
        __syncthreads();
        // sixteen coefficients of c and u per pass over the rows
        for (int k0 = 0; k0 < G; k0 += 16) {
            long long Ck[16], Uk[16];
#pragma unroll
            for (int k = 0; k < 16; ++k) { Ck[k] = 0; Uk[k] = 0; }
#pragma unroll 2
            for (int s = threadIdx.x; s < p.S; s += MOM_THREADS) {
                const double y = MULTI ? s_y[s] * sc : s_y[s];
                const long long vc = to_fix(p.w[s] * y), vu = to_fix(p.t.b[s] * y);
                const uint32_t zb = (uint32_t)(p.z[(size_t)s * W + (k0 >> 6)] >> (k0 & 63));
#pragma unroll
                for (int k = 0; k < 16; ++k)
                    if ((zb >> k) & 1u) { Ck[k] += vc; Uk[k] += vu; }
            }
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const long long rc = warp_sum_ll(Ck[k]), ru = warp_sum_ll(Uk[k]);
                if (lane == 0) { s_part[wib][k] = rc; s_part[wib][16 + k] = ru; }
            }
            __syncthreads();
            if (threadIdx.x < 32) {
                long long acc = 0;
                for (int wq = 0; wq < MOM_THREADS / 32; ++wq) acc += s_part[wq][threadIdx.x];
                const int k = k0 + (threadIdx.x & 15);
                if (k < G) mom[(threadIdx.x < 16 ? 0 : G) + k] = MULTI ? from_fix(acc) * isc : from_fix(acc);
            }
            __syncthreads();
        }
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

__host__ __device__ inline size_t lars_smem_per_warp(int M) {
    return sizeof(double) * ((size_t)M * (M + 1) / 2 + 8 * (size_t)M) + sizeof(int) * (size_t)M;
}

// one warp per instance
__global__ void l1_lars_kernel(Params p, int warps_per_cta, int stage_gram) {
    extern __shared__ __align__(16) unsigned char l1_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int M = p.G, C = p.C;
    const int cnt = *p.count;
    const size_t per_warp = lars_smem_per_warp(M);
    const bool lasso_mode = p.mode != MODE_NUM_FEATURES;
    if (stage_gram) {
        // the Gram matrix of the path (read k (M - k) times per step) shared by the warps of the CTA, behind their private areas
        double* sg = reinterpret_cast<double*>(l1_smem + (size_t)warps_per_cta * per_warp);
        const double* src = lasso_mode ? p.t.gram_norm : p.t.gram_raw;
        for (int idx = threadIdx.x; idx < M * M; idx += blockDim.x) sg[idx] = src[idx];
        __syncthreads();
    }
    double* L = reinterpret_cast<double*>(l1_smem + (size_t)wib * per_warp);    // packed lower triangle
    double* cov = L + (size_t)M * (M + 1) / 2;      // by variable
    double* cov0 = cov + M;
    double* coef = cov0 + M;                        // by variable
    double* ls = coef + M;                          // by active position
    double* corr = ls + M;                          // by variable
    double* sgn = corr + M;                         // by active position
    double* xrow = sgn + M;                         // scratch
    double* cm = xrow + M;                          // c moments (by variable)
    int* perm = reinterpret_cast<int*>(cm + M);     // position -> variable
    const bool lasso = lasso_mode;
    const double* gram = stage_gram ? reinterpret_cast<const double*>(l1_smem + (size_t)warps_per_cta * per_warp)
                                    : (lasso ? p.t.gram_norm : p.t.gram_raw);
    const double nsamp = (double)p.t.n_aug;
    const int max_iter = lasso ? 500 : p.kfeat;
    const size_t slab = (size_t)p.n * M;

    const int nout = p.nout;
    for (int m = blockIdx.x * warps_per_cta + wib; m < cnt * nout; m += gridDim.x * warps_per_cta) {
        // one warp per (instance, output): upstream's solve runs the selection for each output on its own
        const int i = p.list[m / nout];
        const int cls = nout == 1 ? 1 : m % nout;
        const double* mom = p.mom + ((size_t)i * nout + (nout == 1 ? 0 : cls)) * (2 * M + 4);
        const double delta = p.dlink[(size_t)i * C + cls];
        const double T1 = mom[2 * M], Qw = mom[2 * M + 1], R = mom[2 * M + 2];
        const double ybar = lasso ? (R - delta * p.t.sum_sqb) / nsamp : 0.0;
        const double yy = (double)M * Qw - 2.0 * delta * T1 + delta * delta * p.t.sum_b - nsamp * ybar * ybar;
        for (int v = lane; v < M; v += 32) {
            const double c = mom[v], u = mom[M + v];
            double xty = ((double)M * c - u) - ((T1 - u) - delta * (p.t.sum_b - p.t.bz[v]));
            if (lasso) xty = (xty - p.t.colsum[v] * ybar) / p.t.scale[v];
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
        double* phi1 = p.phi + (size_t)cls * slab + (size_t)i * M;
        double* phi0 = p.phi + (size_t)i * M;       // binary head only: class 0 is the negation of class 1
        const bool anti = nout == 1;
        for (int v = lane; v < M; v += 32) { phi1[v] = 0.0; if (anti) phi0[v] = 0.0; }
        __syncwarp();
        if (q == 1) {
            if (lane == 0) { double val = fabs(delta) < 1e-10 ? 0.0 : delta; phi1[perm[0]] = val; if (anti) phi0[perm[0]] = val == 0.0 ? 0.0 : -val; }
        } else if (q >= 2) {
            const int nA = q - 1, Lv = perm[q - 1];
            const double* gw = p.t.gram_w;
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
                phi1[perm[r]] = val;
                if (anti) phi0[perm[r]] = val == 0.0 ? 0.0 : -val;
            }
            sum = wsum(sum);
            if (lane == 0) {
                double last = delta - sum;
                if (fabs(last) < 1e-10) last = 0.0;
                phi1[Lv] = last;
                if (anti) phi0[Lv] = last == 0.0 ? 0.0 : -last;
            }
        }
        __syncwarp();
    }
}

}  // namespace l1
}  // namespace dks
