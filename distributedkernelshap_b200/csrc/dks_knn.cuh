// k-nearest neighbours on the device (DESIGN.md §5.0.15): scikit-learn KNeighborsClassifier.predict_proba and
// KNeighborsRegressor.predict, read into their training rows in the fitted space (KnnDev, dks_set_knn_model).  KernelSHAP
// on a neighbour model needs the real masked forward pass of every (coalition s, background row j): x's value for the
// groups of s that vary, bg_j's for the rest, and its k nearest training rows.
//
// The distance's statistic adds up over columns, as a kernel machine's does (dks_kmach.cuh), so for training row v
//   t(s, j, v) = T[j][v] + sum_{p in s} Delta_j[p][v],   T[j][v] = sum_c h(bg'_j,c - v_c)  (fit time),
//   Delta_j[p][v] = sum_{c in group p} h(x'_c - v_c) - h(bg'_j,c - v_c)                (per instance and row),
// and per (j, tile of training rows) the Delta go into nibble tables: one candidate costs ceil(M / 4) table reads.  What is
// new is the reduction: each (s, j) keeps the k smallest (t, index) over all training rows, then votes or averages.
//
// Rules the NumPy KnnSpec (neighbors.py) restates: rows are ranked by (t, training index); a masked row equal to v column
// for column has t = 0 exactly (decided from equality masks, never from the rounded t), and every other t is at least
// T_FLOOR, so t == 0 is the exactness flag; distance weights give the neighbours at distance 0 weight 1 and the others 0.
#pragma once

#include <climits>

#include "dks_kernels.cuh"

namespace dks {
namespace knn {

constexpr int THREADS = 256;      // = l1::MOM_THREADS: the l1 instantiation forms the moments with block_moments
constexpr int TILE = 32;          // training rows per shared-memory tile
// least t of a training row the row does not equal: a table sum that rounds to 0 or below is not a zero distance, and
// 32 weights 1 / distance(T_FLOOR) still add up to a finite sum for every metric
constexpr double T_FLOOR = 0x1p-1000;

// x'_c: column c of a raw row in the fitted space, rounded as NumPy's x * colw + colo (no fused multiply-add)
__device__ __forceinline__ double knn_col(const KnnDev& k, double x, int c) {
    return __dadd_rn(__dmul_rn(k.colw[c], x), k.colo[c]);
}

// per-column term h(d) of the statistic t
__device__ __forceinline__ double knn_term(const KnnDev& k, double d) {
    if (k.metric == DKS_KNN_METRIC_MANHATTAN) return fabs(d);
    if (k.metric == DKS_KNN_METRIC_MINKOWSKI) return pow(fabs(d), k.p);
    return __dmul_rn(d, d);
}

// the distance of a statistic t >= 0
__device__ __forceinline__ double knn_dist(const KnnDev& k, double t) {
    if (k.metric == DKS_KNN_METRIC_EUCLIDEAN) return sqrt(t);
    if (k.metric == DKS_KNN_METRIC_MINKOWSKI) return pow(t, 1.0 / k.p);
    return t;
}

// (t, v) into the list sorted by (t, index), entries r at lt[r * st] / li[r * st], when it ranks before entry k - 1 (the
// caller has seen t <= that entry's t).  Candidates come in increasing v, so an equal t ranks after every real entry and
// before the empty ones (t = +inf, index INT_MAX).  Returns the new k-th t.
__device__ __forceinline__ double knn_insert(double* lt, int* li, int st, int k, double t, int v) {
    int r = k - 1;
    if (t == lt[(size_t)r * st] && v > li[(size_t)r * st]) return t;
    for (; r > 0; --r) {
        const double u = lt[(size_t)(r - 1) * st];
        if (u < t || (u == t && li[(size_t)(r - 1) * st] < v)) break;
        lt[(size_t)r * st] = u;
        li[(size_t)r * st] = li[(size_t)(r - 1) * st];
    }
    lt[(size_t)r * st] = t;
    li[(size_t)r * st] = v;
    return lt[(size_t)(k - 1) * st];
}

// outputs o[R] of a full neighbour list: the classifier's per-class weight sums in rank order over their sum in class order
// (uniform: count / k), the regressor's rank-order sum of w y over k (uniform) or over the rank-order sum of w
__device__ inline void knn_outputs(const KnnDev& k, const double* lt, const int* li, int st, double* o) {
    const bool dist = k.weights == DKS_KNN_WEIGHTS_DISTANCE;
    bool zero = false;                                  // a neighbour at distance 0: weights 1 there, 0 elsewhere
    if (dist)
        for (int r = 0; r < k.k; ++r) zero |= isinf(1.0 / knn_dist(k, lt[(size_t)r * st]));
    double s[DKS_KNN_MAX_R], den = 0.0;
#pragma unroll
    for (int q = 0; q < DKS_KNN_MAX_R; ++q) s[q] = 0.0;
    for (int r = 0; r < k.k; ++r) {
        double w = 1.0;
        if (dist) {
            w = 1.0 / knn_dist(k, lt[(size_t)r * st]);
            if (zero) w = isinf(w) ? 1.0 : 0.0;
        }
        const int v = li[(size_t)r * st];
        if (k.head == DKS_KNN_HEAD_CLASSIFY) {
            const int lab = (int)k.y[v];
#pragma unroll
            for (int q = 0; q < DKS_KNN_MAX_R; ++q)
                if (q == lab) s[q] += w;
        } else {
#pragma unroll
            for (int q = 0; q < DKS_KNN_MAX_R; ++q)
                if (q < k.R) s[q] += __dmul_rn(k.y[(size_t)v * k.R + q], w);
            den += w;
        }
    }
    if (!dist) {
        den = (double)k.k;                              // uniform: scikit-learn's normaliser, the sum of k ones
    } else if (k.head == DKS_KNN_HEAD_CLASSIFY) {
        den = 0.0;
        for (int q = 0; q < k.R; ++q) den += s[q];
    }
    for (int q = 0; q < k.R; ++q) o[q] = s[q] / den;
}

// f(X) [n][C] (dks_predict_host, the background at fit time) and, with dlink, link(f(x)) - link(fnull) for stage 1.  A row
// holding NaN or an infinity is reported as DKS_ERR_DOMAIN with the row (scikit-learn refuses it) and its outputs are NaN;
// a non-finite link(f(x)) is reported as DKS_ERR_NUMERIC with the instance.
__global__ void knn_predict_kernel(const double* __restrict__ X, int n, int D, KnnDev k, int C, int link,
                                   const double* __restrict__ linkfnull, double* __restrict__ out, double* __restrict__ dlink,
                                   int* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* x = X + (size_t)i * D;
    bool refused = false;
    for (int c = 0; c < D; ++c) refused |= !isfinite(x[c]);
    double o[DKS_KNN_MAX_R];
    if (refused) {
        for (int c = 0; c < C; ++c) o[c] = NAN;
        if (status) report_status(status, DKS_ERR_DOMAIN, i);
    } else {
        double lt[DKS_KNN_MAX_K];
        int li[DKS_KNN_MAX_K];
        for (int r = 0; r < k.k; ++r) { lt[r] = INFINITY; li[r] = INT_MAX; }
        double kt = INFINITY;
        for (int v = 0; v < k.n_fit; ++v) {
            const double* fv = k.fitX + (size_t)v * D;
            double t = 0.0;
            bool exact = true;
            for (int c = 0; c < D; ++c) {
                const double d = knn_col(k, x[c], c) - fv[c];
                t += knn_term(k, d);
                exact &= d == 0.0;
            }
            t = exact ? 0.0 : fmax(t, T_FLOOR);
            if (t <= kt) kt = knn_insert(lt, li, 1, k.k, t, v);
        }
        knn_outputs(k, lt, li, 1, o);
    }
    predict_epilogue(o, C, i, link, linkfnull, out, dlink, status, refused);
}

// fit: T[j][v] = sum_c h(bg'_j,c - v_c), columns in order, and E[j][v] = the groups (bit g) on which bg'_j equals v exactly
__global__ void knn_fit_table_kernel(const double* __restrict__ bg, int N, int D, int G, KnnDev k, double* __restrict__ Tbg,
                                     uint64_t* __restrict__ Ebg) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * k.n_fit) return;
    const int j = (int)(idx / k.n_fit), v = (int)(idx - (long long)j * k.n_fit);
    const double* b = bg + (size_t)j * D;
    const double* fv = k.fitX + (size_t)v * D;
    double t = 0.0;
    uint64_t eq = G == 64 ? ~0ull : (1ull << G) - 1;
    for (int c = 0; c < D; ++c) {
        const double d = knn_col(k, b[c], c) - fv[c];
        t += knn_term(k, d);
        if (d != 0.0) eq &= ~(1ull << k.colgrp[c]);
    }
    Tbg[idx] = t;
    Ebg[idx] = eq;
}

// doubles of the per-tile tables: T_j [TILE], Delta [G][TILE], nibble tables [ceil(G/4)][TILE][16], the equality masks
// [2][TILE] and x's per-group equality bytes [G][TILE]
__host__ __device__ inline size_t tile_doubles(int G) {
    return (size_t)TILE * (1 + G + 16 * ((G + 3) / 4) + 2) + ((size_t)G * TILE + 7) / 8;
}

// shared memory of explain_knn_kernel: [C][S_cap] float64 sums / y, one region the background loop holds a tile's tables in
// and the solve the normal matrix [63 * 63] and rhs [64], the neighbour lists of a chunk of coalitions ([k][chunk] t, then
// [k][chunk] indices) and the varying groups [64]
__host__ __device__ inline size_t smem_bytes(int S_cap, int C, int G, int k, int chunk) {
    const size_t tab = tile_doubles(G), solve = 63 * 63 + 64;
    return sizeof(double) * ((size_t)C * S_cap + (tab > solve ? tab : solve) + (size_t)k * chunk) +
           sizeof(int) * ((size_t)k * chunk + 64);
}

// One CTA per instance (grid-stride), any plan source (shared, per-instance, caller-supplied), up to 64 groups.  The
// coalitions go in chunks of at most `chunk` (the neighbour lists of a chunk fit shared memory); per chunk, background row j
// (zero-weight rows skipped) and tile of TILE training rows:
//   1. threads over (varying position p, v) form Delta_j[p][v] and whether x' equals v on the group, then the nibble
//      tables tb[q][v][pat] and per v the equality masks over the varying positions (mx: x equals v, mb: bg_j does; both 0
//      when no masked row can equal v);
//   2. threads over coalitions read t = T[j][v] + sum_q tb[q][v][z's nibble q] (0 when (z & mx) | (~z & mb) covers every
//      varying position), reject it with one compare against the list's k-th t, and otherwise insert it.
// After the last tile the list's outputs, times w_j, go into the coalition's sums.  Each coalition belongs to one thread
// throughout and every sum runs in a fixed order: the result does not depend on the grid or the chunk size.  Then
// y = link(ey) - link(fnull) for every output (each solved on its own) and the CUDA-core kernel's constrained WLS, or (L1)
// the moments of y for l1_lars_kernel.  A non-finite y or f(x) is reported as DKS_ERR_NUMERIC and nothing of the instance
// is written.
// ACC (a soft-voting ensemble's member): the sums of every output go into ea.ey instead (ens_accumulate); instances
// with M <= 1 or a refused f(x) are left to explain_ensemble_tail_kernel.
template <bool L1, bool ACC = false>
__global__ void __launch_bounds__(THREADS) explain_knn_kernel(ExplainParams p, SimtL1 q, KnnDev k, int chunk,
                                                              const double* __restrict__ X, const double* __restrict__ bg,
                                                              int D, const int* __restrict__ goff,
                                                              const int* __restrict__ gcols, EnsAcc ea) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x;
    const int N = p.N, G = p.G, C = p.C, K = k.k;
    double* acc = reinterpret_cast<double*>(smem_raw);          // [C][S_cap]
    double* region = acc + (size_t)C * p.S_cap;
    const size_t tab = tile_doubles(G), solve = 63 * 63 + 64;
    double* A = region;                                         // [63 * 63] (solve)
    double* rhs = A + 63 * 63;                                  // [64]
    double* tj = region;                                        // [TILE] (background loop)
    double* dl = tj + TILE;                                     // [G][TILE]
    double* tb = dl + (size_t)G * TILE;                         // [ceil(G/4)][TILE][16]
    uint64_t* em = reinterpret_cast<uint64_t*>(tb + (size_t)16 * TILE * ((G + 3) / 4));   // [2][TILE] mx, mb
    unsigned char* eqx = reinterpret_cast<unsigned char*>(em + 2 * TILE);                // [G][TILE]
    double* lt = region + (tab > solve ? tab : solve);          // [K][chunk]
    int* li = reinterpret_cast<int*>(lt + (size_t)K * chunk);   // [K][chunk]
    int* vi = li + (size_t)K * chunk;                           // [64]
    const size_t slab = (size_t)p.n * G;

    const int ninst = dks_inst_count(p);
    for (int qi = blockIdx.x; qi < ninst; qi += gridDim.x) {
        const int i = dks_inst_at(p, qi);
        const int M = p.Mcnt[i];
        const uint64_t vm = p.vmask[i];
        __syncthreads();  // previous instance done with shared memory
        if constexpr (!ACC) zero_phi_rows(p, i);
        bool fx_bad = false;                                    // stage 1 reported a refused row or a non-finite link(f(x))
        for (int c = 0; c < C; ++c) fx_bad |= !isfinite(p.dlink[(size_t)i * C + c]);
        if (M == 0) continue;
        if (M == 1) {
            // the one varying group takes link(f(x)) - link(fnull) of every output
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
        const uint64_t gall = G == 64 ? ~0ull : (1ull << G) - 1;
        const uint64_t full = M == 64 ? ~0ull : (1ull << M) - 1;
        // groups that do not vary: every masked row takes bg_j's values there, so a row reproduces v only where bg_j does
        const uint64_t fixed = gall & ~vm;
        for (int c0 = 0; c0 < S; c0 += chunk) {
            const int nc = min(chunk, S - c0);
            for (int j = 0; j < N; ++j) {
                const double wj = p.wbg[j];
                if (wj == 0.0) continue;                        // block-uniform
                const double* b = bg + (size_t)j * D;
                for (int s = tid; s < nc; s += blockDim.x)
                    for (int r = 0; r < K; ++r) {
                        lt[(size_t)r * chunk + s] = INFINITY;
                        li[(size_t)r * chunk + s] = INT_MAX;
                    }
                for (int v0 = 0; v0 < k.n_fit; v0 += TILE) {
                    const int nv = min(TILE, k.n_fit - v0);
                    for (int idx = tid; idx < nv; idx += blockDim.x) tj[idx] = k.Tbg[(size_t)j * k.n_fit + v0 + idx];
                    for (int idx = tid; idx < M * nv; idx += blockDim.x) {
                        const int pp = idx / nv, v = idx - pp * nv, g = vi[pp];
                        const double* fv = k.fitX + (size_t)(v0 + v) * D;
                        double d = 0.0;
                        bool eq = true;
                        for (int e = goff[g]; e < goff[g + 1]; ++e) {
                            const int c = gcols[e];
                            const double dx = knn_col(k, x[c], c) - fv[c];
                            d += knn_term(k, dx) - knn_term(k, knn_col(k, b[c], c) - fv[c]);
                            eq &= dx == 0.0;
                        }
                        dl[(size_t)pp * TILE + v] = d;
                        eqx[(size_t)pp * TILE + v] = eq;
                    }
                    __syncthreads();
                    for (int idx = tid; idx < nib * nv * 16; idx += blockDim.x) {
                        const int qn = idx / (nv * 16), rem = idx - qn * nv * 16, v = rem >> 4, pat = rem & 15;
                        double t = 0.0;
                        for (int bit = 0; bit < 4; ++bit)
                            if (((pat >> bit) & 1) && 4 * qn + bit < M) t += dl[(size_t)(4 * qn + bit) * TILE + v];
                        tb[((size_t)qn * TILE + v) * 16 + pat] = t;
                    }
                    int possible = 0;
                    for (int v = tid; v < nv; v += blockDim.x) {
                        const uint64_t e = k.Ebg[(size_t)j * k.n_fit + v0 + v];
                        uint64_t mx = 0, mb = 0;
                        for (int pp = 0; pp < M; ++pp) {
                            if (eqx[(size_t)pp * TILE + v]) mx |= 1ull << pp;
                            if ((e >> vi[pp]) & 1ull) mb |= 1ull << pp;
                        }
                        const bool can = (e & fixed) == fixed && ((mx | mb) & full) == full;
                        em[v] = can ? mx : 0;
                        em[TILE + v] = can ? mb : 0;
                        possible |= can;
                    }
                    const bool any_exact = __syncthreads_or(possible);
                    for (int s = tid; s < nc; s += blockDim.x) {
                        const uint64_t z = zp[c0 + s];
                        double* ls = lt + s;
                        int* is = li + s;
                        double kt = ls[(size_t)(K - 1) * chunk];
                        for (int v = 0; v < nv; ++v) {
                            double t = tj[v];
                            for (int qn = 0; qn < nib; ++qn) t += tb[((size_t)qn * TILE + v) * 16 + ((z >> (4 * qn)) & 15)];
                            t = fmax(t, T_FLOOR);
                            if (any_exact && (((z & em[v]) | (~z & em[TILE + v])) & full) == full) t = 0.0;
                            if (t > kt) continue;
                            kt = knn_insert(ls, is, chunk, K, t, v0 + v);
                        }
                    }
                    __syncthreads();
                }
                // the lists are complete: their outputs, times w_j, into the sums
                for (int s = tid; s < nc; s += blockDim.x) {
                    double o[DKS_KNN_MAX_R];
                    knn_outputs(k, lt + s, li + s, chunk, o);
                    for (int c = 0; c < C; ++c)
                        acc[(size_t)c * p.S_cap + c0 + s] = fma(wj, o[c], acc[(size_t)c * p.S_cap + c0 + s]);
                }
            }
        }
        __syncthreads();
        if constexpr (ACC) {
            ens_accumulate(ea, p, i, S, acc);
            continue;
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

}  // namespace knn
}  // namespace dks
