// Tree ensembles on the device (DESIGN.md §5.0.11, §5.0.18): scikit-learn decision trees, random / extra-trees forests,
// gradient boosting, SAMME AdaBoost and isolation forests, read into flat node arrays (TreeDev, dks_set_tree_model).  KernelSHAP on a tree needs the real masked forward
// pass of every (coalition s, background row j): x's value for the groups of s that vary, bg_j's for the rest.  A tree walk
// is a few dependent loads and a compare per level, so this route evaluates all S N of them per instance, in float64.
//
// The reduction that makes it cheap: above the first node where x and bg_j go different ways (on a varying group) the walk
// does not depend on s.  Per (instance, j) one pass over the trees finds that node; trees where x and bg_j agree all the way
// down add their leaf to a per-j constant, and only the others are walked per coalition, from that node.
#pragma once

#include "dks_kernels.cuh"

namespace dks {
namespace trees {

constexpr int THREADS = 256;      // = l1::MOM_THREADS: the l1 instantiation forms the moments with block_moments
constexpr unsigned char NO_POS = 127;

// x <= thr (the float32 cast first under DKS_TREE_CMP_F32); NaN goes where the node says
__device__ __forceinline__ bool goes_left(double x, double thr, unsigned char miss, int cmp) {
    if (isnan(x)) return miss != 0;
    const double v = cmp == DKS_TREE_CMP_F32 ? (double)(float)x : x;
    return v <= thr;
}

// outputs of the head on the raw scores r[R], float64 (C = 2 for the sigmoid head, else R); offset: the anomaly head's
__device__ __forceinline__ void tree_head(const double* r, int R, int head, double offset, double* o) {
    if (head == DKS_TREE_HEAD_SIGMOID) {
        // [1 - expit(r), expit(r)] with neither half formed by cancellation
        const double e = exp(-fabs(r[0]));
        const double big = 1.0 / (1.0 + e), small = e / (1.0 + e);
        o[1] = r[0] >= 0 ? big : small;
        o[0] = r[0] >= 0 ? small : big;
    } else if (head == DKS_TREE_HEAD_SOFTMAX) {
        double m = r[0];
        for (int q = 1; q < R; ++q) m = fmax(m, r[q]);
        double sum = 0;
        for (int q = 0; q < R; ++q) { o[q] = exp(r[q] - m); sum += o[q]; }
        for (int q = 0; q < R; ++q) o[q] /= sum;
    } else if (head == DKS_TREE_HEAD_EXP) {
        o[0] = exp(r[0]);
    } else if (head == DKS_TREE_HEAD_IFOREST) {
        // IsolationForest: r = -(sum of the path lengths) / (T c(max_samples)), the score is -2^r
        o[0] = -exp2(r[0]) - offset;
    } else {
        for (int q = 0; q < R; ++q) o[q] = r[q];
    }
}

// raw scores of one row: base + every tree's leaf, trees in order
__device__ inline void tree_raw(const TreeDev& t, const double* __restrict__ x, double* r) {
    for (int q = 0; q < t.R; ++q) r[q] = t.base[q];
    for (int k = 0; k < t.T; ++k) {
        int nd = t.roots[k];
        for (int f = t.feat[nd]; f >= 0; f = t.feat[nd])
            nd = goes_left(x[f], t.thr[nd], t.miss[nd], t.cmp) ? t.left[nd] : t.right[nd];
        for (int q = 0; q < t.R; ++q) r[q] += t.val[(size_t)nd * t.R + q];
    }
}

// f(X) [n][C] (dks_predict_host, the background at fit time) and, with dlink, link(f(x)) - link(fnull) for stage 1.  A
// non-finite link(f(x)) is reported as DKS_ERR_NUMERIC with the instance.
__global__ void tree_predict_kernel(const double* __restrict__ X, int n, int D, TreeDev t, int C, int link,
                                    const double* __restrict__ linkfnull, double* __restrict__ out, double* __restrict__ dlink,
                                    int* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double r[DKS_TREE_MAX_R], o[DKS_TREE_MAX_R];
    tree_raw(t, X + (size_t)i * D, r);
    tree_head(r, t.R, t.head, t.offset, o);
    predict_epilogue(o, C, i, link, linkfnull, out, dlink, status, false);
}

// fit: every background row's direction at every internal node, bgdir[j][node]
__global__ void tree_bgdir_kernel(const double* __restrict__ bg, int N, int D, TreeDev t, unsigned char* __restrict__ bgdir) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * t.nodes) return;
    const int j = (int)(idx / t.nodes), nd = (int)(idx - (long long)j * t.nodes);
    const int f = t.feat[nd];
    bgdir[idx] = f >= 0 && goes_left(bg[(size_t)j * D + f], t.thr[nd], t.miss[nd], t.cmp) ? 1 : 0;
}

// shared memory of explain_tree_kernel: [C][S_cap] float64 sums / y, the normal matrix, rhs, per-thread constants
// [THREADS][R], the per-j constant [8], the divergent trees of one background row [T], warp counts [8] and the varying
// groups [64]
__host__ __device__ inline size_t smem_bytes(int S_cap, int C, int R, int T) {
    return sizeof(double) * ((size_t)C * S_cap + 63 * 63 + 64 + (size_t)THREADS * R + 8) + sizeof(int) * ((size_t)T + 8 + 64);
}

// One CTA per instance (grid-stride), any plan source (shared, per-instance, caller-supplied).  Background rows are the outer
// loop; per row j:
//   1. threads over trees walk x and bg_j together from the root -- bg_j's way at nodes whose group does not vary (upstream
//      keeps the background value there), else both ways -- to the first node where they part.  A tree with no such node adds
//      its leaf to the constant of j; the others go, in tree order, into the list of divergent trees with that node;
//   2. threads over coalitions walk each divergent tree from its node, taking x's way where the node's group is in s and
//      bg_j's way elsewhere, add the constant, apply the head and accumulate w_j head(r) into the row's float64 sums.
// Every sum runs in a fixed order: the result does not depend on the grid.  Then y = link(ey) - link(fnull) per solved output
// (two outputs: class 1, class 0 its negation), and the CUDA-core kernel's constrained WLS, or (L1) the moments of y for
// l1_lars_kernel.  A non-finite y or f(x) is reported as DKS_ERR_NUMERIC and nothing of the instance is written.  ACC (a
// soft-voting ensemble's member): the sums of every output go into ea.ey instead (ens_accumulate); instances with M <= 1
// or a refused f(x) are left to explain_ensemble_tail_kernel.
template <bool L1, bool ACC = false>
__global__ void __launch_bounds__(THREADS) explain_tree_kernel(ExplainParams p, SimtL1 q, TreeDev t, const double* __restrict__ X,
                                                               int D, EnsAcc ea) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int N = p.N, G = p.G, C = p.C, R = t.R, T = t.T, nodes = t.nodes;
    double* acc = reinterpret_cast<double*>(smem_raw);          // [C][S_cap]
    double* A = acc + (size_t)C * p.S_cap;                      // [63 * 63]
    double* rhs = A + 63 * 63;                                  // [64]
    double* cpart = rhs + 64;                                   // [THREADS][R]
    double* cj = cpart + (size_t)THREADS * R;                   // [8]
    int* dlist = reinterpret_cast<int*>(cj + 8);                // [T]
    int* wcnt = dlist + T;                                      // [8]
    int* vi = wcnt + 8;                                         // [64]
    const size_t slab = (size_t)p.n * G;
    const int nsolve = C == 2 ? 1 : C;                          // two outputs: class 0 is the negation of class 1
    unsigned char* xi = t.xinfo + (size_t)blockIdx.x * nodes;

    const int ninst = dks_inst_count(p);
    for (int qi = blockIdx.x; qi < ninst; qi += gridDim.x) {
        const int i = dks_inst_at(p, qi);
        const int M = p.Mcnt[i];
        const uint64_t vm = p.vmask[i];
        __syncthreads();  // previous instance done with shared memory and xi
        if constexpr (!ACC) zero_phi_rows(p, i);
        bool fx_bad = false;                                    // stage 1 reported a non-finite link(f(x))
        for (int c = 0; c < C; ++c) fx_bad |= !isfinite(p.dlink[(size_t)i * C + c]);
        if (M == 0) continue;
        if (M == 1) {
            // the one varying group takes link(f(x)) - link(fnull); two outputs: class 0 is the negation of class 1, as below
            if (!ACC && tid < C && !fx_bad) {
                const double v = p.dlink[(size_t)i * C + (C == 2 ? 1 : tid)];
                p.phi[(size_t)tid * slab + (size_t)i * G + (__ffsll((long long)vm) - 1)] =
                    (C == 2 && tid == 0) ? ((v == 0.0) ? 0.0 : -v) : v;
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
        // x's way at every internal node and the coalition bit of its group (NO_POS: the group does not vary)
        for (int nd = tid; nd < nodes; nd += blockDim.x) {
            const int f = t.feat[nd];
            unsigned char info = NO_POS;
            if (f >= 0) {
                const int g = t.colgrp[f];
                const unsigned char pos = ((vm >> g) & 1ull) ? (unsigned char)__popcll(vm & ((1ull << g) - 1ull)) : NO_POS;
                info = (unsigned char)((goes_left(X[(size_t)i * D + f], t.thr[nd], t.miss[nd], t.cmp) ? 0x80 : 0) | pos);
            }
            xi[nd] = info;
        }
        for (int idx = tid; idx < C * S; idx += blockDim.x) acc[(size_t)(idx / S) * p.S_cap + idx % S] = 0.0;
        __syncthreads();

        for (int j = 0; j < N; ++j) {
            const double wj = p.wbg[j];
            if (wj == 0.0) continue;                            // block-uniform
            const unsigned char* bd = t.bgdir + (size_t)j * nodes;
            double cl[DKS_TREE_MAX_R];
            for (int u = 0; u < R; ++u) cl[u] = 0.0;
            int ndiv = 0;
            for (int t0 = 0; t0 < T; t0 += blockDim.x) {
                const int k = t0 + tid;
                int dn = -1;
                if (k < T) {
                    int nd = t.roots[k];
                    while (t.feat[nd] >= 0) {
                        const unsigned char info = xi[nd], b = bd[nd];
                        if ((info & 0x7f) != NO_POS && (info >> 7) != b) { dn = nd; break; }
                        nd = b ? t.left[nd] : t.right[nd];
                    }
                    if (dn < 0)
                        for (int u = 0; u < R; ++u) cl[u] += t.val[(size_t)nd * R + u];
                }
                // the divergent trees of this chunk, appended in tree order
                const unsigned bal = __ballot_sync(0xffffffffu, dn >= 0);
                if (lane == 0) wcnt[warp] = __popc(bal);
                __syncthreads();
                int off = ndiv, total = 0;
                for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { if (w < warp) off += wcnt[w]; total += wcnt[w]; }
                if (dn >= 0) dlist[off + __popc(bal & ((1u << lane) - 1u))] = dn;
                ndiv += total;
                __syncthreads();
            }
            for (int u = 0; u < R; ++u) cpart[(size_t)tid * R + u] = cl[u];
            __syncthreads();
            if (tid < R) {
                double s = t.base[tid];
                for (int k = 0; k < (int)blockDim.x; ++k) s += cpart[(size_t)k * R + tid];
                cj[tid] = s;
            }
            __syncthreads();
            for (int s = tid; s < S; s += blockDim.x) {
                const uint64_t z = zp[s];
                double r[DKS_TREE_MAX_R], o[DKS_TREE_MAX_R];
                for (int u = 0; u < R; ++u) r[u] = cj[u];
                for (int e = 0; e < ndiv; ++e) {
                    int nd = dlist[e];
                    while (t.feat[nd] >= 0) {
                        const unsigned char info = xi[nd], pos = info & 0x7f;
                        const bool lft = (pos != NO_POS && ((z >> pos) & 1ull)) ? (info >> 7) != 0 : bd[nd] != 0;
                        nd = lft ? t.left[nd] : t.right[nd];
                    }
                    for (int u = 0; u < R; ++u) r[u] += t.val[(size_t)nd * R + u];
                }
                tree_head(r, R, t.head, t.offset, o);
                for (int c = 0; c < C; ++c) acc[(size_t)c * p.S_cap + s] = fma(wj, o[c], acc[(size_t)c * p.S_cap + s]);
            }
            __syncthreads();
        }
        if constexpr (ACC) {
            ens_accumulate(ea, p, i, S, acc);
            continue;
        }

        // y = link(ey) - link(fnull) per solved output, written over the sums (row u of acc); the logit's 1 - ey is the sum
        // of the other outputs when there are several (no cancellation)
        int bad = 0;
        for (int s = tid; s < S; s += blockDim.x) {
            double e[DKS_TREE_MAX_R], y[DKS_TREE_MAX_R];
            for (int c = 0; c < C; ++c) e[c] = acc[(size_t)c * p.S_cap + s];
            for (int u = 0; u < nsolve; ++u) {
                const int c = C == 2 ? 1 : u;
                if (p.link == DKS_LINK_LOGIT) {
                    double rest = 0.0;
                    if (C == 1) rest = 1.0 - e[0];
                    else for (int c2 = 0; c2 < C; ++c2) if (c2 != c) rest += e[c2];
                    y[u] = log(e[c] / rest) - p.linkfnull[c];
                } else {
                    y[u] = e[c] - p.fnull[c];
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
        for (int u = 0; u < nsolve; ++u) {
            const int c = C == 2 ? 1 : u;
            __syncthreads();
            block_solve_one(pl, M, acc + (size_t)u * p.S_cap, p.dlink[(size_t)i * C + c], A, rhs, vi,
                            p.phi + (size_t)c * slab + (size_t)i * G);
        }
        if (C == 2 && tid == 0) write_class0_negation(p.phi + (size_t)i * G, p.phi + slab + (size_t)i * G, M, vi);
    }
}

}  // namespace trees
}  // namespace dks
