// Multi-layer perceptrons on the device (DESIGN.md §5.0.14): scikit-learn MLPClassifier.predict_proba and
// MLPRegressor.predict with 1 to 4 hidden layers, read into float64 layers in raw feature space (MlpDev, dks_set_mlp).
// KernelSHAP on an MLP needs the real masked forward pass of every (coalition s, background row j): x's value for the groups
// of s that vary, bg_j's for the rest.
//
// The reduction that makes it cheap: layer 1's pre-activation adds up over columns, so
//   a1(s, j) = B[j] + sum_{p in s} Delta_j[p],   B[j] = b_0 + bg_j W_0                       (fit time, [N][H1]),
//   Delta_j[p][h] = sum_{c in group p} W_0[c][h] (x_c - bg_j,c)                               (per instance and row).
// Over a tile of 16 coalitions layer 1 is the product of the 0/1 coalition matrix Z [16 x M, M padded to 16] and Delta_j
// [M x H1], plus B[j]; layers 2 .. L are ordinary products [16 x H_{l-1}] [H_{l-1} x H_l].  Every product runs on the FP64
// tensor cores (mma.sync m16n8k16 .f64, SASS DMMA.16x8x16; wgmma has no f64 type).
#pragma once

#include "dks_kernels.cuh"

namespace dks {
namespace mlp {

constexpr int THREADS = 256;      // = l1::MOM_THREADS: the l1 instantiation forms the moments with block_moments
constexpr int WARPS = THREADS / 32;
constexpr int NTC = 4;            // n-tiles (8 units each) one accumulator chunk holds

__device__ __forceinline__ double act_f(int act, double v) {
    if (act == DKS_MLP_ACT_LOGISTIC) return 1.0 / (1.0 + exp(-v));
    if (act == DKS_MLP_ACT_TANH) return tanh(v);
    if (act == DKS_MLP_ACT_RELU) return v > 0.0 ? v : 0.0;
    return v;
}

// outputs o[C] of the head on the output layer's values z[R]; the sigmoid head's two halves are neither formed by
// cancellation (class 0 is exp(-|z|) / (1 + exp(-|z|)) where z >= 0), the softmax subtracts the maximum as scikit-learn does
__device__ __forceinline__ void mlp_head(int head, const double* z, int R, double* o) {
    if (head == DKS_MLP_HEAD_SIGMOID) {
        const double e = exp(-fabs(z[0]));
        const double big = 1.0 / (1.0 + e), small = e / (1.0 + e);
        o[1] = z[0] >= 0 ? big : small;
        o[0] = z[0] >= 0 ? small : big;
    } else if (head == DKS_MLP_HEAD_SOFTMAX) {
        double mx = z[0];
        for (int q = 1; q < R; ++q) mx = fmax(mx, z[q]);
        double sum = 0.0;
        for (int q = 0; q < R; ++q) { o[q] = exp(z[q] - mx); sum += o[q]; }
        for (int q = 0; q < R; ++q) o[q] /= sum;
    } else {
        for (int q = 0; q < R; ++q) o[q] = z[q];
    }
}

// f(X) [n][C] (dks_predict_host, the background at fit time) and, with dlink, link(f(x)) - link(fnull) for stage 1: one CTA
// per row (grid-stride), thread u computes unit u of each layer with its inputs summed in order.  A row holding NaN or an
// infinity is reported as DKS_ERR_DOMAIN with the row (scikit-learn refuses it) and its outputs are NaN; a non-finite
// link(f(x)) is reported as DKS_ERR_NUMERIC with the instance.
__global__ void __launch_bounds__(THREADS) mlp_predict_kernel(const double* __restrict__ X, int n, int D, MlpDev m, int C,
                                                              int link, const double* __restrict__ linkfnull,
                                                              double* __restrict__ out, double* __restrict__ dlink,
                                                              int* __restrict__ status) {
    __shared__ double h[2][DKS_MLP_MAX_WIDTH];
    __shared__ double z[DKS_MLP_MAX_OUT];
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const double* x = X + (size_t)i * D;
        bool bad = false;
        for (int c = threadIdx.x; c < D; c += blockDim.x) bad |= !isfinite(x[c]);
        const bool refused = __syncthreads_or(bad);      // also: the previous row is done with h and z
        if (!refused) {
            const double* in = x;
            for (int l = 0; l < m.L; ++l) {
                const int K = m.width[l], H = m.width[l + 1];
                const bool last = l == m.L - 1;
                double* dst = last ? z : h[l & 1];
                const double* W = m.W + m.woff[l];
                for (int u = threadIdx.x; u < H; u += blockDim.x) {
                    double t = m.b[m.boff[l] + u];
                    for (int k = 0; k < K; ++k) t = fma(in[k], W[(size_t)k * H + u], t);
                    dst[u] = last ? t : act_f(m.act, t);
                }
                __syncthreads();
                in = dst;
            }
        }
        if (threadIdx.x == 0) {
            double o[DKS_MLP_MAX_OUT];
            if (refused) {
                for (int c = 0; c < C; ++c) o[c] = NAN;
                if (status) report_status(status, DKS_ERR_DOMAIN, i);
            } else {
                mlp_head(m.head, z, m.R, o);
            }
            predict_epilogue(o, C, i, link, linkfnull, out, dlink, status, refused);
        }
    }
}

// fit: B[j][h] = b_0[h] + sum_c bg_j,c W_0[c][h], columns in order
__global__ void mlp_fit_table_kernel(const double* __restrict__ bg, int N, int D, MlpDev m, double* __restrict__ Bbg) {
    const int H1 = m.width[1];
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * H1) return;
    const int j = (int)(idx / H1), h = (int)(idx - (long long)j * H1);
    const double* b = bg + (size_t)j * D;
    double t = m.b[h];
    for (int c = 0; c < D; ++c) t = fma(b[c], m.W[(size_t)c * H1 + h], t);
    Bbg[idx] = t;
}

// D += A B on the FP64 tensor cores, one 16 x 8 x 16 step.  Lane (g = lane / 4, t = lane % 4) holds
//   A (16 x 16, row-major): a[i] at row g + 8 (i % 2), column t + 4 (i / 2);
//   B (16 x 8, column-major): b[i] at row t + 4 i, column g;
//   C / D (16 x 8): c[i] at row g + 8 (i / 2), column 2 t + i % 2.
__device__ __forceinline__ void dmma(double (&c)[4], const double (&a)[8], const double2 b01, const double2 b23) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7, %8, %9, %10, %11}, "
        "{%12, %13, %14, %15}, {%0, %1, %2, %3};\n"
        : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b01.x), "d"(b01.y),
          "d"(b23.x), "d"(b23.y));
}

__host__ __device__ inline int pad16(int v) { return (v + 15) & ~15; }

// doubles of one warp's region: nbuf activation buffers [16][hmax] (A-fragment order) and the output layer's [16][8]
__host__ __device__ inline size_t warp_doubles(const MlpDev& m) { return (size_t)16 * ((size_t)m.nbuf * m.hmax + 8); }

// doubles of the region the background loop holds -- Delta_j [pad16(G)][pad[1]] in B-fragment order, B[j] [pad[1]] and nw
// warps' regions -- and the solve the normal matrix [63 * 63] and rhs [64] in
__host__ __device__ inline size_t region_doubles(int G, const MlpDev& m, int nw) {
    const size_t loop = (size_t)pad16(G) * m.pad[1] + m.pad[1] + (size_t)nw * warp_doubles(m), solve = 63 * 63 + 64;
    return loop > solve ? loop : solve;
}

// shared memory of explain_mlp_kernel with nw warps evaluating coalitions: [C][S_cap] float64 sums / y (rounded up to an even
// count: the warps' buffers are read as double2), the region, and the varying groups [64]
__host__ __device__ inline size_t smem_bytes(int S_cap, int C, int G, const MlpDev& m, int nw) {
    return sizeof(double) * ((((size_t)C * S_cap + 1) & ~(size_t)1) + region_doubles(G, m, nw)) + sizeof(int) * 64;
}

// the column pair (c[2k], c[2k + 1]) of rows (g, g + 8) -> the A-fragment slot of unit col of a [16][K] buffer: double2
// (kc * 4 + i) * 32 + lane' holds a[2 i], a[2 i + 1] of lane' = g * 4 + (col % 16) % 4 in k-chunk kc = col / 16
__device__ __forceinline__ void store_pair(double2* buf, int col, int g, double lo, double hi) {
    const int kk = col & 15;
    buf[((col >> 4) * 4 + (kk >> 2)) * 32 + g * 4 + (kk & 3)] = make_double2(lo, hi);
}

// the 16 coalition rows zg (row g) and zh (row g + 8) of one warp through every layer; returns the output layer's values in
// lg [16][8].  Layer 1: A from the coalition bits, B = Delta_j (shared), accumulators start at B[j]; hidden layers: A from
// the warp's buffer, B = the layer's fragment-ordered weights (global, L1/L2-resident), accumulators start at the biases.
__device__ __forceinline__ void forward_tile(const MlpDev& m, int KC1, uint64_t zg, uint64_t zh, const double* dl,
                                             const double* bj, double2* buf0, double2* buf1, double* lg) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    for (int l = 0; l < m.L; ++l) {
        const int NT = m.pad[l + 1] >> 3, KC = l == 0 ? KC1 : m.pad[l] >> 4;
        const double2* in = (l & 1) ? buf0 : buf1;          // layer l >= 1 reads what layer l - 1 wrote
        double2* outb = (l & 1) ? buf1 : buf0;
        const double* bias = l == 0 ? bj : m.bp + m.bpoff[l];
        const double* Bf = l == 0 ? dl : m.Wf + m.wfoff[l];
        const bool last = l == m.L - 1;
        for (int nt0 = 0; nt0 < NT; nt0 += NTC) {
            double c[NTC][4];
#pragma unroll
            for (int u = 0; u < NTC; ++u) {
                const int col = (nt0 + u) * 8 + 2 * t;
                const bool on = nt0 + u < NT;
                c[u][0] = c[u][2] = on ? bias[col] : 0.0;
                c[u][1] = c[u][3] = on ? bias[col + 1] : 0.0;
            }
            for (int kc = 0; kc < KC; ++kc) {
                double a[8];
                if (l == 0) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int k = kc * 16 + t + 4 * i;
                        a[2 * i] = ((zg >> k) & 1ull) ? 1.0 : 0.0;
                        a[2 * i + 1] = ((zh >> k) & 1ull) ? 1.0 : 0.0;
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const double2 v = in[(kc * 4 + i) * 32 + lane];
                        a[2 * i] = v.x;
                        a[2 * i + 1] = v.y;
                    }
                }
#pragma unroll
                for (int u = 0; u < NTC; ++u) {
                    if (nt0 + u < NT) {
                        const double2* bf = reinterpret_cast<const double2*>(Bf + (((size_t)kc * NT + nt0 + u) * 32 + lane) * 4);
                        dmma(c[u], a, bf[0], bf[1]);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < NTC; ++u) {
                if (nt0 + u >= NT) continue;
                const int col = (nt0 + u) * 8 + 2 * t;
                if (last) {
                    lg[g * 8 + col] = c[u][0];
                    lg[g * 8 + col + 1] = c[u][1];
                    lg[(g + 8) * 8 + col] = c[u][2];
                    lg[(g + 8) * 8 + col + 1] = c[u][3];
                } else {
                    store_pair(outb, col, g, act_f(m.act, c[u][0]), act_f(m.act, c[u][2]));
                    store_pair(outb, col + 1, g, act_f(m.act, c[u][1]), act_f(m.act, c[u][3]));
                }
            }
        }
        __syncwarp();
    }
}

// One CTA per instance (grid-stride), any plan source (shared, per-instance, caller-supplied), up to 64 groups.  Background
// rows are the outer loop (zero-weight rows skipped); per row j:
//   1. every thread forms Delta_j in B-fragment order (positions padded to 16 and units to pad[1] with zeros) and B[j];
//   2. warps 0 .. nw - 1 take tiles of 16 coalitions in turn (warp w: rows 16 w, 16 (w + nw), ...) through every layer on
//      the tensor cores, in their own buffers, then lanes 0 .. 15 apply the head to one row each and add w_j head(z) to the
//      coalition's sums.
// A coalition's sums are added to in background-row order by the one lane that owns its row, and its forward pass does not
// depend on the other rows of its tile: the result depends neither on the grid nor on nw.  Then y = link(ey) - link(fnull)
// per solved output (sigmoid head: class 1, class 0 its negation) and the CUDA-core kernel's constrained WLS, or (L1) the
// moments of y for l1_lars_kernel.  A non-finite y or f(x) is reported as DKS_ERR_NUMERIC and nothing of the instance is
// written.
// ACC (a soft-voting ensemble's member): the sums of every output go into ea.ey instead (ens_accumulate); instances
// with M <= 1 or a refused f(x) are left to explain_ensemble_tail_kernel.
// ROWS (a stacking ensemble's member, with ACC): each masked row's kept outputs go to er.ws instead (rows_store), for the
// background rows of the chunk only; nothing is summed.
template <bool L1, bool ACC = false, bool ROWS = false>
__global__ void __launch_bounds__(THREADS) explain_mlp_kernel(ExplainParams p, SimtL1 q, MlpDev m, int nw,
                                                              const double* __restrict__ X, const double* __restrict__ bg,
                                                              int D, const int* __restrict__ goff,
                                                              const int* __restrict__ gcols, EnsAcc ea, EnsRows er) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int N = p.N, G = p.G, C = p.C;
    const bool bin = m.head == DKS_MLP_HEAD_SIGMOID;
    const int H1 = m.width[1], H1p = m.pad[1], NT1 = H1p >> 3;
    double* acc = reinterpret_cast<double*>(smem_raw);                        // [C][S_cap]
    double* region = acc + ((((size_t)C * p.S_cap) + 1) & ~(size_t)1);
    double* A = region;                                                       // [63 * 63] (solve)
    double* rhs = A + 63 * 63;                                                // [64]
    double* dl = region;                                                      // Delta_j (background loop)
    double* bj = dl + (size_t)pad16(G) * H1p;                                 // [H1p]
    double* wreg = bj + H1p + (size_t)warp * warp_doubles(m);                 // this warp's buffers and output tile
    double2* buf0 = reinterpret_cast<double2*>(wreg);
    double2* buf1 = reinterpret_cast<double2*>(wreg + (size_t)(m.nbuf - 1) * 16 * m.hmax);
    double* lg = wreg + (size_t)m.nbuf * 16 * m.hmax;                         // [16][8]
    int* vi = reinterpret_cast<int*>(region + region_doubles(G, m, nw));      // [64]
    const size_t slab = (size_t)p.n * G;
    const int nsolve = bin ? 1 : C;                   // sigmoid head: class 0 is the negation of class 1

    const int ninst = dks_inst_count(p);
    for (int qi = blockIdx.x; qi < ninst; qi += gridDim.x) {
        const int i = dks_inst_at(p, qi);
        const int M = p.Mcnt[i];
        const uint64_t vm = p.vmask[i];
        __syncthreads();  // previous instance done with shared memory
        if constexpr (!ACC) zero_phi_rows(p, i);
        bool fx_bad = false;                          // stage 1 reported a refused row or a non-finite link(f(x))
        if constexpr (ROWS) fx_bad = rows_fx_bad(er, i);
        else for (int c = 0; c < C; ++c) fx_bad |= !isfinite(p.dlink[(size_t)i * C + c]);
        if (M == 0) continue;
        if (M == 1) {
            // the one varying group takes link(f(x)) - link(fnull); sigmoid head: class 0 is the negation of class 1
            if (!ACC && tid < C && !fx_bad) {
                const double v = p.dlink[(size_t)i * C + (bin ? 1 : tid)];
                p.phi[(size_t)tid * slab + (size_t)i * G + (__ffsll((long long)vm) - 1)] =
                    (bin && tid == 0) ? ((v == 0.0) ? 0.0 : -v) : v;
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
        __syncthreads();

        const double* x = X + (size_t)i * D;
        const int MP = pad16(M), KC1 = MP >> 4;
        for (int j = ROWS ? er.j0 : 0; j < (ROWS ? er.j1 : N); ++j) {
            const double wj = p.wbg[j];
            if (wj == 0.0) continue;                  // block-uniform
            const double* b = bg + (size_t)j * D;
            __syncthreads();                          // the warps are done with the previous row's Delta
            for (int idx = tid; idx < MP * H1p; idx += blockDim.x) {
                const int pp = idx / H1p, h = idx - pp * H1p;
                double d = 0.0;
                if (pp < M && h < H1) {
                    const int grp = vi[pp];
                    for (int e = goff[grp]; e < goff[grp + 1]; ++e) {
                        const int c = gcols[e];
                        d = fma(m.W[(size_t)c * H1 + h], x[c] - b[c], d);
                    }
                }
                const int kk = pp & 15;
                dl[(((size_t)(pp >> 4) * NT1 + (h >> 3)) * 32 + (h & 7) * 4 + (kk & 3)) * 4 + (kk >> 2)] = d;
            }
            for (int h = tid; h < H1p; h += blockDim.x) bj[h] = h < H1 ? m.Bbg[(size_t)j * H1 + h] : 0.0;
            __syncthreads();
            if (warp >= nw) continue;
            for (int s0 = warp * 16; s0 < S; s0 += nw * 16) {
                const int g = lane >> 2;
                const uint64_t zg = s0 + g < S ? zp[s0 + g] : 0ull;
                const uint64_t zh = s0 + g + 8 < S ? zp[s0 + g + 8] : 0ull;
                forward_tile(m, KC1, zg, zh, dl, bj, buf0, buf1, lg);
                const int s = s0 + lane;
                if (lane < 16 && s < S) {
                    double o[DKS_MLP_MAX_OUT];
                    mlp_head(m.head, lg + lane * 8, m.R, o);
                    if constexpr (ROWS) rows_store<DKS_MLP_MAX_OUT>(er, p.S_cap, i, j, s, o);
                    else for (int c = 0; c < C; ++c) acc[(size_t)c * p.S_cap + s] = fma(wj, o[c], acc[(size_t)c * p.S_cap + s]);
                }
                __syncwarp();                         // lg is rewritten by the next tile
            }
        }
        __syncthreads();
        if constexpr (ROWS) continue;
        if constexpr (ACC) {
            ens_accumulate(ea, p, i, S, acc);
            continue;
        }

        // y = link(ey) - link(fnull) per solved output, written over the sums (row u of acc); under the logit link the
        // 1 - ey of a classifier is the sum of its other classes' sums (no cancellation)
        int bad = 0;
        for (int s = tid; s < S; s += blockDim.x) {
            double y[DKS_MLP_MAX_OUT];
            for (int u = 0; u < nsolve; ++u) {
                const int c = bin ? 1 : u;
                const double e = acc[(size_t)c * p.S_cap + s];
                if (p.link == DKS_LINK_LOGIT) {
                    double rest = 0.0;
                    if (m.head == DKS_MLP_HEAD_IDENTITY) {
                        rest = 1.0 - e;
                    } else {
                        for (int o = 0; o < C; ++o)
                            if (o != c) rest += acc[(size_t)o * p.S_cap + s];
                    }
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
        block_solve(p, i, pl, M, acc, p.S_cap, nsolve, bin, A, rhs, vi);
    }
}

}  // namespace mlp
}  // namespace dks
