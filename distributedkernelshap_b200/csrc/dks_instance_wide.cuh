// CUDA-core coalition kernel for per-instance plans of 65..128 groups (two 64-bit words per coalition row), for the
// instances whose groups all vary (M = G, so varying position k is group k).  Binary-logistic, identity and exp heads.
//
// One CTA per instance (grid-stride over the instance list).  Binary head: the background is streamed in chunks of NC
// rows; for each chunk the CTA builds nibble tables T[j][t][x] = sum_{b in x} BWs[4t + b][j] (scaled grouped background
// contributions, 32 nibbles x 16 values per background row), and every thread takes coalition rows s = tid, tid + 256, ...:
// the background part of the masked score is 32 table reads, one per nibble of the row, instead of up to 128 adds.  The
// lanes of a warp read the 16 entries of the same (j, t) row, which lie in 16 consecutive banks: conflict-free whatever
// the nibble values.  (sum p1, sum p0) of each row carries across chunks in shared memory, in the place where y(s) goes
// afterwards.  Identity head: ey = fnull + sum_k z_sk (XW_k - Bbar_k) in float64, no background loop.
// The solve reads the instance's inverse normal matrix (factor_wide_plans_kernel) from global memory: beta = A^-1 rhs.
#pragma once

#include "dks_common.cuh"
#include "dks_kernels.cuh"

namespace dks {
namespace iwide {

constexpr int THREADS = 256;
constexpr int NC = 32;        // background rows per chunk
constexpr int NT = 32;        // nibbles of a two-word row

// y(s) (double) / per-row (sum p1, sum p0) [S_cap], a(s) [S_cap] floats, tables [NC][NT][16], bases / weights of the chunk,
// xw / rhs / beta [128] doubles
inline size_t smem_bytes(int S_cap) {
    return sizeof(double) * (size_t)S_cap + sizeof(float) * (size_t)S_cap + sizeof(float) * ((size_t)NC * NT * 16 + 2 * NC) +
           sizeof(double) * 3 * 128;
}

// rhs[k] = sum_s w_s e_sk (y_s - z_sL delta) over two-word rows, warp-per-k
__device__ inline void build_rhs2(const uint64_t* __restrict__ zp, const double* __restrict__ wp, const double* ys, int S,
                                  int M, double delta, double* rhs) {
    const int nA = M - 1, L = M - 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int k = warp; k < nA; k += nwarps) {
        double acc = 0;
#pragma unroll 4
        for (int s = lane; s < S; s += 32) {
            const uint64_t* row = zp + (size_t)s * 2;
            const int zl = zbit2(row, L) ? 1 : 0, zk = zbit2(row, k) ? 1 : 0;
            const int e = zk - zl;
            if (e != 0) acc += wp[s] * (double)e * (ys[s] - (zl ? delta : 0.0));
        }
        acc = warp_sum(acc);
        if (lane == 0) rhs[k] = acc;
    }
}

// beta = A^-1 rhs (A^-1 symmetric: thread r reads column r, coalesced), then phi of output slab `out` (and its negation
// into slab `neg` for the binary head's output 0)
__device__ inline void solve_write(const double* __restrict__ ainv, const double* rhs, double* beta, int M, double delta,
                                   double* __restrict__ phi_out, double* __restrict__ phi_neg) {
    const int nA = M - 1;
    for (int r = threadIdx.x; r < nA; r += blockDim.x) {
        double v = 0.0;
        for (int k = 0; k < nA; ++k) v += ainv[(size_t)k * nA + r] * rhs[k];
        beta[r] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double sum = 0;
        for (int k = 0; k < nA; ++k) {
            double v = beta[k];
            sum += v;
            if (fabs(v) < 1e-10) v = 0;
            phi_out[k] = v;
            if (phi_neg) phi_neg[k] = v == 0.0 ? 0.0 : -v;
        }
        double last = delta - sum;
        if (fabs(last) < 1e-10) last = 0;
        phi_out[nA] = last;
        if (phi_neg) phi_neg[nA] = last == 0.0 ? 0.0 : -last;
    }
}

// EXP: the instantiation of the exp head, which compiles its branch only (the other heads' instantiation is unchanged)
template <bool EXP = false>
__global__ void __launch_bounds__(THREADS, 2) explain_wide_instance_kernel(ExplainParams p, ExpBackground eb) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* ys = reinterpret_cast<double*>(smem_raw);                // [S_cap]
    float2* acc = reinterpret_cast<float2*>(ys);                      // [S_cap] (sum p1, sum p0): same bytes as ys[s]
    float* afs = reinterpret_cast<float*>(ys + p.S_cap);              // [S_cap] scaled instance part a(s)
    float* T = afs + p.S_cap;                                         // [NC][NT][16]
    float* bch = T + NC * NT * 16;                                    // [NC]
    float* wch = bch + NC;                                            // [NC]
    double* xw = reinterpret_cast<double*>(wch + NC);                 // [128]
    double* rhs = xw + 128;                                           // [128]
    double* beta = rhs + 128;                                         // [128]
    const int tid = threadIdx.x;
    const int N = p.N, G = p.G, C = p.C;
    const size_t slab = (size_t)p.n * G;

    const int ninst = dks_inst_count(p);
    for (int qi = blockIdx.x; qi < ninst; qi += gridDim.x) {
        const int i = dks_inst_at(p, qi);
        const int M = p.Mcnt[i];
        __syncthreads();  // previous instance done with shared memory
        if (M != G || M < 65 || M > 128) {
            if (tid == 0) { if (atomicCAS(&p.status[0], 0, DKS_ERR_UNSUPPORTED) == 0) p.status[1] = M; }
            continue;
        }
        const int S = dks_effective_S(M, p.S_req);
        if (S > p.S_cap) {
            if (tid == 0) { if (atomicCAS(&p.status[0], 0, DKS_ERR_INVALID) == 0) p.status[1] = i; }
            continue;
        }
        const uint64_t* zp = p.ext_z + (size_t)i * p.ext_stride * 2;
        const double* wp = p.ext_w + (size_t)i * p.ext_stride;
        const double* ainv = p.ext_ainv + (size_t)i * p.ext_fstride;

        if constexpr (EXP) {
            // exp head (DESIGN.md §5.0.8): the binary head's chunk tables give the background part; per row acc[s] carries
            // (sum_j 2^t'_j, max_j t'_j) across chunks, t'_j = bases_j - c (bases carry log2 w_j), and afs[s] is unused.
            // ey = 2^a(s) sum with the instance part a(s) in float64; rows outside the range rule take exp_row_f64.
            if (tid < M) xw[tid] = p.scale * p.XW[(size_t)i * G + tid];
            for (int s = tid; s < S; s += THREADS) acc[s] = make_float2(0.f, -INFINITY);
            const int tbase = (int)(reinterpret_cast<unsigned char*>(T) - smem_raw);
            for (int j0 = 0; j0 < N; j0 += NC) {
                const int nc = min(NC, N - j0);
                __syncthreads();  // the previous chunk's tables are no longer read
                // rows past the end of the background: zero tables and base -inf, so 2^t' = 0 and the maximum is unchanged
                for (int idx = tid; idx < NC * NT * 16; idx += THREADS) {
                    const int jj = idx / (NT * 16), t = (idx >> 4) & (NT - 1), x = idx & 15;
                    float v = 0.f;
#pragma unroll
                    for (int b = 0; b < 4; ++b)
                        if (jj < nc && ((x >> b) & 1) && 4 * t + b < M) v += p.BWs[(size_t)(4 * t + b) * N + j0 + jj];
                    T[idx] = v;
                }
                if (tid < NC) bch[tid] = tid < nc ? p.bases[j0 + tid] : -INFINITY;
                __syncthreads();
                for (int s = tid; s < S; s += THREADS) {
                    const uint64_t z0 = zp[2 * s], z1 = zp[2 * s + 1];
                    int off[NT];
#pragma unroll
                    for (int t = 0; t < NT; ++t)
                        off[t] = tbase + 4 * (t * 16 + (int)(((t < 16 ? z0 : z1) >> (4 * (t & 15))) & 15ull));
                    float2 a2 = acc[s];
                    float sum = a2.x, thi = a2.y;
#pragma unroll
                    for (int jj = 0; jj < NC; ++jj) {
                        float c4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                        for (int t = 0; t < NT; ++t)
                            c4[t & 3] += *reinterpret_cast<const float*>(smem_raw + off[t] + jj * (NT * 16 * 4));
                        const float tt = bch[jj] - ((c4[0] + c4[1]) + (c4[2] + c4[3]));
                        thi = fmaxf(thi, tt);
                        sum += ex2_approx(tt);
                    }
                    acc[s] = make_float2(sum, thi);
                }
            }
            __syncthreads();
            const double fn = p.fnull[0], delta = p.dlink[i];
            int bad = !isfinite(delta);
            for (int s = tid; s < S; s += THREADS) {
                const uint64_t z0 = zp[2 * s], z1 = zp[2 * s + 1];
                double a = 0;
                for (int k = 0; k < M; ++k) if (((k < 64 ? z0 : z1) >> (k & 63)) & 1ull) a += xw[k];
                const float2 a2 = acc[s];
                const double y = exp_row_ey(p, eb, i, a, a2.x, a2.y, z0, z1, M, nullptr) - fn;
                bad |= !isfinite(y);
                ys[s] = y;             // the same bytes as acc[s], read above by this thread only
            }
            if (__syncthreads_or(bad)) {
                // a non-finite ey (or f(x)) is reported, never solved
                if (tid == 0 && atomicCAS(&p.status[0], 0, DKS_ERR_NUMERIC) == 0) p.status[1] = i;
                continue;
            }
            build_rhs2(zp, wp, ys, S, M, delta, rhs);
            __syncthreads();
            solve_write(ainv, rhs, beta, M, delta, p.phi + (size_t)i * G, nullptr);
        } else if (p.act == DKS_ACT_BINARY_LOGISTIC) {
            if (tid < M) xw[tid] = p.scale * p.XW[(size_t)i * G + tid];
            __syncthreads();
            for (int s = tid; s < S; s += THREADS) {
                const uint64_t z0 = zp[2 * s], z1 = zp[2 * s + 1];
                double a = 0;
                for (int k = 0; k < M; ++k) if (((k < 64 ? z0 : z1) >> (k & 63)) & 1ull) a += xw[k];
                afs[s] = (float)a;
                acc[s] = make_float2(0.f, 0.f);
            }
            // byte offset of the tables from the start of shared memory: a table read is then one LDS with the
            // background row's offset as an immediate (the loop over the NC rows of a chunk is unrolled)
            const int tbase = (int)(reinterpret_cast<unsigned char*>(T) - smem_raw);
            for (int j0 = 0; j0 < N; j0 += NC) {
                const int nc = min(NC, N - j0);
                __syncthreads();  // the previous chunk's tables are no longer read
                // rows past the end of the background get zero tables and zero weight: they add exactly nothing
                for (int idx = tid; idx < NC * NT * 16; idx += THREADS) {
                    const int jj = idx / (NT * 16), t = (idx >> 4) & (NT - 1), x = idx & 15;
                    float v = 0.f;
#pragma unroll
                    for (int b = 0; b < 4; ++b)
                        if (jj < nc && ((x >> b) & 1) && 4 * t + b < M) v += p.BWs[(size_t)(4 * t + b) * N + j0 + jj];
                    T[idx] = v;
                }
                if (tid < NC) { bch[tid] = tid < nc ? p.bases[j0 + tid] : 0.f; wch[tid] = tid < nc ? p.wbf[j0 + tid] : 0.f; }
                __syncthreads();
                for (int s = tid; s < S; s += THREADS) {
                    const uint64_t z0 = zp[2 * s], z1 = zp[2 * s + 1];
                    int off[NT];
#pragma unroll
                    for (int t = 0; t < NT; ++t)
                        off[t] = tbase + 4 * (t * 16 + (int)(((t < 16 ? z0 : z1) >> (4 * (t & 15))) & 15ull));
                    const float af = afs[s];
                    float2 a2 = acc[s];
                    float acc1 = a2.x, acc0 = a2.y;
#pragma unroll
                    for (int jj = 0; jj < NC; ++jj) {
                        // four partial sums: the table reads of a row are independent of each other
                        float c4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                        for (int t = 0; t < NT; ++t)
                            c4[t & 3] += *reinterpret_cast<const float*>(smem_raw + off[t] + jj * (NT * 16 * 4));
                        const float c = (c4[0] + c4[1]) + (c4[2] + c4[3]);
                        float tt = (bch[jj] - c) + af;     // = -kappa*log2(e) * masked score
                        tt = fminf(fmaxf(tt, -120.f), 120.f);
                        const float u = ex2_approx(tt);    // exp(-kappa*score)
                        const float r = rcp_approx(1.f + u);
                        acc1 = fmaf(wch[jj], r, acc1);
                        acc0 = fmaf(wch[jj], u * r, acc0);
                    }
                    acc[s] = make_float2(acc1, acc0);
                }
            }
            __syncthreads();
            const double lf1 = p.linkfnull[1], f1 = p.fnull[1];
            for (int s = tid; s < S; s += THREADS) {
                const float2 a2 = acc[s];
                ys[s] = p.link == DKS_LINK_LOGIT ? log((double)a2.x / (double)a2.y) - lf1 : (double)a2.x - f1;
            }
            __syncthreads();
            // WLS for output 1; output 0 is its exact negation (p0 = 1 - p1 row-wise)
            const double delta = p.dlink[(size_t)i * C + 1];
            build_rhs2(zp, wp, ys, S, M, delta, rhs);
            __syncthreads();
            solve_write(ainv, rhs, beta, M, delta, p.phi + slab + (size_t)i * G, p.phi + (size_t)i * G);
        } else {
            // identity head: the background average commutes with the head -- float64 throughout
            for (int r = 0; r < p.R; ++r) {
                __syncthreads();
                if (tid < M) xw[tid] = p.XW[((size_t)i * G + tid) * p.R + r] - p.Bbar[(size_t)tid * p.R + r];
                __syncthreads();
                const double fn = p.fnull[r], lfn = p.linkfnull[r];
                for (int s = tid; s < S; s += THREADS) {
                    const uint64_t z0 = zp[2 * s], z1 = zp[2 * s + 1];
                    double a = fn;
                    for (int k = 0; k < M; ++k) if (((k < 64 ? z0 : z1) >> (k & 63)) & 1ull) a += xw[k];
                    ys[s] = link_f(a, p.link) - lfn;
                }
                __syncthreads();
                const double delta = p.dlink[(size_t)i * C + r];
                build_rhs2(zp, wp, ys, S, M, delta, rhs);
                __syncthreads();
                solve_write(ainv, rhs, beta, M, delta, p.phi + (size_t)r * slab + (size_t)i * G, nullptr);
            }
        }
    }
}

}  // namespace iwide
}  // namespace dks
