// Shared-plan fast path of the fused coalition evaluation (binary-logistic head).
//
// When every instance of a bucket evaluates the SAME coalition plan and all G groups vary (the common case: on
// Adult-shaped data every instance has M = G), the masked score separates:
//     t(i, s, j) = a(i, s) + d(s, j),   a(i, s) = scale * sum_k z_sk XW_i[k],   d(s, j) = scale * (score_j - sum_k z_sk BW[j][k])
// so  2^t = A(i, s) * Dm(s, j)  with Dm = 2^d independent of the instance.  Dm (S x N floats, 0.8 MB for Adult) is
// computed once per plan, row-normalised; a warp owns 32 coalition rows and streams the instances through them.  Two
// elements share a reciprocal,  p1a + p1b = (2 + sm) / (1 + sm + q),  sm = A (Dma + Dmb),  q = A^2 (Dma Dmb),  so what the
// kernel keeps per row are the pair sums and pair products of Dm, in shared memory (explain_shared_smem_kernel).  No
// GEMM, no EX2 per element: 3.5 fp32 ops + 0.5 MUFU.  Output: (sum p1, sum p0) per (instance, coalition);
// wls_pmat_kernel / wls_shared_kernel apply the link and solve with what the plan precomputed.
// Instances with a partial varying set, per-instance plans and other heads go through the general kernels.
#pragma once

#include "dks_kernels.cuh"

namespace dks {
namespace shared_path {

constexpr int MAXN = 128;            // background rows per launch (a warp's slice of shared memory)
constexpr float U_CLAMP = 1.152921504606846976e18f;   // 2^60: (1 + ua)(1 + ub) stays finite in fp32

// d(s, j) = scale * (score_j - sum_k z_sk BW[j][k])  for the full varying set (k = group index), in log2 units.
// Rows are normalised: dme[s] = rint(max_j d(s, j)), DmT[j][s] = 2^(d(s, j) - dme[s]) <= sqrt(2), float32, transposed so that
// consecutive coalitions are contiguous (coalesced row loads by lanes).  The exponent goes back in through a(i, s), so
// products of two entries of a row (the kernel stores pair sums and pair products) cannot overflow or vanish together.
__device__ __forceinline__ double plan_d(const uint64_t* __restrict__ zz, const double* __restrict__ BW,
                                         const double* __restrict__ scores, int j, int G, double scale) {
    double c = 0.0;
    for (int k = 0; k < G; ++k)
        if ((zz[k >> 6] >> (k & 63)) & 1ull) c += BW[(size_t)j * G + k];
    return scale * (scores[j] - c);
}
__global__ void plan_dme_kernel(const uint64_t* __restrict__ z, int W, int S, int S_pad, const double* __restrict__ BW,
                                const double* __restrict__ scores, int N, int G, double scale, double* __restrict__ dme) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S_pad) return;
    double mx = 0.0;
    if (s < S) {
        mx = -1.0e300;
        for (int j = 0; j < N; ++j) mx = fmax(mx, plan_d(z + (size_t)s * W, BW, scores, j, G, scale));
        mx = rint(mx);
    }
    dme[s] = mx;
}
__global__ void plan_dm_kernel(const uint64_t* __restrict__ z, int W, int S, int S_pad, const double* __restrict__ BW,
                               const double* __restrict__ scores, int N, int G, double scale, const double* __restrict__ dme,
                               float* __restrict__ DmT) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * S_pad) return;
    const int j = idx / S_pad, s = idx - j * S_pad;
    float out = 0.f;
    if (s < S) out = (float)exp2(plan_d(z + (size_t)s * W, BW, scores, j, G, scale) - dme[s]);
    DmT[idx] = out;
}

struct SharedParams {
    int n, N, G, S, S_pad;
    double scale;
    const float* DmT;        // [N][S_pad] rows normalised by 2^-dme[s]
    const double* dme;       // [S_pad]
    const uint64_t* z;       // [S][W]
    const double* XT;        // [n][ceil(G/4)][16] nibble tables: scale * sum of the contributions a nibble selects
    const int* list;         // instances on this path
    const int* count;        // their number (device)
    float2* sums;            // [n][S_pad] (sum p1, sum p0)
    int accumulate;          // add to sums instead of overwriting them (second and later background chunks)
    float* acache;           // [n][S_pad] A(i, s) of sixteen-word rows, kept between the launches of the background chunks
    int acache_mode;         // 0: off, 1: this launch writes it (first chunk), 2: this launch reads it
    const float* wn;         // [N] weighted backgrounds: N w_j with the w_j summing to 1 (the weighted kernels only)
};

// Two sigmoids with one reciprocal.  With ua = 2^ta, ub = 2^tb:  (1+ua)(1+ub) = 1 + sm + q,  sm = ua + ub, q = ua*ub
//   p1a + p1b = (2 + sm) / (1 + sm + q)          p0a + p0b = (sm + 2q) / (1 + sm + q)
// 12 FP32-pipe ops + 1 MUFU per pair.  CLAMP: bound u at 2^60 so q cannot overflow (only needed for extreme scores).
template <bool CLAMP>
__device__ __forceinline__ void pair_acc(float A, float dma, float dmb, float& a1, float& a0) {
    float ua = A * dma, ub = A * dmb;
    if (CLAMP) { ua = fminf(ua, U_CLAMP); ub = fminf(ub, U_CLAMP); }
    const float q = ua * ub, sm = ua + ub;
    const float t1 = 1.f + sm;
    const float r = rcp_approx(fmaf(ua, ub, t1));
    a1 = fmaf(r, t1 + 1.f, a1);
    a0 = fmaf(r, fmaf(2.f, q, sm), a0);
}
__device__ __forceinline__ void single_acc(float A, float dma, float& a1, float& a0) {
    const float ua = fminf(A * dma, U_CLAMP);
    const float r = rcp_approx(1.f + ua);
    a1 += r;
    a0 = fmaf(ua, r, a0);
}

// ---- the coalition kernel, the Dm rows parked in shared memory ------------------------------------------------------
// A lane's row of Dm (up to 128 floats) held in registers costs 168 registers per thread, 12 warps per SM, and leaves
// the kernel latency bound.  Instead every warp parks its 32 rows in its own slice of shared memory, one float4 per
// (quad of columns, lane): a lane reads back only what it wrote itself (no barrier), and the 128-bit loads of one quad by
// a warp cover 512 consecutive bytes (no bank conflicts).  The number of warps per CTA follows from the shared memory a
// slice takes.
constexpr int TM_MAX_WARPS = 20;
__host__ __device__ inline int dm_quads(int N) { return (N + 3) / 4; }
__host__ __device__ inline size_t dm_slice_bytes(int N) { return (size_t)dm_quads(N) * 32 * sizeof(float4); }

// columns 16c .. 16c + 15 of this lane's row: quads 4c .. 4c + 3 of the slice, those below nq
__device__ __forceinline__ void dm_st16(float4* sl, int c, int nq, int lane, const float (&v)[16]) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (4 * c + k < nq) sl[(4 * c + k) * 32 + lane] = make_float4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
}
__device__ __forceinline__ void dm_ld16(const float4* sl, int c, int nq, int lane, float (&v)[16]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float4 t = 4 * c + k < nq ? sl[(4 * c + k) * 32 + lane] : make_float4(0.f, 0.f, 0.f, 0.f);
        v[4 * k] = t.x; v[4 * k + 1] = t.y; v[4 * k + 2] = t.z; v[4 * k + 3] = t.w;
    }
}

// Four sigmoids (two pairs, each sharing one reciprocal) in packed arithmetic, from what the slice holds for a quad of
// columns (0,2) (1,3): ds = (dm0 + dm2, dm1 + dm3) and dq = (dm0 dm2, dm1 dm3), both independent of the instance:
// sm = A ds,  q = A^2 dq.  14 fp32 ops + 2 MUFU per four elements (A2 = (A, A), AA2 = (A^2, A^2), AA2x2 = 2 AA2).
__device__ __forceinline__ void quad_acc_sq(f32x2 A2, f32x2 AA2, f32x2 AA2x2, f32x2 ds, f32x2 dq, f32x2 one2, f32x2 two2,
                                            f32x2& a1, f32x2& a0) {
    const f32x2 sm = f2_mul(A2, ds);
    const f32x2 t1 = f2_add(sm, one2);
    const f32x2 den = f2_fma(AA2, dq, t1);
    const f32x2 w = f2_fma(AA2x2, dq, sm);
    float dlo, dhi;
    f2_unpack(den, dlo, dhi);
    const f32x2 r = f2_pack(rcp_approx(dlo), rcp_approx(dhi));
    a1 = f2_fma(r, f2_add(sm, two2), a1);
    a0 = f2_fma(r, w, a0);
}

// one 16-column chunk of a row: four packed quads (or the clamped scalar pairs), NV = valid columns of this chunk
// v holds, per full quad of columns, (ds.lo, ds.hi, dq.lo, dq.hi); columns past the last full quad of the tail chunk are
// raw Dm values.
template <int NV>
__device__ __forceinline__ void chunk_sums(const float (&v)[16], float A, f32x2 A2, f32x2 AA2, f32x2 AA2x2, f32x2 one2,
                                           f32x2 two2, f32x2 (&acc1)[2], f32x2 (&acc0)[2], float& t1s, float& t0s) {
#pragma unroll
    for (int jj = 0; jj + 3 < NV; jj += 4)
        quad_acc_sq(A2, AA2, AA2x2, f2_pack(v[jj], v[jj + 1]), f2_pack(v[jj + 2], v[jj + 3]), one2, two2, acc1[(jj >> 2) & 1],
                    acc0[(jj >> 2) & 1]);
    constexpr int Q = NV & ~3;
    if ((NV & 3) >= 2) pair_acc<false>(A, v[Q], v[Q + 1], t1s, t0s);
    if (NV & 1) single_acc(A, v[NV - 1], t1s, t0s);
}

// ---- weighted backgrounds (k-means centroids, user weights) ----------------------------------------------------------
// The kernels see w'_j = N w_j (the w_j sum to 1), so the weighted sums have the magnitude of the uniform ones and every
// consumer (the logit link, the identity link's sum * (1 / N), the solves) is unchanged.  A pair (a, b) still shares one
// reciprocal:  with ua = A Dma, ub = A Dmb, den = (1 + ua)(1 + ub) = 1 + A (Dma + Dmb) + A^2 Dma Dmb,
//   wa p1a + wb p1b = (W2 + A X) / den                   X = wa Dmb + wb Dma
//   wa p0a + wb p0b = (A Y + A^2 W2 Dma Dmb) / den       Y = wa Dma + wb Dmb,   W2 = wa + wb
// X and Y are per row and column pair, W2 per column pair only.  The weighted slice holds two float4 per quad of columns
// (0,2) (1,3) and lane: (ds, dq) as in the uniform slice, then (X, Y); W2 comes from a small per-CTA array (a broadcast
// load).  Columns past N have Dm = 0 and weight 0 and contribute exactly nothing, so a partial last quad needs no tail
// code.  p0 keeps its own sum (forming it as W - sum p1 would cancel at saturated scores).  The weighted slice holds an
// even number of quads (a zero quad past an odd count), so that loops with a run-time trip count can take them in pairs,
// each pair member on its own accumulator chain, with register-resident accumulators.
__host__ __device__ inline int dm_quads_w(int N) { return (dm_quads(N) + 1) & ~1; }
__host__ __device__ inline size_t dm_slice_bytes_w(int N) { return (size_t)dm_quads_w(N) * 2 * 32 * sizeof(float4); }

// quad q of row s for the weighted slice, from the raw columns of Dm and their weights
__device__ __forceinline__ void dm_quad_w(const float* __restrict__ DmT, const float* __restrict__ wn, int N, int S_pad, int s,
                                          int q, float4& sq, float4& xy) {
    float d[4], w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int j = 4 * q + k;
        d[k] = j < N ? DmT[(size_t)j * S_pad + s] : 0.f;
        w[k] = j < N ? wn[j] : 0.f;
    }
    sq = make_float4(__fadd_rn(d[0], d[2]), __fadd_rn(d[1], d[3]), __fmul_rn(d[0], d[2]), __fmul_rn(d[1], d[3]));
    xy = make_float4(__fadd_rn(__fmul_rn(w[0], d[2]), __fmul_rn(w[2], d[0])), __fadd_rn(__fmul_rn(w[1], d[3]), __fmul_rn(w[3], d[1])),
                     __fadd_rn(__fmul_rn(w[0], d[0]), __fmul_rn(w[2], d[2])), __fadd_rn(__fmul_rn(w[1], d[1]), __fmul_rn(w[3], d[3])));
}
// W2 of quad q (zero past N)
__device__ __forceinline__ float2 w2_quad(const float* __restrict__ wn, int N, int q) {
    const int j = 4 * q;
    const float w0 = j < N ? wn[j] : 0.f, w1 = j + 1 < N ? wn[j + 1] : 0.f;
    const float w2 = j + 2 < N ? wn[j + 2] : 0.f, w3 = j + 3 < N ? wn[j + 3] : 0.f;
    return make_float2(__fadd_rn(w0, w2), __fadd_rn(w1, w3));
}

// four weighted sigmoids, two reciprocals: 10 packed ops + 2 MUFU (the uniform quad_acc_sq: 7 + 2).  The A^2 W2 Dma Dmb
// term is formed as (r q) W2: q = A^2 Dma Dmb reaches 2^121 below the clamped path's threshold (A <= 1e18, Dm <= sqrt 2)
// and W2 is bounded only by the background size, so q W2 could pass the fp32 range, while r q = q / den < 1.
__device__ __forceinline__ void quad_acc_w(f32x2 A2, f32x2 AA2, float4 sq, float4 xy, float2 w2, f32x2 one2, f32x2& a1,
                                           f32x2& a0) {
    const f32x2 W2 = f2_pack(w2.x, w2.y);
    const f32x2 sm = f2_mul(A2, f2_pack(sq.x, sq.y));
    const f32x2 q = f2_mul(AA2, f2_pack(sq.z, sq.w));
    const f32x2 den = f2_add(f2_add(sm, one2), q);
    float dlo, dhi;
    f2_unpack(den, dlo, dhi);
    const f32x2 r = f2_pack(rcp_approx(dlo), rcp_approx(dhi));
    a1 = f2_fma(r, f2_fma(A2, f2_pack(xy.x, xy.y), W2), a1);
    a0 = f2_fma(f2_mul(r, q), W2, f2_fma(r, f2_mul(A2, f2_pack(xy.z, xy.w)), a0));
}

// the clamped scalar path of a weighted row (A > 1e18: saturated scores), one element at a time from the raw row
__device__ __forceinline__ void row_sums_clamped_w(const float* __restrict__ DmT, const float* __restrict__ wn, int N, int S_pad,
                                                   int s, float A, float& s1, float& s0) {
    float r1 = 0.f, r0 = 0.f;
    for (int j = 0; j < N; ++j) {
        const float w = wn[j];
        const float ua = fminf(A * DmT[(size_t)j * S_pad + s], U_CLAMP);
        const float r = rcp_approx(1.f + ua);
        r1 = fmaf(w, r, r1);
        r0 = fmaf(w * ua, r, r0);
    }
    s1 = r1; s0 = r0;
}

// one warp = 32 coalition rows (one per lane) x a strided subset of the instances
// NTAIL = N % 16 (compile time): the last, partial chunk is straight-line code
// W = 64-bit words per coalition row (1: up to 64 groups, 2: up to 128, 16: up to 1024)
// WT: weighted background (the weighted slice and quad_acc_w above; NTAIL is unused and 0)
template <int NTAIL, int W, bool WT = false>
__global__ void __launch_bounds__(32 * TM_MAX_WARPS, 1) explain_shared_smem_kernel(SharedParams p, int warps_used) {
    extern __shared__ float4 s_dm[];                      // [warps_used][dm_quads(N)][32]  (weighted: [warps_used][2 nqw][32])
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    const int n_rg = p.S_pad / 32;                       // row groups
    const int total_warps = gridDim.x * warps_used;
    const int nparts = total_warps / n_rg;               // replicas of every row group
    const int gw = blockIdx.x * warps_used + warp;
    const bool active = warp < warps_used && nparts > 0 && gw < nparts * n_rg;
    float2* sW2 = nullptr;                               // weighted: [nqw] W2 per quad, after the slices
    if constexpr (WT) {
        const int nqw = dm_quads_w(p.N);
        sW2 = reinterpret_cast<float2*>(s_dm + (size_t)warps_used * 2 * nqw * 32);
        for (int q = threadIdx.x; q < nqw; q += blockDim.x) sW2[q] = w2_quad(p.wn, p.N, q);
        __syncthreads();
    }
    if (active) {
        const int rg = gw % n_rg, part = gw / n_rg;
        const int s = rg * 32 + lane;
        const int cnt = *p.count;
        const int N = p.N, G = p.G;
        const int nfull = N / 16;
        const int nq = dm_quads(N);
        const int nqw = dm_quads_w(N);                  // weighted: quads of the slice (even)
        float4* sl = s_dm + (size_t)warp * (WT ? 2 * nqw : nq) * 32;    // this warp's slice
        const double es = p.dme[s];                      // exponent the row of Dm was normalised by (entries <= sqrt 2)
        if constexpr (WT) {
            for (int q = 0; q < nqw; ++q) {
                float4 sq, xy;
                dm_quad_w(p.DmT, p.wn, N, p.S_pad, s, q, sq, xy);
                sl[(2 * q) * 32 + lane] = sq;
                sl[(2 * q + 1) * 32 + lane] = xy;
            }
        }
        for (int c = 0; !WT && c * 16 < N; ++c) {
            float v[16];
#pragma unroll
            for (int jj = 0; jj < 16; ++jj) {
                const int j = c * 16 + jj;
                v[jj] = j < N ? p.DmT[(size_t)j * p.S_pad + s] : 0.f;
            }
            // every full quad of columns (0,2) (1,3) is stored as pair sums and pair products
            const int nv = c < nfull ? 16 : NTAIL;
#pragma unroll
            for (int jj = 0; jj < 16; jj += 4) {
                if (jj + 3 < nv) {
                    const float d0 = v[jj], d1 = v[jj + 1], d2 = v[jj + 2], d3 = v[jj + 3];
                    v[jj] = d0 + d2; v[jj + 1] = d1 + d3; v[jj + 2] = d0 * d2; v[jj + 3] = d1 * d3;
                }
            }
            dm_st16(sl, c, nq, lane, v);
        }
        // rows of one or two words stay in registers; sixteen-word rows (more than 128 groups) are re-read per instance
        constexpr int WR = W <= 2 ? W : 1;
        uint64_t zz[WR];
#pragma unroll
        for (int w = 0; w < WR; ++w) zz[w] = s < p.S ? p.z[(size_t)s * W + w] : 0ull;
        const int ntab = (G + 3) / 4;
        const f32x2 one2 = f2_pack(1.f, 1.f), two2 = f2_pack(2.f, 2.f);

        // Up to 16 groups (four nibbles): the table entries of the NEXT instance are loaded one iteration ahead (the row's
        // nibbles, hence the offsets, do not depend on the instance), so neither the index load nor the table load sits
        // in front of A.  Wider problems load in place: their per-instance arithmetic is long enough to hide it.
        const bool ahead = W <= 2 && ntab <= 4;
        int off[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) off[t] = t * 16 + (int)((zz[0] >> (4 * t)) & 15ull);
        int i_cur = part < cnt ? p.list[part] : 0;
        int i_nx = part + nparts < cnt ? p.list[part + nparts] : 0;
        double nx[4] = {0.0, 0.0, 0.0, 0.0};
        if (ahead && part < cnt) {
#pragma unroll
            for (int t = 0; t < 4; ++t)
                if (t < ntab) nx[t] = __ldg(p.XT + (size_t)i_cur * ntab * 16 + off[t]);
        }
        for (int m = part; m < cnt; m += nparts) {
            int i;
            double a;
            bool cached = false;                             // only ever set for sixteen-word rows
            if (ahead) {
                i = i_cur;
                a = (nx[0] + nx[1]) + (nx[2] + nx[3]);
                i_cur = i_nx;
                if (m + nparts < cnt) {
#pragma unroll
                    for (int t = 0; t < 4; ++t)
                        if (t < ntab) nx[t] = __ldg(p.XT + (size_t)i_cur * ntab * 16 + off[t]);
                }
                if (m + 2 * nparts < cnt) i_nx = p.list[m + 2 * nparts];
            } else if (W <= 2) {
                i = p.list[m];
                const double* xt = p.XT + (size_t)i * ntab * 16;
                double a0 = 0.0, a1 = 0.0;
#pragma unroll
                for (int w = 0; w < WR; ++w) {
#pragma unroll 4
                    for (int t = 0; t < 16 && 16 * w + t < ntab; t += 2) {
                        a0 += __ldg(xt + (16 * w + t) * 16 + (int)((zz[w] >> (4 * t)) & 15ull));
                        if (16 * w + t + 1 < ntab) a1 += __ldg(xt + (16 * w + t + 1) * 16 + (int)((zz[w] >> (4 * t + 4)) & 15ull));
                    }
                }
                a = a0 + a1;
            } else if (p.acache_mode == 2) {
                // sixteen-word rows, second and later background chunks: A(i, s) does not depend on the chunk (the row
                // exponent dme[s] covers the whole background) -- the first chunk's launch left it in acache
                i = p.list[m];
                a = 0.0;
                cached = true;
            } else {
                // sixteen-word rows: one word (sixteen nibble tables) at a time, the word re-read from the plan (L1/L2
                // resident: 128 B per row); four partial sums keep the float64 add chains short
                i = p.list[m];
                const double* xt = p.XT + (size_t)i * ntab * 16;
                const uint64_t* zrow = p.z + (size_t)s * W;
                const int nwords = (ntab + 15) >> 4;
                double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
                for (int w = 0; w < nwords; ++w) {
                    const uint64_t zw = s < p.S ? __ldg(zrow + w) : 0ull;
                    const double* xw = xt + (size_t)w * 256;
                    const int nt = ntab - 16 * w < 16 ? ntab - 16 * w : 16;      // tables this word addresses
                    if (nt == 16) {
#pragma unroll
                        for (int t = 0; t < 16; t += 4) {
                            a0 += __ldg(xw + t * 16 + (int)((zw >> (4 * t)) & 15ull));
                            a1 += __ldg(xw + (t + 1) * 16 + (int)((zw >> (4 * t + 4)) & 15ull));
                            a2 += __ldg(xw + (t + 2) * 16 + (int)((zw >> (4 * t + 8)) & 15ull));
                            a3 += __ldg(xw + (t + 3) * 16 + (int)((zw >> (4 * t + 12)) & 15ull));
                        }
                    } else {
                        for (int t = 0; t < nt; ++t) a0 += __ldg(xw + t * 16 + (int)((zw >> (4 * t)) & 15ull));
                    }
                }
                a = (a0 + a1) + (a2 + a3);
            }
            float A;
            if (W > 2 && cached) {
                A = p.acache[(size_t)i * p.S_pad + s];
            } else {
                a += es;
                a = fmin(fmax(a, -120.0), 120.0);
                const double an = rint(a);
                A = ex2_approx((float)(a - an)) * __int_as_float((127 + (int)an) << 23);
                if (W > 2 && p.acache_mode == 1) p.acache[(size_t)i * p.S_pad + s] = A;
            }
            // A^2 must stay finite in fp32 (the normalised entries are <= sqrt 2, so A bounds every u): rows beyond that
            // take the clamped scalar path on the raw row from global memory (rare: saturated scores)
            const bool risky = __any_sync(0xffffffffu, A > 1.0e18f);
            if constexpr (WT) {
                float s1, s0;
                if (risky) {
                    row_sums_clamped_w(p.DmT, p.wn, N, p.S_pad, s, A, s1, s0);
                } else {
                    const f32x2 A2 = f2_pack(A, A);
                    const float AA = A * A;
                    const f32x2 AA2 = f2_pack(AA, AA);
                    f32x2 acc1[2] = {f2_pack(0.f, 0.f), f2_pack(0.f, 0.f)}, acc0[2] = {f2_pack(0.f, 0.f), f2_pack(0.f, 0.f)};
#pragma unroll 2
                    for (int q = 0; q < nqw; q += 2) {
                        quad_acc_w(A2, AA2, sl[(2 * q) * 32 + lane], sl[(2 * q + 1) * 32 + lane], sW2[q], one2, acc1[0],
                                   acc0[0]);
                        quad_acc_w(A2, AA2, sl[(2 * q + 2) * 32 + lane], sl[(2 * q + 3) * 32 + lane], sW2[q + 1], one2,
                                   acc1[1], acc0[1]);
                    }
                    float q0, q1, q2, q3;
                    f2_unpack(f2_add(acc1[0], acc1[1]), q0, q1);
                    f2_unpack(f2_add(acc0[0], acc0[1]), q2, q3);
                    s1 = q0 + q1; s0 = q2 + q3;
                }
                if (s < p.S) {
                    float2* dst = p.sums + (size_t)i * p.S_pad + s;
                    if (p.accumulate) { const float2 o = *dst; s1 += o.x; s0 += o.y; }
                    *dst = make_float2(s1, s0);
                }
                continue;
            }
            if (risky) {
                float r1 = 0.f, r0 = 0.f;
                for (int j = 0; j + 1 < N; j += 2)
                    pair_acc<true>(A, p.DmT[(size_t)j * p.S_pad + s], p.DmT[(size_t)(j + 1) * p.S_pad + s], r1, r0);
                if (N & 1) single_acc(A, p.DmT[(size_t)(N - 1) * p.S_pad + s], r1, r0);
                if (s < p.S) {
                    float2* dst = p.sums + (size_t)i * p.S_pad + s;
                    if (p.accumulate) { const float2 o = *dst; r1 += o.x; r0 += o.y; }
                    *dst = make_float2(r1, r0);
                }
                continue;
            }
            const f32x2 A2 = f2_pack(A, A);
            const float AA = A * A;
            const f32x2 AA2 = f2_pack(AA, AA), AA2x2 = f2_pack(2.f * AA, 2.f * AA);
            f32x2 acc1[2] = {f2_pack(0.f, 0.f), f2_pack(0.f, 0.f)}, acc0[2] = {f2_pack(0.f, 0.f), f2_pack(0.f, 0.f)};
            float t1s = 0.f, t0s = 0.f;
            // chunks of 16 columns, the next one in flight while this one is consumed
            float va[16], vb[16];
            const int nch = nfull + (NTAIL > 0 ? 1 : 0);
            dm_ld16(sl, 0, nq, lane, va);
            for (int c = 0; c < nch; c += 2) {
                if (c + 1 < nch) dm_ld16(sl, c + 1, nq, lane, vb);
                if (c < nfull) chunk_sums<16>(va, A, A2, AA2, AA2x2, one2, two2, acc1, acc0, t1s, t0s);
                else if (NTAIL > 0) chunk_sums<NTAIL>(va, A, A2, AA2, AA2x2, one2, two2, acc1, acc0, t1s, t0s);
                if (c + 1 < nch) {
                    if (c + 2 < nch) dm_ld16(sl, c + 2, nq, lane, va);
                    if (c + 1 < nfull) chunk_sums<16>(vb, A, A2, AA2, AA2x2, one2, two2, acc1, acc0, t1s, t0s);
                    else if (NTAIL > 0) chunk_sums<NTAIL>(vb, A, A2, AA2, AA2x2, one2, two2, acc1, acc0, t1s, t0s);
                }
            }
            float q0, q1, q2, q3;
            f2_unpack(f2_add(acc1[0], acc1[1]), q0, q1);
            f2_unpack(f2_add(acc0[0], acc0[1]), q2, q3);
            float s1 = (q0 + q1) + t1s, s0 = (q2 + q3) + t0s;
            if (s < p.S) {
                float2* dst = p.sums + (size_t)i * p.S_pad + s;
                if (p.accumulate) { const float2 o = *dst; s1 += o.x; s0 += o.y; }
                *dst = make_float2(s1, s0);
            }
        }
    }
}

// What the launches of the unfused coalition kernel used (reported by dks_last_path): the fewest warps per CTA and the
// largest grid over the background chunks.
struct SharedLaunch { int warps, grid, chunks; };

// CTAs for n_rg row groups at `warps` warps per CTA: at least one per SM, and enough that every row group has a warp (a
// warp without a row group does nothing, so a grid of fewer warps than row groups would leave sums unwritten).  The
// kernels need no co-resident CTAs: every warp works on its own rows, so the extra CTAs simply run in later waves.
inline int shared_grid(int n_rg, int warps, int sm_count) {
    const int need = (n_rg + warps - 1) / warps;
    return need > sm_count ? need : sm_count;
}

inline cudaError_t launch_explain_shared_chunk(const SharedParams& p, int words, int sm_count, int max_smem, cudaStream_t stream,
                                               SharedLaunch* info) {
    const int n_rg = p.S_pad / 32;
    if (p.wn != nullptr) {
        // weighted background: the shared-memory kernel with the weighted slice (twice the bytes), W2 after the slices
        const size_t slice = dm_slice_bytes_w(p.N), w2 = sizeof(float2) * (size_t)dm_quads_w(p.N);
        int warps_used = (int)(((size_t)max_smem - 1024 - w2) / slice);
        if (warps_used > TM_MAX_WARPS) warps_used = TM_MAX_WARPS;
        const size_t smem = (size_t)warps_used * slice + w2;
        const int grid = shared_grid(n_rg, warps_used, sm_count);
        if (info->warps == 0 || warps_used < info->warps) info->warps = warps_used;
        if (grid > info->grid) info->grid = grid;
        cudaError_t err = cudaSuccess;
#define DKS_CASE_WT(W)                                                                                                        \
    err = cudaFuncSetAttribute(explain_shared_smem_kernel<0, W, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
    if (err == cudaSuccess) explain_shared_smem_kernel<0, W, true><<<grid, 32 * TM_MAX_WARPS, smem, stream>>>(p, warps_used);
        if (words == 1) { DKS_CASE_WT(1) }
        else if (words == 2) { DKS_CASE_WT(2) }
        else { DKS_CASE_WT(16) }
#undef DKS_CASE_WT
        return err;
    }
    // uniform background
    const size_t slice = dm_slice_bytes(p.N);
    int warps_used = (int)(((size_t)max_smem - 1024) / slice);
    if (warps_used > TM_MAX_WARPS) warps_used = TM_MAX_WARPS;
    const size_t smem = (size_t)warps_used * slice;
    const int grid = shared_grid(n_rg, warps_used, sm_count);
    if (info->warps == 0 || warps_used < info->warps) info->warps = warps_used;
    if (grid > info->grid) info->grid = grid;
    cudaError_t err = cudaSuccess;
    switch (p.N % 16) {
#define DKS_CASE_W(T, W)                                                                                                  \
    err = cudaFuncSetAttribute(explain_shared_smem_kernel<T, W>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
    if (err == cudaSuccess) explain_shared_smem_kernel<T, W><<<grid, 32 * TM_MAX_WARPS, smem, stream>>>(p, warps_used);
#define DKS_CASE(T)                                                                                          \
    case T:                                                                                                  \
        if (words == 1) { DKS_CASE_W(T, 1) }                                                                 \
        else if (words == 2) { DKS_CASE_W(T, 2) }                                                            \
        else { DKS_CASE_W(T, 16) }                                                                           \
        break;
        DKS_CASE(0) DKS_CASE(1) DKS_CASE(2) DKS_CASE(3) DKS_CASE(4) DKS_CASE(5) DKS_CASE(6) DKS_CASE(7)
        DKS_CASE(8) DKS_CASE(9) DKS_CASE(10) DKS_CASE(11) DKS_CASE(12) DKS_CASE(13) DKS_CASE(14) DKS_CASE(15)
#undef DKS_CASE
#undef DKS_CASE_W
    }
    return err;
}

// Backgrounds larger than MAXN rows go through in chunks of MAXN columns of Dm (one launch each, sums accumulated; a
// weighted chunk uses its own columns' weights).  Returns the number of launches (0 when one of them could not be
// configured).
inline int launch_explain_shared(SharedParams p, int words, int sm_count, int max_smem, cudaStream_t stream, SharedLaunch* info) {
    const int N = p.N;
    const float* dm = p.DmT;
    const float* wn = p.wn;
    int launches = 0;
    info->grid = 0; info->warps = 0;
    const bool use_cache = words > 2 && p.acache != nullptr && N > MAXN;
    for (int j0 = 0; j0 < N; j0 += MAXN, ++launches) {
        p.N = N - j0 < MAXN ? N - j0 : MAXN;
        p.DmT = dm + (size_t)j0 * p.S_pad;
        if (wn != nullptr) p.wn = wn + j0;
        p.accumulate = j0 > 0;
        p.acache_mode = use_cache ? (j0 == 0 ? 1 : 2) : 0;
        if (launch_explain_shared_chunk(p, words, sm_count, max_smem, stream, info) != cudaSuccess) return 0;
    }
    info->chunks = launches;
    return launches;
}

// Where the softmax, one-vs-rest and identity heads' y(i, c, s) comes from on the shared-plan path: the per-class sums of
// the class-sum coalition kernels (dks_multi.cuh), or the identity head's float64 nibble tables of XW - Bbar (prep_kernel),
// for which ey_c(s) = fnull_c + sum_k z_sk (XW_i[k][c] - Bbar[k][c]) needs no coalition kernel at all.  The exp head
// factorises the same way (DESIGN.md §3): ey(s) = 2^(a(s) + l(s)) with a(s) from the nibble tables of log2 e XW and
// l(s) = log2 sum_j w_j 2^(log2 e d(s, j)) from the plan (plan_exp_kernel) -- no coalition kernel either.
struct HeadSource {
    int act;                 // DKS_ACT_SOFTMAX, DKS_ACT_OVR, DKS_ACT_IDENTITY or DKS_ACT_EXP
    int ntab;                // nibble tables per class: ceil(G / 4)
    const float* msums;      // [n][C][S_pad] sum_j w'_j p_c(s, j), w'_j = N w_j
    const double* XT;        // [n][C][ntab][16]
    const double* ell;       // [S_pad] exp head: l(s)
};

// exp head, plan upload (M = G): l(s) = log2 e (m + ln sum_j w_j e^(d_j - m)) in float64, d_j = score_j - sum_{k in s} BW[j][k],
// m = max_j d_j (running, the sum rescaled when it grows), zero-weight background rows skipped.  Padding rows get 0.
template <int W>
__global__ void plan_exp_kernel(const uint64_t* __restrict__ z, int S, int S_pad, const double* __restrict__ BW,
                                const double* __restrict__ scores, const double* __restrict__ wbg, int N, int G, double scale,
                                double* __restrict__ ell) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S_pad) return;
    if (s >= S) { ell[s] = 0.0; return; }
    uint64_t zz[W];
#pragma unroll
    for (int q = 0; q < W; ++q) zz[q] = z[(size_t)s * W + q];
    double m = -INFINITY, e = 0.0;
    for (int j = 0; j < N; ++j) {
        const double wj = wbg[j];
        if (!(wj > 0.0)) continue;
        double c = 0.0;
        for (int k = 0; k < G; ++k)
            if (((W == 1 || k < 64 ? zz[0] : zz[W - 1]) >> (k & 63)) & 1ull) c += BW[(size_t)j * G + k];
        const double d = scores[j] - c;
        if (d > m) { e = e * exp(m - d) + wj; m = d; }
        else e += wj * exp(d - m);
    }
    ell[s] = scale * (m + log(e));
}

template <int W>
__device__ __forceinline__ double head_y(const HeadSource& h, int i, int c, int C, int s, int S_pad, const uint64_t* zrow,
                                         int link, double inv_n, double fn, double lf) {
    if (h.act != DKS_ACT_IDENTITY && h.act != DKS_ACT_EXP) {
        const float* ms = h.msums + (size_t)i * C * S_pad + s;
        const double e = (double)ms[(size_t)c * S_pad];
        if (link == DKS_LINK_LOGIT) {
            double rest = 0.0;                   // 1 - ey_c as the sum of the other classes: no cancellation
            for (int c2 = 0; c2 < C; ++c2) if (c2 != c) rest += (double)ms[(size_t)c2 * S_pad];
            return log(e / rest) - lf;
        }
        return e * inv_n - fn;
    }
    const double* xt = h.XT + ((size_t)i * C + c) * h.ntab * 16;
    double a0 = 0.0, a1 = 0.0;
    for (int t = 0; t < h.ntab; t += 2) {
        a0 += __ldg(xt + t * 16 + (int)((zrow[t >> 4] >> (4 * (t & 15))) & 15ull));
        if (t + 1 < h.ntab) a1 += __ldg(xt + (t + 1) * 16 + (int)((zrow[(t + 1) >> 4] >> (4 * ((t + 1) & 15))) & 15ull));
    }
    if (h.act == DKS_ACT_EXP) return link_f(exp2((a0 + a1) + __ldg(h.ell + s)), link) - lf;
    return link_f(fn + (a0 + a1), link) - lf;
}

// The 2^-40 fixed point holds |values| < 8e6.  Regression outputs have no such bound and small ones would lose relative
// precision, so the multi-output solves scale each (instance, output) by 2^e, exact, chosen so that `bound` (a bound of
// every fixed-point sum) becomes at most 2^22; the scale is undone before any absolute threshold.
__device__ __forceinline__ int fix_exponent(double bound) {
    if (!(bound > 0.0) || !isfinite(bound)) return 0;
    int ex;
    frexp(bound, &ex);                           // bound < 2^ex
    const int e = 22 - ex;
    return e < -1000 ? -1000 : (e > 1000 ? 1000 : e);
}

struct WlsSharedParams {
    int n, N, G, C, S, S_pad, link, uniform_w;
    HeadSource src;          // softmax / identity heads (the MULTI instantiation)
    const float2* sums;      // [n][S_pad]
    const uint64_t* z;
    const double* w;
    const double* ainv;      // [(G-1) x (G-1)]
    const double* dlink;     // [n][C]
    const double* linkfnull;
    const double* fnull;
    const int* list;
    const int* count;
    double* phi;             // [C][n][G]
    int* status;             // exp head (MULTI): a task whose y or delta is not finite is reported here, not solved
};

// ---- projection form of the solve for a shared plan ----------------------------------------------------------------
// beta = inv(A) E^T W (y - z_L delta) = P y - delta d,  P[k][s] = w_s sum_l inv(A)[k][l] (z_sl - z_sL),  d = P z_L.
// P depends only on the plan: computed once (float32 copy for the kernel, float64 for d).
__global__ void plan_pmat_kernel(const uint64_t* __restrict__ z, const double* __restrict__ w,
                                 const double* __restrict__ ainv, int S, int S_pad, int M, float* __restrict__ pmat) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int nA = M - 1, L = M - 1;
    if (idx >= nA * S_pad) return;
    const int k = idx / S_pad, s = idx - k * S_pad;
    double acc = 0.0;
    if (s < S) {
        const uint64_t zz = z[s];
        const int zl = (int)((zz >> L) & 1ull);
        for (int l = 0; l < nA; ++l) {
            const int e = (int)((zz >> l) & 1ull) - zl;
            if (e) acc += ainv[k * nA + l] * (double)e;
        }
        acc *= w[s];
    }
    pmat[idx] = (float)acc;
}
__global__ void plan_dvec_kernel(const uint64_t* __restrict__ z, const float* __restrict__ pmat, int S, int S_pad, int M,
                                 double* __restrict__ dvec) {
    // d = P z_L with the SAME float32 P the kernel multiplies y by, so the delta term is removed consistently
    const int k = blockIdx.x, nA = M - 1, L = M - 1;
    if (k >= nA) return;
    double acc = 0.0;
    for (int s = threadIdx.x; s < S; s += 32)
        if ((z[s] >> L) & 1ull) acc += (double)pmat[(size_t)k * S_pad + s];
    acc = warp_sum(acc);
    if (threadIdx.x == 0) dvec[k] = acc;
}

struct WlsPmatParams {
    int n, N, G, C, S, S_pad, link, uniform_w;
    const float2* sums;
    const float* pmat;       // [(G-1)][S_pad]
    const double* dvec;      // [(G-1)]
    const double* dlink;
    const double* linkfnull;
    const double* fnull;
    const int* list;
    const int* count;
    double* phi;
};
constexpr int PMAT_MAXK = 24;        // coefficients held in registers per thread
constexpr int PMAT_THREADS = 256;
inline int wls_pmat_kpad(int G) { return (G - 1 + 3) / 4 * 4; }       // coefficient rows padded to a multiple of four
inline size_t wls_pmat_smem(int G, int S_pad) { return (size_t)wls_pmat_kpad(G) * S_pad * sizeof(float); }

// Persistent CTAs; P resident in shared memory.  Per coalition row: y, then KPAD multiply-adds in float64.
// KPAD (compile time) = coefficients rounded up to a multiple of four, the padding rows of P are zero: the inner loop has
// no bounds checks (the checks were a fifth of the instructions).  P is staged as float32: a float64 copy (no float ->
// double conversions in the loop, but half the CTAs per SM) measured slower.
template <int KPAD>
__global__ void __launch_bounds__(PMAT_THREADS) wls_pmat_kernel(WlsPmatParams p) {
    extern __shared__ __align__(16) unsigned char s_praw[];
    float* s_P = reinterpret_cast<float*>(s_praw);                  // [KPAD][S_pad]
    __shared__ double s_part[PMAT_THREADS / 32][KPAD];
    __shared__ LogTabEntry s_logtab[DKS_LOGTAB_SIZE];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int G = p.G, nA = G - 1;
    const int cnt = *p.count;
    if ((int)blockIdx.x >= cnt) return;
    if (threadIdx.x < DKS_LOGTAB_SIZE) logtab_fill(s_logtab, threadIdx.x);
    for (int idx = threadIdx.x; idx < KPAD * p.S_pad; idx += PMAT_THREADS) s_P[idx] = idx < nA * p.S_pad ? p.pmat[idx] : 0.f;
    __syncthreads();
    const double lf1 = p.linkfnull[1], f1 = p.fnull[1], inv_n = 1.0 / (double)p.N;
    const size_t slab = (size_t)p.n * G;
    int i_next = p.list[blockIdx.x];
    double delta_next = p.dlink[(size_t)i_next * p.C + 1];
    constexpr int INFLIGHT = 8;                                        // independent loads in flight per thread
    for (int m = blockIdx.x; m < cnt; m += gridDim.x) {
        const int i = i_next;
        const double delta = delta_next;
        if (m + (int)gridDim.x < cnt) {            // next instance's index and delta: off the critical path
            i_next = p.list[m + gridDim.x];
            delta_next = p.dlink[(size_t)i_next * p.C + 1];
        }
        const float2* sums = p.sums + (size_t)i * p.S_pad;
        double Tk[KPAD];
#pragma unroll
        for (int k = 0; k < KPAD; ++k) Tk[k] = 0.0;
        for (int s0 = 0; s0 < p.S; s0 += INFLIGHT * PMAT_THREADS) {
            float2 a[INFLIGHT];
#pragma unroll
            for (int r = 0; r < INFLIGHT; ++r) {
                const int s = s0 + r * PMAT_THREADS + threadIdx.x;
                a[r] = s < p.S ? sums[s] : make_float2(1.f, 1.f);
            }
#pragma unroll
            for (int r = 0; r < INFLIGHT; ++r) {
                const int s = s0 + r * PMAT_THREADS + threadIdx.x;
                if (s < p.S) {
                    double y;
                    if (p.link == DKS_LINK_LOGIT) y = fast_log_ratio(a[r].x, a[r].y, s_logtab) - lf1;
                    else y = (p.uniform_w ? (double)a[r].x * inv_n : (double)a[r].x) - f1;
#pragma unroll
                    for (int k = 0; k < KPAD; ++k) Tk[k] = fma((double)s_P[(size_t)k * p.S_pad + s], y, Tk[k]);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < KPAD; ++k) {
            const double r = warp_sum(Tk[k]);
            if (lane == 0) s_part[wib][k] = r;
        }
        __syncthreads();
        if (wib == 0) {
            double beta = 0.0;
            if (lane < nA) {
#pragma unroll
                for (int wq = 0; wq < PMAT_THREADS / 32; ++wq) beta += s_part[wq][lane];      // fixed order: reproducible
                beta -= delta * p.dvec[lane];
            }
            const double sum = warp_sum(beta);
            if (lane < G) {
                double val = lane < nA ? beta : delta - sum;       // the eliminated (last) group takes the remainder
                if (fabs(val) < 1e-10) val = 0.0;
                p.phi[slab + (size_t)i * G + lane] = val;
                p.phi[(size_t)i * G + lane] = (val == 0.0) ? 0.0 : -val;
            }
        }
        __syncthreads();
    }
}

// picks the instantiation; returns false when P does not fit shared memory
inline bool launch_wls_pmat(const WlsPmatParams& p, int n, int sm_count, int max_smem, cudaStream_t stream, cudaError_t* err) {
    const size_t smem = wls_pmat_smem(p.G, p.S_pad);
    if (smem + 8192 > (size_t)max_smem) return false;
    int per_sm = (int)((size_t)max_smem / (smem + 8192));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 4) per_sm = 4;
    const int grid = n < sm_count * per_sm ? n : sm_count * per_sm;
    *err = cudaSuccess;
#define DKS_PM(K)                                                                                                  \
    case K:                                                                                                        \
        *err = cudaFuncSetAttribute(wls_pmat_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);   \
        if (*err == cudaSuccess) wls_pmat_kernel<K><<<grid, PMAT_THREADS, smem, stream>>>(p);                      \
        break;
    switch (wls_pmat_kpad(p.G)) {
        DKS_PM(4) DKS_PM(8) DKS_PM(12) DKS_PM(16) DKS_PM(20) DKS_PM(24)
        default: return false;
    }
#undef DKS_PM
    return true;
}

// Persistent CTAs of 8 warps, each looping over instances: y = link(ey) - link(fnull) per coalition, E^T W y in 2^-40
// fixed point (integer adds: exact, order-independent), beta = inv(E^T W E) (E^T W y), phi.
// MULTI: the softmax and identity heads -- one task per (instance, output), y from p.src, each output's phi written on its
// own (no antisymmetry), the fixed point scaled per task (fix_exponent).
constexpr int WLS_THREADS = 256;
inline size_t wls_shared_smem(int G) { return sizeof(double) * (size_t)(G - 1) * (G - 1); }
template <int W, bool MULTI = false>
__global__ void __launch_bounds__(WLS_THREADS) wls_shared_kernel(WlsSharedParams p) {
    extern __shared__ double s_ainv[];                   // [(G-1)][(G-1)]
    __shared__ long long s_part[WLS_THREADS / 32][64 * W];
    __shared__ double s_rhs[64 * W];
    __shared__ LogTabEntry s_logtab[DKS_LOGTAB_SIZE];
    __shared__ double s_bound[WLS_THREADS / 32];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int G = p.G, nA = G - 1, L = G - 1;
    const int nout = MULTI ? p.C : 1;
    const int cnt = *p.count * nout;
    if ((int)blockIdx.x >= cnt) return;
    if (threadIdx.x < DKS_LOGTAB_SIZE) logtab_fill(s_logtab, threadIdx.x);
    for (int idx = threadIdx.x; idx < nA * nA; idx += blockDim.x) s_ainv[idx] = p.ainv[idx];
    __syncthreads();
    const double lf1 = p.linkfnull[1], f1 = p.fnull[1], inv_n = 1.0 / (double)p.N;
    const size_t slab = (size_t)p.n * G;
    for (int m = blockIdx.x; m < cnt; m += gridDim.x) {
        const int i = p.list[MULTI ? m / nout : m];
        const int cls = MULTI ? m % nout : 1;
        const double delta = p.dlink[(size_t)i * p.C + cls];
        const float2* sums = p.sums + (size_t)i * p.S_pad;
        const double fnc = p.fnull[cls], lfc = p.linkfnull[cls];
        double sc = 1.0, isc = 1.0;
        if constexpr (MULTI) {
            double b = 0.0;                              // sum_s |w_s (y_s - z_sL delta)| bounds every coefficient's sum
            for (int s = threadIdx.x; s < p.S; s += WLS_THREADS) {
                const uint64_t* zrow = p.z + (size_t)s * W;
                const bool zl = (zrow[L >> 6] >> (L & 63)) & 1ull;
                const double y = head_y<W>(p.src, i, cls, p.C, s, p.S_pad, zrow, p.link, inv_n, fnc, lfc);
                b += fabs(p.w[s] * (y - (zl ? delta : 0.0)));
            }
            b = warp_sum(b);
            if (lane == 0) s_bound[wib] = b;
            // exp head: any non-finite y or delta makes the bound non-finite; the task is reported and skipped (the barrier
            // is the same for every thread, so is the decision)
            if (__syncthreads_or(p.src.act == DKS_ACT_EXP && !isfinite(b))) {
                if (threadIdx.x == 0 && atomicCAS(&p.status[0], 0, DKS_ERR_NUMERIC) == 0) p.status[1] = i;
                continue;
            }
            double tot = 0.0;
#pragma unroll
            for (int wq = 0; wq < WLS_THREADS / 32; ++wq) tot += s_bound[wq];     // fixed order: the same e every run
            const int e = fix_exponent(tot);
            sc = ldexp(1.0, e); isc = ldexp(1.0, -e);
        }
        // thread handles coalitions tid, tid+256, ...; sixteen coefficients of E^T W y per pass over the rows
        for (int k0 = 0; k0 < nA; k0 += 16) {
            long long Tk[16];
#pragma unroll
            for (int k = 0; k < 16; ++k) Tk[k] = 0;
#pragma unroll 2
            for (int s = threadIdx.x; s < p.S; s += WLS_THREADS) {
                double y;
                const uint64_t* zrow = p.z + (size_t)s * W;
                if constexpr (MULTI) {
                    y = head_y<W>(p.src, i, cls, p.C, s, p.S_pad, zrow, p.link, inv_n, fnc, lfc);
                } else {
                    const float2 a = sums[s];
                    if (p.link == DKS_LINK_LOGIT) y = fast_log_ratio(a.x, a.y, s_logtab) - lf1;
                    else y = (p.uniform_w ? (double)a.x * inv_n : (double)a.x) - f1;
                }
                const bool zl = (zrow[L >> 6] >> (L & 63)) & 1ull;
                const double v = MULTI ? p.w[s] * (y - (zl ? delta : 0.0)) * sc : p.w[s] * (y - (zl ? delta : 0.0));
                const uint64_t zw = zrow[k0 >> 6];               // a 16-bit window never straddles two words
                const uint32_t zb = (uint32_t)((zl ? ~zw : zw) >> (k0 & 63));
                const long long vi = zl ? -to_fix(v) : to_fix(v);
#pragma unroll
                for (int k = 0; k < 16; ++k)
                    if (k0 + k < nA && ((zb >> k) & 1u)) Tk[k] += vi;
            }
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                if (k0 + k < nA) {
                    const long long r = warp_sum_ll(Tk[k]);
                    if (lane == 0) s_part[wib][k0 + k] = r;
                }
            }
        }
        __syncthreads();
        if ((int)threadIdx.x < nA) {
            long long acc = 0;
#pragma unroll
            for (int wq = 0; wq < WLS_THREADS / 32; ++wq) acc += s_part[wq][threadIdx.x];
            s_rhs[threadIdx.x] = MULTI ? from_fix(acc) * isc : from_fix(acc);
        }
        __syncthreads();
        if (wib == 0) {
            double sum = 0.0;
            double beta[2 * W];
#pragma unroll
            for (int h = 0; h < 2 * W; ++h) beta[h] = 0.0;
#pragma unroll
            for (int h = 0; h < 2 * W; ++h) {
                const int k = lane + 32 * h;
                if (k < nA) {
                    double b0 = 0.0, b1 = 0.0;      // two chains: the dot product is latency bound otherwise
                    int l = 0;
                    for (; l + 1 < nA; l += 2) {
                        b0 = fma(s_ainv[k * nA + l], s_rhs[l], b0);
                        b1 = fma(s_ainv[k * nA + l + 1], s_rhs[l + 1], b1);
                    }
                    if (l < nA) b0 = fma(s_ainv[k * nA + l], s_rhs[l], b0);
                    beta[h] = b0 + b1;
                    sum += beta[h];
                }
            }
            sum = warp_sum(sum);
#pragma unroll
            for (int h = 0; h < 2 * W; ++h) {
                const int k = lane + 32 * h;
                if (k < G) {
                    double val = k < nA ? beta[h] : delta - sum;       // the eliminated (last) group takes the remainder
                    if (fabs(val) < 1e-10) val = 0.0;
                    p.phi[(size_t)cls * slab + (size_t)i * G + k] = val;
                    if (!MULTI) p.phi[(size_t)i * G + k] = (val == 0.0) ? 0.0 : -val;
                }
            }
        }
        // s_part / s_rhs / s_bound are rewritten only after the next task's row loop, which ends with __syncthreads
    }
}

}  // namespace shared_path
}  // namespace dks
