// Shared-plan fast path with the link and the projection solve FUSED into the coalition kernel.
//
// explain_shared_smem_kernel (dks_shared.cuh) writes (sum p1, sum p0) per (instance, coalition) to a global buffer (42 MB
// on the Adult-shaped workload) that wls_pmat_kernel reads back.  Here the same warp that produced a row's sums finishes
// the job: y = link(ey) - link(fnull) in place, then beta_k(i) = sum_s P[k][s] y(i, s) with P = inv(E^T W E) E^T W of the
// shared plan (float64, the warp's 32 rows of it resident in shared memory).  The sum over s runs across the lanes of a warp
// (lane = coalition row), so instead of shuffling per instance the warp parks y for a batch of B instances in shared
// memory ([row][instance], conflict-free both ways) and then turns the tile around on the FP64 tensor cores: eight
// DMMA.16x8x4 per eight instances sum P y over the 32 rows (P from shared memory, no shuffles).  Each warp adds its
// partial beta to a per-instance accumulator in 2^-40 FIXED POINT with relaxed 64-bit integer reductions (exact and
// order-independent: results are bit-reproducible whatever the scheduling), and that is all it does with it: no
// counter, no fence.  The end of the kernel makes every reduction visible to the next kernel on the stream,
// finish_fused_kernel, which applies the delta term, back-fills the eliminated group, snaps |phi| < 1e-10 and writes
// phi for both classes (and, on a multi-GPU run with push_in_kernel, stores them into every peer's gathered buffer over
// NVLink).  It also zeroes the accumulator, so the next launch needs no memset.
//
// A CTA holds `slices` row groups: each slice is the group's 32 rows of Dm (pair sums and pair products, as in
// explain_shared_smem_kernel) and of P.  kw warps share a slice and stream disjoint subsets of the instances through it,
// each with its own staging tile.  kw = 1 is one slice per warp, which fits the most row groups into a CTA (the largest
// plans); kw > 1 runs more warps per SM than slices of their own would fit.
#pragma once

#include "dks_shared.cuh"

namespace dks {
namespace shared_path {

// ---- per-row link table ----------------------------------------------------------------------------------------------
// With a shared plan and all groups varying, an instance enters coalition row s only through one scalar, x = a(i, s) + dme[s]:
//     y(i, s) + link(fnull) = L_s(x) = ln sum_j w'_j / (1 + 2^x Dm(s, j)) - ln sum_j w'_j 2^x Dm(s, j) / (1 + 2^x Dm(s, j))
// (identity link: sum_j w'_j / (1 + 2^x Dm(s, j)) / N), with w'_j = N w_j.  L_s depends on the plan and the background only,
// so dks_set_shared_plan tabulates it per row in float64 (DESIGN.md 5.0.1), and the fused kernel reads y from the table in a
// constant number of operations instead of summing N sigmoids.  Row s covers [x_lo, x_lo + nint h): x_lo is
// -LTAB_MARGIN - max_j log2 Dm(s, j) rounded down to the grid, the end is at or past LTAB_MARGIN - min_j log2 Dm(s, j) (columns
// of zero weight excluded).  Beyond either end every 2^x Dm is below 2^-33 or above 2^33; the kernel takes the exact loop
// there.  Interval k holds the degree-5 polynomial in t = (x - x_lo) / h - k in [0, 1) through L_s at six Chebyshev nodes:
// c0, c1 in float64, c2 .. c5 (at most ~1e-2) in float32, 32 bytes.  The build evaluates every interval against float64
// L_s at t = 0, t = 1 and midway between consecutive nodes, exactly as the kernel evaluates it; a plan that misses LTAB_TOL
// at h = 1/4 is rebuilt at h = 1/8, and one that misses it again, or whose table would pass LTAB_BUDGET bytes, has no table.
constexpr double LTAB_MARGIN = 33.0;
constexpr double LTAB_TOL = 1e-9;
constexpr size_t LTAB_BUDGET = (size_t)256 << 20;
constexpr int LTAB_NODES = 6;

struct __align__(16) LinkTabEntry { double c0, c1; float c2, c3, c4, c5; };
struct __align__(16) LinkTabRow { double x_lo; int off, nint; };       // nint = 0: padding row
static_assert(sizeof(LinkTabEntry) == 32, "one interval is 32 bytes");

// the fitting nodes in [0, 1] and the inverse of their Vandermonde matrix (monomial coefficients from node values)
struct LinkTabFit { double t[LTAB_NODES]; double vinv[LTAB_NODES * LTAB_NODES]; };

__host__ __device__ __forceinline__ double ltab_poly(const LinkTabEntry& e, double t) {
    const float tf = (float)t;
    const float q = fmaf(tf, fmaf(tf, fmaf(tf, e.c5, e.c4), e.c3), e.c2);
    return fma(t, fma(t, (double)q, e.c1), e.c0);
}

// float64 L_s(x) from the row's log2 Dm (ld, stride S_pad); wd = w'_j, NULL for a uniform background.  With u = 2^z, z = x +
// log2 Dm: p1 = 1 / (1 + u) and p0 = 1 / (1 + 1 / u) from e = 2^-|z| (no overflow, no cancellation)
__device__ double ltab_exact(double x, const double* __restrict__ ld, int S_pad, const double* __restrict__ wd, int N, int link) {
    double s1 = 0.0, s0 = 0.0;
    for (int j = 0; j < N; ++j) {
        const double w = wd ? wd[j] : 1.0;
        const double z = x + ld[(size_t)j * S_pad];
        const double e = exp2(-fabs(z));
        const double r = w / (1.0 + e);
        if (z > 0.0) { s1 += e * r; s0 += r; }
        else { s1 += r; s0 += e * r; }
    }
    return link == DKS_LINK_LOGIT ? log(s1) - log(s0) : s1 / (double)N;
}

// per row: log2 Dm in float64 (the exponents plan_dm_kernel rounds to float32) and the row's domain at step h
__global__ void plan_ltab_rows_kernel(const uint64_t* __restrict__ z, int S, int S_pad, const double* __restrict__ BW,
                                      const double* __restrict__ scores, int N, int G, double scale,
                                      const double* __restrict__ dme, const double* __restrict__ wd, double h,
                                      double* __restrict__ ld, LinkTabRow* __restrict__ rows) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S_pad) return;
    LinkTabRow r;
    r.x_lo = 0.0; r.off = 0; r.nint = 0;
    if (s < S) {
        double lmin = 1.0e300, lmax = -1.0e300;
        for (int j = 0; j < N; ++j) {
            const double v = plan_d(z + s, BW, scores, j, G, scale) - dme[s];
            ld[(size_t)j * S_pad + s] = v;
            if (wd == nullptr || wd[j] > 0.0) { lmin = fmin(lmin, v); lmax = fmax(lmax, v); }
        }
        r.x_lo = floor((-LTAB_MARGIN - lmax) / h) * h;
        const double n = ceil((LTAB_MARGIN - lmin - r.x_lo) / h);
        r.nint = n < 1.0e9 ? (int)n : 1000000000;         // the host's budget check turns such a plan down
    }
    rows[s] = r;
}

// one thread per interval (blockIdx.x = row): fit, store, and the largest error against float64 L_s (as ordered bits)
__global__ void plan_ltab_fit_kernel(LinkTabFit f, const LinkTabRow* __restrict__ rows, const double* __restrict__ ld, int S_pad,
                                     const double* __restrict__ wd, int N, int link, double h, LinkTabEntry* __restrict__ tab,
                                     unsigned long long* __restrict__ maxerr) {
    const int s = blockIdx.x, k = blockIdx.y * blockDim.x + threadIdx.x;
    const LinkTabRow r = rows[s];
    if (k >= r.nint) return;
    const double x0 = r.x_lo + (double)k * h;
    const double* lds = ld + s;
    double fv[LTAB_NODES], c[LTAB_NODES];
    for (int m = 0; m < LTAB_NODES; ++m) fv[m] = ltab_exact(x0 + h * f.t[m], lds, S_pad, wd, N, link);
    for (int a = 0; a < LTAB_NODES; ++a) {
        double v = 0.0;
        for (int m = 0; m < LTAB_NODES; ++m) v = fma(f.vinv[a * LTAB_NODES + m], fv[m], v);
        c[a] = v;
    }
    LinkTabEntry e;
    e.c0 = c[0]; e.c1 = c[1]; e.c2 = (float)c[2]; e.c3 = (float)c[3]; e.c4 = (float)c[4]; e.c5 = (float)c[5];
    double err = 0.0;
    for (int q = 0; q <= LTAB_NODES; ++q) {
        const double t = q == 0 ? 0.0 : (q == LTAB_NODES ? 1.0 : 0.5 * (f.t[q - 1] + f.t[q]));
        err = fmax(err, fabs(ltab_poly(e, t) - ltab_exact(x0 + h * t, lds, S_pad, wd, N, link)));
    }
    if (!(err <= 1.0)) err = 1.0;                          // NaN or worse: the plan fails verification
    atomicMax(maxerr, (unsigned long long)__double_as_longlong(err));
    tab[(size_t)r.off + k] = e;
}

struct FusedParams {
    int n, N, G, C, S, S_pad, link, B;
    double scale;
    const float* DmT;        // [N][S_pad]
    const double* dme;       // [S_pad]
    const uint64_t* z;       // [S]
    const double* XT;        // [n][ceil(G/4)][16]
    const int* list;
    const int* count;
    const double* pmat64;    // [S_pad][KPAD] row s: P[0..KPAD)[s], zero beyond G-1 coefficients and beyond S rows
    const double* dvec;      // [KPAD] P z_L (float64 P)
    const double* dlink;     // [n][C]
    const double* linkfnull;
    const double* fnull;
    long long* acc;          // [n][KPAD] fixed-point partial beta (zero between launches)
    const float* wn;         // [N] weighted backgrounds: N w_j (the weighted instantiations only; dks_shared.cuh)
    const LinkTabEntry* ltab;        // the plan's link table (below), NULL: every pass takes the exact loop
    const LinkTabRow* ltab_rows;     // [S_pad]
    double ltab_inv_h;               // 1 / grid step
    unsigned long long* ltab_fb;     // passes that left the table's domain and took the exact loop (cumulative)
};

// one 16-column chunk whose valid columns are a run-time count: nq full quads (pair sums / products), then rem < 4 raw
// columns starting at column 4 * nq
__device__ __forceinline__ void chunk_sums_rt(const float (&v)[16], int nq, int rem, float A, f32x2 A2, f32x2 AA2, f32x2 AA2x2,
                                              f32x2 one2, f32x2 two2, f32x2 (&acc1)[2], f32x2 (&acc0)[2], float& t1s, float& t0s) {
    if (nq > 0) quad_acc_sq(A2, AA2, AA2x2, f2_pack(v[0], v[1]), f2_pack(v[2], v[3]), one2, two2, acc1[0], acc0[0]);
    if (nq > 1) quad_acc_sq(A2, AA2, AA2x2, f2_pack(v[4], v[5]), f2_pack(v[6], v[7]), one2, two2, acc1[1], acc0[1]);
    if (nq > 2) quad_acc_sq(A2, AA2, AA2x2, f2_pack(v[8], v[9]), f2_pack(v[10], v[11]), one2, two2, acc1[0], acc0[0]);
    if (rem) {
        float r0, r1, r2;
        switch (nq) {
            case 0: r0 = v[0]; r1 = v[1]; r2 = v[2]; break;
            case 1: r0 = v[4]; r1 = v[5]; r2 = v[6]; break;
            case 2: r0 = v[8]; r1 = v[9]; r2 = v[10]; break;
            default: r0 = v[12]; r1 = v[13]; r2 = v[14]; break;
        }
        if (rem >= 2) pair_acc<false>(A, r0, r1, t1s, t0s);
        if (rem & 1) single_acc(A, rem == 1 ? r0 : r2, t1s, t0s);
    }
}

// every row group has delivered: phi of both classes for the count[0] instances of `list`, from the fixed-point
// accumulators explain_shared_fused_kernel left (its end made every reduction visible), then the accumulators zeroed for
// the next launch.  Sixteen lanes per instance (G <= 16 on the fused path): lane k takes coefficient k, lane nA the
// eliminated group, so each class's phi row is one contiguous store.  Every lane forms the eliminated group's sum over
// k = 0 .. nA - 1 in order from shuffles, the operations and order of a one-lane loop.  peers: on a multi-GPU run with
// push_in_kernel, the rows also go to every peer's gathered buffer (npeers = 0 otherwise).
__global__ void __launch_bounds__(256) finish_fused_kernel(const int* __restrict__ list, const int* __restrict__ count,
                                                           long long* __restrict__ acc, int kpad, const double* __restrict__ dvec,
                                                           const double* __restrict__ dlink, int n, int G, int C,
                                                           double* __restrict__ phi, PeerPush peers) {
    const int t = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 4), k = threadIdx.x & 15;
    if (t >= *count) return;                                   // the same on the instance's sixteen lanes
    const unsigned half = 0xffffu << (threadIdx.x & 16);
    const int i = list[t], nA = G - 1;
    long long* a = acc + (size_t)i * kpad;
    const double delta = dlink[(size_t)i * C + 1];
    double val = 0.0;
    if (k < nA) {
        val = from_fix(a[k]) - delta * dvec[k];
        a[k] = 0;
    }
    double sum = 0.0;
    for (int m = 0; m < nA; ++m) sum += __shfl_sync(half, val, m, 16);
    if (k == nA) val = delta - sum;                            // the eliminated (last) group takes the remainder
    if (k > nA) return;
    if (fabs(val) < 1e-10) val = 0.0;
    const double neg = (val == 0.0) ? 0.0 : -val;
    const size_t slab = (size_t)n * G, off = (size_t)i * G + k;
    phi[slab + off] = val;
    phi[off] = neg;
    for (int r = 0; r < peers.npeers; ++r) {
        peers.dst[r][slab + off] = val;
        peers.dst[r][off] = neg;
    }
}

// weighted: the weighted slice (twice the bytes) and the per-CTA W2 array of dks_shared.cuh
inline size_t fused_smem_bytes(int slices, int kw, int kpad, int B, int N, bool weighted = false) {
    return (size_t)slices * (weighted ? dm_slice_bytes_w(N) : dm_slice_bytes(N)) + (size_t)slices * 32 * kpad * sizeof(double) +
           (size_t)slices * kw * 32 * (B + 1) * sizeof(double) + DKS_LOGTAB_SIZE * sizeof(LogTabEntry) +
           (weighted ? sizeof(float2) * (size_t)dm_quads_w(N) : 0);
}

// one slice per CTA with the flat split of the kernel below: a second slice of Dm and P (no second set of staging tiles)
inline size_t fused_flat_smem_bytes(int kw, int kpad, int B, int N, bool weighted = false) {
    return fused_smem_bytes(1, kw, kpad, B, N, weighted) + (weighted ? dm_slice_bytes_w(N) : dm_slice_bytes(N)) +
           (size_t)32 * kpad * sizeof(double);
}

// NCT: background rows at compile time (0 = run-time p.N): with NCT the chunk loop unrolls completely (static shared-memory
// offsets, no loop control, the tail folded).  B (instances parked per warp) is a power of two.  Warp w of a CTA works on
// slice w / kw; warps from slices * kw on idle.  WT: weighted background (quad_acc_w, dks_shared.cuh).
// flat (one slice per CTA, at least as many CTAs as row groups): instead of whole replicas of a row group, CTA c takes the
// c-th of gridDim.x equal contiguous ranges of the (row group, instance ordinal) pairs, row group major, and its kw warps
// split that range into equal contiguous pieces.  A range spans at most two row groups, so the CTA holds two slices of Dm
// and P; every CTA of the grid works, however the row groups divide into the SMs.  Each (instance, row group) pair is
// still delivered exactly once.
template <int NCT, int KPAD, int NWARPS, bool WT = false>
__global__ void __launch_bounds__(32 * NWARPS, 1) explain_shared_fused_kernel(FusedParams p, int slices, int kw, int flat) {
    constexpr int NI = 1;                                // instances per pass over the slice
    extern __shared__ __align__(16) unsigned char fsm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int slice = warp / kw, sub = warp - slice * kw;
    const int B = p.B, ystride = B + 1;
    const int nq = dm_quads(NCT ? NCT : p.N);
    const int nqw = dm_quads_w(NCT ? NCT : p.N);                                 // weighted: quads of the slice (even)
    const int sq4 = WT ? 2 * nqw : nq;                                           // float4 per lane and slice
    const int nsl = flat ? 2 : slices;                                            // slices of Dm and P held
    float4* sDm = reinterpret_cast<float4*>(fsm);                                // [nsl][sq4][32]
    double* sP = reinterpret_cast<double*>(sDm + (size_t)nsl * sq4 * 32);        // [nsl][32][KPAD]
    double* sY = sP + (size_t)nsl * 32 * KPAD;                                   // [slices * kw][32][B + 1]
    LogTabEntry* s_logtab = reinterpret_cast<LogTabEntry*>(sY + (size_t)slices * kw * 32 * ystride);
    float2* sW2 = reinterpret_cast<float2*>(s_logtab + DKS_LOGTAB_SIZE);         // weighted: [nqw]
    if (threadIdx.x >= 64 && threadIdx.x < 64 + DKS_LOGTAB_SIZE) logtab_fill(s_logtab, threadIdx.x - 64);
    if constexpr (WT) {
        for (int q = threadIdx.x; q < nqw; q += blockDim.x) sW2[q] = w2_quad(p.wn, NCT ? NCT : p.N, q);
    }

    constexpr int MAXCH = MAXN / 16;
    const int N = NCT ? NCT : p.N;
    const int nfull = N / 16, ntail = N - nfull * 16;
    const int nch = nfull + (ntail > 0 ? 1 : 0);
    const int n_rg = p.S_pad / 32;                       // row groups
    const int nparts = gridDim.x * slices / n_rg;        // replicas of every row group (>= 1: checked by the host)
    const int gs = blockIdx.x * slices + slice;
    const bool active = slice < slices && (flat || gs < nparts * n_rg);
    double* sYw = sY + (size_t)warp * 32 * ystride;
    // flat: the CTA's pairs [c0, c1) and this warp's [u0, u1); row groups rg_lo .. rg_lo + 1 in slices 0 and 1
    const int cnt_f = flat ? *p.count : 0;
    const long long U = (long long)n_rg * cnt_f;
    const long long c0 = U * blockIdx.x / gridDim.x, c1 = U * (blockIdx.x + 1) / gridDim.x;
    const long long u0 = c0 + (c1 - c0) * sub / kw, u1 = c0 + (c1 - c0) * (sub + 1) / kw;
    const int rg_lo = cnt_f > 0 ? (int)(c0 / cnt_f) : 0;
    const int nfill = flat ? (c1 > c0 ? (int)((c1 - 1) / cnt_f) - rg_lo + 1 : 0) : 1;
    for (int f = 0; active && f < nfill; ++f) {
        const int fs = flat ? f : slice;
        const int rg = flat ? rg_lo + f : gs % n_rg;
        const int s = rg * 32 + lane;
        double* sPw = sP + (size_t)fs * 32 * KPAD;
        float4* sl = sDm + (size_t)fs * sq4 * 32;
        // ---- the slice's 32 rows of P and of Dm, split over its kw warps; Dm as pair sums and pair products per quad of
        // columns (0,2) (1,3)
        const double* src = p.pmat64 + (size_t)rg * 32 * KPAD;     // the slice's 32 rows are contiguous
        for (int idx = sub * 32 + lane; idx < 32 * KPAD; idx += 32 * kw) sPw[idx] = src[idx];
        if constexpr (WT) {
            for (int q = sub; q < nqw; q += kw) {
                float4 sq, xy;
                dm_quad_w(p.DmT, p.wn, N, p.S_pad, s, q, sq, xy);
                sl[(2 * q) * 32 + lane] = sq;
                sl[(2 * q + 1) * 32 + lane] = xy;
            }
        }
#pragma unroll
        for (int c = 0; c < MAXCH; ++c) {
            if (!WT && c < nch && c % kw == sub) {
                float v[16];
#pragma unroll
                for (int jj = 0; jj < 16; ++jj) {
                    const int j = c * 16 + jj;
                    v[jj] = j < N ? p.DmT[(size_t)j * p.S_pad + s] : 0.f;
                }
                const int nv = c < nfull ? 16 : ntail;
#pragma unroll
                for (int jj = 0; jj < 16; jj += 4) {
                    if (jj + 3 < nv) {
                        const float d0 = v[jj], d1 = v[jj + 1], d2 = v[jj + 2], d3 = v[jj + 3];
                        v[jj] = d0 + d2; v[jj + 1] = d1 + d3; v[jj + 2] = d0 * d2; v[jj + 3] = d1 * d3;
                    }
                }
                dm_st16(sl, c, nq, lane, v);
            }
        }
    }
    __syncthreads();

    if (active) {
        const int cnt = *p.count;
        const int G = p.G, nA = G - 1;
        const int nq_t = ntail >> 2, rem_t = ntail & 3;
        // segments of this warp's work: one row group each, instance ordinals first, first + stride, ...; flat: up to two
        // row groups, contiguous ordinals; otherwise the part's instances dealt round-robin over the slice's kw warps
        const long long seg_end = flat && u0 < u1 ? ((u0 / cnt) + 1) * cnt : 0;
        const int nseg = flat ? (u0 < u1 ? (u1 > seg_end ? 2 : 1) : 0) : 1;
        // what the segments need of the flat range, formed once (the 64-bit bounds are not held through the passes)
        const int rg0 = flat ? (u0 < u1 ? (int)(u0 / cnt) : 0) : gs % n_rg;
        const int first0 = flat ? (u0 < u1 ? (int)(u0 % cnt) : 0) : gs / n_rg + sub * nparts;
        const int my_n0 = flat ? (int)((u1 < seg_end ? u1 : seg_end) - u0) : 0, my_n1 = flat ? (int)(u1 - seg_end) : 0;
        for (int seg = 0; seg < nseg; ++seg) {
            const int rg = rg0 + seg;
            const int s = rg * 32 + lane;
            const int fs = flat ? rg - rg_lo : slice;
            const double* sPw = sP + (size_t)fs * 32 * KPAD;
            const float4* sl = sDm + (size_t)fs * sq4 * 32;
            const int first = seg == 0 ? first0 : 0;
            const int stride = flat ? 1 : nparts * kw;
            const int my_n = flat ? (seg == 0 ? my_n0 : my_n1) : (first < cnt ? (cnt - first + stride - 1) / stride : 0);
            const double es = p.dme[s];
            const uint64_t zz = s < p.S ? p.z[s] : 0ull;
            const int ntab = (G + 3) / 4;                     // <= 4 (the host sends wider problems down the unfused path)
            const f32x2 one2 = f2_pack(1.f, 1.f), two2 = f2_pack(2.f, 2.f);
            const double yf = p.link == DKS_LINK_LOGIT ? p.linkfnull[1] : p.fnull[1], inv_n = 1.0 / (double)N;   // link(fnull)
            const bool row_ok = s < p.S;
            const int bmask = B - 1;

            // ---- the turn-around on the FP64 tensor cores: eight instances of the batch per round, beta = P y over the
            // warp's 32 rows as eight mma.m16n8k4 k-steps (rows 4 kk .. 4 kk + 3, kk = 0 .. 7, in order).  Lane (tig =
            // lane & 3, gid = lane >> 2) feeds P[gid][s] and P[gid + 8][s] (A) and y of instance gid (B) at row
            // s = 4 kk + tig, and receives coefficients gid and gid + 8 of instances 2 tig and 2 tig + 1 (D).  A D column
            // depends on its own B column only, so an instance's partial does not depend on the batch it shares; the
            // partial goes to the instance's accumulator (finish_fused_kernel reads the sums once the kernel has ended)
            auto flush = [&](int bstart, int bcount) {
                const int tig = lane & 3, gid = lane >> 2;
                for (int b0 = 0; b0 < bcount; b0 += 8) {
                    double d0 = 0.0, d1 = 0.0, d2 = 0.0, d3 = 0.0;
                    // by two: fully unrolled, some instantiations spill at their register bound
#pragma unroll 2
                    for (int kk = 0; kk < 8; ++kk) {
                        const int sr = 4 * kk + tig;
                        const double a0 = sPw[sr * KPAD + gid], a1 = gid + 8 < KPAD ? sPw[sr * KPAD + gid + 8] : 0.0;
                        const double y = sYw[sr * ystride + b0 + gid];      // columns past bcount: not delivered
                        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, "
                                     "{%0,%1,%2,%3};"
                                     : "+d"(d0), "+d"(d1), "+d"(d2), "+d"(d3) : "d"(a0), "d"(a1), "d"(y));
                    }
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int b = b0 + 2 * tig + h;
                        if (b < bcount) {
                            long long* acc = p.acc + (size_t)p.list[first + (bstart + b) * stride] * KPAD;
                            if (gid < nA)
                                asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(acc + gid),
                                             "l"((unsigned long long)to_fix(h ? d1 : d0)) : "memory");
                            if (gid + 8 < nA)
                                asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(acc + gid + 8),
                                             "l"((unsigned long long)to_fix(h ? d3 : d2)) : "memory");
                        }
                    }
                }
            };

            // a(i, s) = sum over the row's nibbles of one table entry each; the entries of the NEXT instance are loaded one
            // iteration ahead (the offsets depend on the row only), the instance index two ahead.  No branches: tables the
            // problem does not have point at entry [0][0] (the empty subset: exactly 0.0), and past the last instance the
            // loads repeat the last one.
            const size_t xstride = (size_t)ntab * 16;
            const double* xb0 = p.XT + (int)(zz & 15ull);
            const double* xb1 = p.XT + (ntab > 1 ? 16 + (int)((zz >> 4) & 15ull) : 0);
            const double* xb2 = p.XT + (ntab > 2 ? 32 + (int)((zz >> 8) & 15ull) : 0);
            const double* xb3 = p.XT + (ntab > 3 ? 48 + (int)((zz >> 12) & 15ull) : 0);
            const int last_it = my_n > 0 ? my_n - 1 : 0;
            // NI instances share one pass over the warp's rows of Dm: instance ordinals it .. it + NI - 1
            int i_nx[NI];
            double nx[NI][4];
#pragma unroll
            for (int u = 0; u < NI; ++u) {
                const int o0 = u < last_it ? u : last_it, o1 = NI + u < last_it ? NI + u : last_it;
                i_nx[u] = my_n > 0 ? p.list[first + o1 * stride] : 0;
                nx[u][0] = nx[u][1] = nx[u][2] = nx[u][3] = 0.0;
                if (my_n > 0) {
                    const size_t o = (size_t)p.list[first + o0 * stride] * xstride;
                    nx[u][0] = __ldg(xb0 + o); nx[u][1] = __ldg(xb1 + o); nx[u][2] = __ldg(xb2 + o); nx[u][3] = __ldg(xb3 + o);
                }
            }

            // the row's domain in the link table (a padding row has none and needs none: its y is 0).  With the background
            // size compiled in it stays in registers for the whole segment; the run-time-N instantiations reload it every
            // pass (an L1 hit), because holding it through their exact loop spills at 20 warps
            LinkTabRow trow_seg;
            trow_seg.x_lo = 0.0; trow_seg.off = 0; trow_seg.nint = 0;
            if (NCT != 0 && p.ltab != nullptr && row_ok) trow_seg = p.ltab_rows[s];

            for (int it = 0; it < my_n; it += NI) {
                double a[NI], v[NI], y[NI];
                bool in_tab = true;
                LinkTabRow trow = trow_seg;
                if (NCT == 0 && p.ltab != nullptr && row_ok) trow = p.ltab_rows[s];
#pragma unroll
                for (int u = 0; u < NI; ++u) {
                    a[u] = ((nx[u][0] + nx[u][1]) + (nx[u][2] + nx[u][3])) + es;
                    {
                        const size_t o = (size_t)i_nx[u] * xstride;
                        nx[u][0] = __ldg(xb0 + o); nx[u][1] = __ldg(xb1 + o); nx[u][2] = __ldg(xb2 + o); nx[u][3] = __ldg(xb3 + o);
                        const int it2 = it + 2 * NI + u < last_it ? it + 2 * NI + u : last_it;
                        i_nx[u] = p.list[first + it2 * stride];
                    }
                    v[u] = (a[u] - trow.x_lo) * p.ltab_inv_h;
                    in_tab = in_tab && (!row_ok || (v[u] >= 0.0 && v[u] < (double)trow.nint));
                }
                if (p.ltab != nullptr && __all_sync(0xffffffffu, in_tab)) {
                    // y from the row's table: one 32-byte interval and a Horner evaluation
#pragma unroll
                    for (int u = 0; u < NI; ++u) {
                        y[u] = 0.0;
                        if (row_ok) {
                            const int k = (int)v[u];
                            const LinkTabEntry* ep = p.ltab + (size_t)trow.off + k;
                            const double2 c01 = __ldg(reinterpret_cast<const double2*>(ep));
                            const float4 c25 = __ldg(reinterpret_cast<const float4*>(ep) + 1);
                            LinkTabEntry e;
                            e.c0 = c01.x; e.c1 = c01.y; e.c2 = c25.x; e.c3 = c25.y; e.c4 = c25.z; e.c5 = c25.w;
                            y[u] = ltab_poly(e, v[u] - (double)k) - yf;
                        }
                    }
                } else {
                    // a lane's x is outside its row's table (or the plan has none): the exact loop over the background
                    if (p.ltab != nullptr && lane == 0) atomicAdd(p.ltab_fb, 1ull);
                    float A[NI];
                    bool risky_l = false;
#pragma unroll
                    for (int u = 0; u < NI; ++u) {
                        // A = 2^a = 2^n 2^f, n = rint(a) through the 1.5 * 2^52 trick (no conversion instructions), |f| <= 1/2; the
                        // exponent is clamped to [-120, 120] (saturated scores; the clamped scalar path below takes A > 1e18)
                        const double tm = a[u] + 6755399441055744.0;
                        int an_i = __double2loint(tm);
                        an_i = an_i < -120 ? -120 : (an_i > 120 ? 120 : an_i);
                        A[u] = ex2_approx((float)(a[u] - (tm - 6755399441055744.0))) * __int_as_float((127 + an_i) << 23);
                        risky_l = risky_l || A[u] > 1.0e18f;
                    }
                    float s1[NI], s0[NI];
                    if constexpr (WT) {
                        if (__any_sync(0xffffffffu, risky_l)) {
#pragma unroll
                            for (int u = 0; u < NI; ++u) row_sums_clamped_w(p.DmT, p.wn, N, p.S_pad, s, A[u], s1[u], s0[u]);
                        } else {
                            // every quad of the slice (all columns compiled in with NCT), two accumulator chains per instance
                            f32x2 A2[NI], AA2[NI], acc1[NI][2], acc0[NI][2];
#pragma unroll
                            for (int u = 0; u < NI; ++u) {
                                const float AA = A[u] * A[u];
                                A2[u] = f2_pack(A[u], A[u]); AA2[u] = f2_pack(AA, AA);
                                acc1[u][0] = acc1[u][1] = acc0[u][0] = acc0[u][1] = f2_pack(0.f, 0.f);
                            }
                            // quad q on accumulator chain h (a constant after unrolling: the accumulators stay in registers)
                            auto quad = [&](int q, int h) {
                                const float4 sq = sl[(2 * q) * 32 + lane], xy = sl[(2 * q + 1) * 32 + lane];
                                const float2 w2 = sW2[q];
#pragma unroll
                                for (int u = 0; u < NI; ++u) quad_acc_w(A2[u], AA2[u], sq, xy, w2, one2, acc1[u][h], acc0[u][h]);
                            };
                            if (NCT) {
#pragma unroll
                                for (int q = 0; q < dm_quads(NCT); ++q) quad(q, q & 1);
                            } else {
                                // run-time N: the slice's even number of quads in pairs (a zero quad past an odd count adds 0)
#pragma unroll 2
                                for (int q = 0; q < nqw; q += 2) { quad(q, 0); quad(q + 1, 1); }
                            }
#pragma unroll
                            for (int u = 0; u < NI; ++u) {
                                float q0, q1, q2, q3;
                                f2_unpack(f2_add(acc1[u][0], acc1[u][1]), q0, q1);
                                f2_unpack(f2_add(acc0[u][0], acc0[u][1]), q2, q3);
                                s1[u] = q0 + q1;
                                s0[u] = q2 + q3;
                            }
                        }
                    } else if (__any_sync(0xffffffffu, risky_l)) {
                        // A^2 would leave the fp32 range: clamped scalar path on the raw row from global memory (saturated scores)
#pragma unroll
                        for (int u = 0; u < NI; ++u) {
                            float r1 = 0.f, r0 = 0.f;
                            for (int j = 0; j + 1 < N; j += 2)
                                pair_acc<true>(A[u], p.DmT[(size_t)j * p.S_pad + s], p.DmT[(size_t)(j + 1) * p.S_pad + s], r1, r0);
                            if (N & 1) single_acc(A[u], p.DmT[(size_t)(N - 1) * p.S_pad + s], r1, r0);
                            s1[u] = r1; s0[u] = r0;
                        }
                    } else {
                        f32x2 A2[NI], AA2[NI], AA2x2[NI];
                        f32x2 acc1[NI][2], acc0[NI][2];
                        float t1s[NI], t0s[NI];
#pragma unroll
                        for (int u = 0; u < NI; ++u) {
                            const float AA = A[u] * A[u];
                            A2[u] = f2_pack(A[u], A[u]); AA2[u] = f2_pack(AA, AA); AA2x2[u] = f2_pack(2.f * AA, 2.f * AA);
                            acc1[u][0] = acc1[u][1] = acc0[u][0] = acc0[u][1] = f2_pack(0.f, 0.f);
                            t1s[u] = t0s[u] = 0.f;
                        }
                        float v[2][16];
                        dm_ld16(sl, 0, nq, lane, v[0]);
#pragma unroll
                        for (int c = 0; c < MAXCH; ++c) {
                            if (c < nch) {
                                if (c + 1 < nch) dm_ld16(sl, c + 1, nq, lane, v[(c + 1) & 1]);
#pragma unroll
                                for (int u = 0; u < NI; ++u) {
                                    if (c < nfull) chunk_sums<16>(v[c & 1], A[u], A2[u], AA2[u], AA2x2[u], one2, two2, acc1[u], acc0[u], t1s[u], t0s[u]);
                                    else chunk_sums_rt(v[c & 1], nq_t, rem_t, A[u], A2[u], AA2[u], AA2x2[u], one2, two2, acc1[u], acc0[u], t1s[u], t0s[u]);
                                }
                            }
                        }
#pragma unroll
                        for (int u = 0; u < NI; ++u) {
                            float q0, q1, q2, q3;
                            f2_unpack(f2_add(acc1[u][0], acc1[u][1]), q0, q1);
                            f2_unpack(f2_add(acc0[u][0], acc0[u][1]), q2, q3);
                            s1[u] = (q0 + q1) + t1s[u];
                            s0[u] = (q2 + q3) + t0s[u];
                        }
                    }
                    // ---- link in place
#pragma unroll
                    for (int u = 0; u < NI; ++u) {
                        y[u] = 0.0;
                        if (row_ok) {
                            if (p.link == DKS_LINK_LOGIT) y[u] = fast_log_ratio(s1[u], s0[u], s_logtab) - yf;
                            else y[u] = (double)s1[u] * inv_n - yf;
                        }
                    }
                }
                // ---- rows parked for the turn-around (B is a multiple of NI: a pass never straddles a batch)
#pragma unroll
                for (int u = 0; u < NI; ++u)
                    if (it + u < my_n) sYw[lane * ystride + ((it + u) & bmask)] = y[u];
                const int last_done = it + NI - 1 < last_it ? it + NI - 1 : last_it;      // last ordinal this pass completed
                const int slot = last_done & bmask;
                if (slot == bmask || last_done == last_it) {
                    __syncwarp();
                    flush(last_done - slot, slot + 1);
                    __syncwarp();
                }
            }
        }
    }
}

// P in float64, one row of KPAD coefficients per coalition: pmat64[s][k] = w_s sum_l inv(A)[k][l] (z_sl - z_sL)
__global__ void plan_pmat64_kernel(const uint64_t* __restrict__ z, const double* __restrict__ w,
                                   const double* __restrict__ ainv, int S, int S_pad, int M, int kpad,
                                   double* __restrict__ pmat64) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int nA = M - 1, L = M - 1;
    if (idx >= kpad * S_pad) return;
    const int s = idx / kpad, k = idx - s * kpad;
    double acc = 0.0;
    if (s < S && k < nA) {
        const uint64_t zz = z[s];
        const int zl = (int)((zz >> L) & 1ull);
        for (int l = 0; l < nA; ++l) {
            const int e = (int)((zz >> l) & 1ull) - zl;
            if (e) acc += ainv[k * nA + l] * (double)e;
        }
        acc *= w[s];
    }
    pmat64[idx] = acc;
}
// d = P z_L (sum of the rows whose last bit is set), one warp per coefficient
__global__ void plan_dvec64_kernel(const uint64_t* __restrict__ z, const double* __restrict__ pmat64, int S, int M, int kpad,
                                   double* __restrict__ dvec) {
    const int k = blockIdx.x, L = M - 1;
    if (k >= kpad) return;
    double acc = 0.0;
    if (k < M - 1)
        for (int s = threadIdx.x; s < S; s += 32)
            if ((z[s] >> L) & 1ull) acc += pmat64[(size_t)s * kpad + k];
    acc = warp_sum(acc);
    if (threadIdx.x == 0) dvec[k] = acc;
}

inline int fused_kpad(int G) { return G - 1 <= 12 ? 12 : 16; }

// slices: row groups per CTA; kw: warps per slice; warps: the slices a CTA holds at kw = 1 (the most row groups the fused
// kernel covers per CTA: the fused / unfused boundary is S_pad / 32 <= sm_count * warps)
struct FusedConfig { int warps, slices, kw, B, flat; size_t smem; };

// warps per CTA with kw > 1: at most 20 (up to 96 registers per thread) with the background size compiled in (NCT = 100,
// or 128 with 12 coefficients; weighted: NCT = 100 or 128), 16 (up to 128) elsewhere.  24 warps fit the register file
// at 80 registers without spilling for the uniform NCT = 100 kernel, but with the flat split the 20-warp build is the
// faster one (DESIGN.md 5.0.1); the weighted kernel spills at 80.  The kw = 1 layouts of weighted backgrounds hold at
// most 16 slices.
inline int fused_max_cta_warps(int N, int kpad, bool weighted = false) {
    if (weighted) return N == 100 || N == 128 ? 20 : 16;
    return N == 100 || (N == 128 && kpad == 12) ? 20 : 16;
}

// picks the layout (slices, warps per slice) and the batch for a shape; returns false when the fused kernel does not apply.
// want_warps (warps per CTA) / want_B: 0 = default (tuning knobs, dks_set_option)
inline bool fused_config(int N, int G, int S_pad, int sm_count, int max_smem, int want_warps, int want_B,
                         FusedConfig* cfg, bool weighted = false) {
    if (G < 2 || G > 16 || N > MAXN) return false;                        // at most four nibble tables, 15 coefficients
    const int kpad = fused_kpad(G);
    // kw = 1: as many slices as the shared memory holds (each brings its rows of Dm and P and one warp's staging tile), at
    // most 20 (weighted: 16).  B = 16 unless B = 8 buys more warps.
    auto max_warps = [&](int b) {
        int w = weighted ? 16 : 20;
        while (w > 0 && fused_smem_bytes(w, 1, kpad, b, N, weighted) + 1024 > (size_t)max_smem) --w;
        return w;
    };
    int B = 16;
    if (want_B == 32 || want_B == 8) B = want_B;
    int warps = max_warps(B);
    if (want_B == 0 && max_warps(8) > warps) { B = 8; warps = max_warps(8); }
    if (want_warps > 0 && want_warps < warps) warps = want_warps;
    if (warps < 1) return false;
    const int n_rg = S_pad / 32;
    if ((long long)sm_count * warps < n_rg) return false;                // every row group needs a slice
    // kw > 1: R slices of floor(cap / R) warps each, where that keeps more warps streaming than kw = 1 does (replicas of
    // every row group: floor(sm_count * R / n_rg); the slices beyond them idle).  One slice per CTA takes the flat split
    // where its two slices fit: every CTA streams.
    auto flat_fits = [&](int R, int K) {
        return R == 1 && fused_flat_smem_bytes(K, kpad, B, N, weighted) + 1024 <= (size_t)max_smem;
    };
    auto busy = [&](int R, int K) {
        if (K > 1 && flat_fits(R, K)) return (long long)K * sm_count;
        return (long long)K * ((long long)sm_count * R / n_rg) * n_rg;
    };
    const int max_cta = fused_max_cta_warps(N, kpad, weighted);
    const int cap = want_warps > 0 && want_warps < max_cta ? want_warps : max_cta;
    int slices = warps, kw = 1;
    for (int R = 1; R <= warps && cap / R >= 2; ++R) {
        const int K = cap / R;
        if ((long long)sm_count * R < n_rg || fused_smem_bytes(R, K, kpad, B, N, weighted) + 1024 > (size_t)max_smem) continue;
        if (busy(R, K) > busy(slices, kw)) { slices = R; kw = K; }
    }
    cfg->warps = warps; cfg->slices = slices; cfg->kw = kw; cfg->B = B;
    cfg->flat = kw > 1 && flat_fits(slices, kw) ? 1 : 0;
    cfg->smem = cfg->flat ? fused_flat_smem_bytes(kw, kpad, B, N, weighted) : fused_smem_bytes(slices, kw, kpad, B, N, weighted);
    return true;
}

inline cudaError_t launch_explain_fused(const FusedParams& p, const FusedConfig& cfg, int grid, cudaStream_t stream) {
    const int kpad = fused_kpad(p.G);
    cudaError_t err = cudaSuccess;
#define DKS_FUSED_LAUNCH(NCT, KP, NW)                                                                                 \
    do {                                                                                                              \
        err = cudaFuncSetAttribute(explain_shared_fused_kernel<NCT, KP, NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                   (int)cfg.smem);                                                                    \
        if (err == cudaSuccess)                                                                                       \
            explain_shared_fused_kernel<NCT, KP, NW><<<grid, 32 * NW, cfg.smem, stream>>>(p, cfg.slices, cfg.kw, cfg.flat); \
    } while (0)
    // background sizes with a compile-time specialisation (the chunk loop unrolls completely); everything else takes the
    // run-time version.  Block size: the smallest of 12 / 16 / 20 warps that holds slices x kw (20 only where
    // fused_max_cta_warps allows it).
    const int cta_warps = cfg.slices * cfg.kw;
    if (p.wn != nullptr) {
        // weighted background: 12 / 16 / 20 warps (20 only where fused_max_cta_warps allows it)
#define DKS_FUSED_LAUNCH_WT(NCT, KP, NW)                                                                              \
    do {                                                                                                              \
        err = cudaFuncSetAttribute(explain_shared_fused_kernel<NCT, KP, NW, true>,                                 \
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.smem);                       \
        if (err == cudaSuccess)                                                                                       \
            explain_shared_fused_kernel<NCT, KP, NW, true><<<grid, 32 * NW, cfg.smem, stream>>>(p, cfg.slices, cfg.kw, cfg.flat); \
    } while (0)
#define DKS_FUSED_WT(NCT, KP)                                                                                         \
    do {                                                                                                              \
        if (cta_warps > 16) DKS_FUSED_LAUNCH_WT(NCT, KP, 20);                                                         \
        else if (cta_warps > 12) DKS_FUSED_LAUNCH_WT(NCT, KP, 16);                                                    \
        else DKS_FUSED_LAUNCH_WT(NCT, KP, 12);                                                                        \
    } while (0)
#define DKS_FUSED_WT16(NCT, KP)                                                                                       \
    do {                                                                                                              \
        if (cta_warps > 12) DKS_FUSED_LAUNCH_WT(NCT, KP, 16);                                                         \
        else DKS_FUSED_LAUNCH_WT(NCT, KP, 12);                                                                        \
    } while (0)
        if (kpad == 12) {
            if (p.N == 100) DKS_FUSED_WT(100, 12);
            else if (p.N == 128) DKS_FUSED_WT(128, 12);
            else DKS_FUSED_WT16(0, 12);
        } else {
            if (p.N == 100) DKS_FUSED_WT(100, 16);
            else if (p.N == 128) DKS_FUSED_WT(128, 16);
            else DKS_FUSED_WT16(0, 16);
        }
#undef DKS_FUSED_WT16
#undef DKS_FUSED_WT
#undef DKS_FUSED_LAUNCH_WT
        return err;
    }
    const int nw = cta_warps > 16 ? 20 : (cta_warps > 12 ? 16 : 12);
#define DKS_FUSED_NW(NCT, KP)                                                                                         \
    do {                                                                                                              \
        if (nw == 12) DKS_FUSED_LAUNCH(NCT, KP, 12);                                                                  \
        else if (nw == 16) DKS_FUSED_LAUNCH(NCT, KP, 16);                                                             \
        else DKS_FUSED_LAUNCH(NCT, KP, 20);                                                                           \
    } while (0)
    if (kpad == 12) {
        if (p.N == 100) DKS_FUSED_NW(100, 12);
        else if (p.N == 128) DKS_FUSED_NW(128, 12);
        else if (p.N == 64) DKS_FUSED_NW(64, 12);
        else DKS_FUSED_NW(0, 12);
    } else {
        if (p.N == 100) DKS_FUSED_NW(100, 16);
        else DKS_FUSED_NW(0, 16);
    }
#undef DKS_FUSED_NW
#undef DKS_FUSED_LAUNCH
    return err;
}

}  // namespace shared_path
}  // namespace dks
