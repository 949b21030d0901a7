// Shared-plan fast path with the link and the projection solve FUSED into the coalition kernel.
//
// explain_shared_smem_kernel (dks_shared.cuh) writes (sum p1, sum p0) per (instance, coalition) to a global buffer (42 MB
// on the Adult-shaped workload) that wls_pmat_kernel reads back.  Here the same warp that produced a row's sums finishes
// the job: y = link(ey) - link(fnull) in place, then beta_k(i) = sum_s P[k][s] y(i, s) with P = inv(E^T W E) E^T W of the
// shared plan (float64, the warp's 32 rows of it resident in shared memory).  The sum over s runs across the lanes of a warp
// (lane = coalition row), so instead of shuffling per instance the warp parks y for a batch of B instances in shared
// memory ([row][instance], conflict-free both ways) and then turns the tile around: lane = instance, loop over its 32
// rows with P broadcast from shared memory -- 12 DFMA + 7 shared loads per (instance, row group) on the otherwise idle
// FP64 pipe, no shuffles.  Each warp adds its partial beta to a per-instance accumulator in 2^-40 FIXED POINT with 64-bit
// integer atomics (exact and order-independent: results are bit-reproducible whatever the scheduling), and the warp that
// delivers the last of the S/32 partials of an instance (a per-instance counter) applies the delta term, back-fills the
// eliminated group, snaps |phi| < 1e-10 and writes phi for both classes (and, on a multi-GPU run, stores them into every
// peer's gathered buffer over NVLink).  It also resets the accumulator and the counter, so the next launch needs no memset.
//
// The warp's 32 rows of Dm (pair sums and pair products) sit in its slice of shared memory, as in
// explain_shared_smem_kernel.  NI = 1 or 2 instances share one pass over them (one load feeds both).
#pragma once

#include "dks_shared.cuh"

namespace dks {
namespace shared_path {

constexpr int FUSED_MAX_PEERS = 16;

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
    int* done;               // [n] row groups that have delivered (zero between launches)
    double* phi;             // [C][n][G]
    int npeers;              // multi-GPU push: phi of every finished instance also goes to these buffers ([C][n][G] each)
    double* const* peer_phi; // [npeers] device array of the peers' slab addresses (NULL on one GPU)
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

// multi-GPU: the phi rows of the instances this warp just finished go to every peer's gathered buffer, stored by the whole warp
// (lanes = groups: coalesced NVLink packets instead of one 8-byte store per value from the finishing lane).  Out of line so
// that the single-GPU instantiation of the kernel does not pay registers for it.
__device__ __noinline__ void peer_push_finished(const double* __restrict__ phi, double* const* __restrict__ peers, int npeers,
                                                int fin_i, int lane, int G, size_t slab) {
    unsigned fin = __ballot_sync(0xffffffffu, fin_i >= 0);
    while (fin) {
        const int src = __ffs(fin) - 1;
        fin &= fin - 1;
        const int i = __shfl_sync(0xffffffffu, fin_i, src);
        __syncwarp();
        for (int idx = lane; idx < 2 * G; idx += 32) {
            const size_t off = (idx < G ? 0 : slab) + (size_t)i * G + (idx < G ? idx : idx - G);
            const double v = __ldcg(phi + off);
            for (int r = 0; r < npeers; ++r) peers[r][off] = v;
        }
    }
}

inline size_t fused_smem_bytes(int warps, int kpad, int B, int N) {
    return (size_t)warps * dm_slice_bytes(N) + (size_t)warps * 32 * kpad * sizeof(double) +
           (size_t)warps * 32 * (B + 1) * sizeof(double) + DKS_LOGTAB_SIZE * sizeof(LogTabEntry);
}

// NCT: background rows at compile time (0 = run-time p.N): with NCT the chunk loop unrolls completely (static shared-memory
// offsets, no loop control, the tail folded).  B (instances parked per warp) is a power of two.
template <int NCT, int KPAD, int NWARPS, int NI>
__global__ void __launch_bounds__(32 * NWARPS, 1) explain_shared_fused_kernel(FusedParams p, int warps_used) {
    extern __shared__ __align__(16) unsigned char fsm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int B = p.B, ystride = B + 1;
    const int nq = dm_quads(NCT ? NCT : p.N);
    float4* sDm = reinterpret_cast<float4*>(fsm);                                // [warps_used][nq][32]
    double* sP = reinterpret_cast<double*>(sDm + (size_t)warps_used * nq * 32);  // [warps_used][32][KPAD]
    double* sY = sP + (size_t)warps_used * 32 * KPAD;                            // [warps_used][32][B + 1]
    LogTabEntry* s_logtab = reinterpret_cast<LogTabEntry*>(sY + (size_t)warps_used * 32 * ystride);
    if (threadIdx.x >= 64 && threadIdx.x < 64 + DKS_LOGTAB_SIZE) logtab_fill(s_logtab, threadIdx.x - 64);

    const int n_rg = p.S_pad / 32;                       // row groups
    const int total_warps = gridDim.x * warps_used;
    const int nparts = total_warps / n_rg;               // replicas of every row group (>= 1: checked by the host)
    const int gw = blockIdx.x * warps_used + warp;
    const bool active = warp < warps_used && gw < nparts * n_rg;
    const int rg = active ? gw % n_rg : 0, part = active ? gw / n_rg : 0;
    double* sPw = sP + (size_t)warp * 32 * KPAD;
    double* sYw = sY + (size_t)warp * 32 * ystride;
    if (active) {
        const double* src = p.pmat64 + (size_t)rg * 32 * KPAD;     // the warp's 32 rows are contiguous
        for (int idx = lane; idx < 32 * KPAD; idx += 32) sPw[idx] = src[idx];
    }
    __syncthreads();

    if (active) {
        constexpr int MAXCH = MAXN / 16;
        const int s = rg * 32 + lane;
        const int cnt = *p.count;
        const int N = NCT ? NCT : p.N, G = p.G, nA = G - 1;
        const int nfull = N / 16, ntail = N - nfull * 16;
        const int nq_t = ntail >> 2, rem_t = ntail & 3;
        const int nch = nfull + (ntail > 0 ? 1 : 0);
        float4* sl = sDm + (size_t)warp * nq * 32;          // this warp's slice
        const double es = p.dme[s];
        // ---- this warp's 32 rows of Dm into its slice: pair sums and pair products per quad of columns (0,2) (1,3)
#pragma unroll
        for (int c = 0; c < MAXCH; ++c) {
            if (c < nch) {
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

        const uint64_t zz = s < p.S ? p.z[s] : 0ull;
        const int ntab = (G + 3) / 4;                     // <= 4 (the host sends wider problems down the unfused path)
        const f32x2 one2 = f2_pack(1.f, 1.f), two2 = f2_pack(2.f, 2.f);
        const double lf1 = p.linkfnull[1], f1 = p.fnull[1], inv_n = 1.0 / (double)N;
        const size_t slab = (size_t)p.n * G;
        const int my_n = part < cnt ? (cnt - part + nparts - 1) / nparts : 0;     // instances this warp streams
        const bool row_ok = s < p.S;
        const int bmask = B - 1;

        // ---- the turn-around: lane = instance of the batch, loop over the warp's 32 rows
        auto flush = [&](int bstart, int bcount) {
            int fin_i = -1;                 // instance this lane finished in this flush (its phi is complete in local memory)
            if (lane < bcount) {
                double beta[KPAD];
#pragma unroll
                for (int k = 0; k < KPAD; ++k) beta[k] = 0.0;
#pragma unroll 4
                for (int sr = 0; sr < 32; ++sr) {
                    const double y = sYw[sr * ystride + lane];
                    const double2* pr = reinterpret_cast<const double2*>(sPw + sr * KPAD);
#pragma unroll
                    for (int k2 = 0; k2 < KPAD / 2; ++k2) {
                        const double2 pp = pr[k2];
                        beta[2 * k2] = fma(pp.x, y, beta[2 * k2]);
                        beta[2 * k2 + 1] = fma(pp.y, y, beta[2 * k2 + 1]);
                    }
                }
                const int i = p.list[part + (bstart + lane) * nparts];
                long long* acc = p.acc + (size_t)i * KPAD;
#pragma unroll
                for (int k = 0; k < KPAD; ++k)
                    if (k < nA) atomicAdd(reinterpret_cast<unsigned long long*>(acc + k), (unsigned long long)to_fix(beta[k]));
                __threadfence();
                const int old = atomicAdd(p.done + i, 1);
                if (old == n_rg - 1) {
                    // every row group has delivered: finish the instance
                    __threadfence();
                    const double delta = p.dlink[(size_t)i * p.C + 1];
                    double sum = 0.0;
                    double* phi1 = p.phi + slab + (size_t)i * G;
                    double* phi0 = p.phi + (size_t)i * G;
                    for (int k = 0; k < nA; ++k) {
                        double val = from_fix(__ldcg(acc + k)) - delta * p.dvec[k];
                        sum += val;
                        if (fabs(val) < 1e-10) val = 0.0;
                        phi1[k] = val;
                        phi0[k] = (val == 0.0) ? 0.0 : -val;
                        acc[k] = 0;
                    }
                    double last = delta - sum;                  // the eliminated (last) group takes the remainder
                    if (fabs(last) < 1e-10) last = 0.0;
                    phi1[nA] = last;
                    phi0[nA] = (last == 0.0) ? 0.0 : -last;
                    p.done[i] = 0;
                    fin_i = i;
                }
            }
            if (p.npeers > 0) peer_push_finished(p.phi, p.peer_phi, p.npeers, fin_i, lane, G, slab);     // multi-GPU only (kept out of line: no registers here)
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
            i_nx[u] = my_n > 0 ? p.list[part + o1 * nparts] : 0;
            nx[u][0] = nx[u][1] = nx[u][2] = nx[u][3] = 0.0;
            if (my_n > 0) {
                const size_t o = (size_t)p.list[part + o0 * nparts] * xstride;
                nx[u][0] = __ldg(xb0 + o); nx[u][1] = __ldg(xb1 + o); nx[u][2] = __ldg(xb2 + o); nx[u][3] = __ldg(xb3 + o);
            }
        }

        for (int it = 0; it < my_n; it += NI) {
            float A[NI];
            bool risky_l = false;
#pragma unroll
            for (int u = 0; u < NI; ++u) {
                const double a = ((nx[u][0] + nx[u][1]) + (nx[u][2] + nx[u][3])) + es;
                {
                    const size_t o = (size_t)i_nx[u] * xstride;
                    nx[u][0] = __ldg(xb0 + o); nx[u][1] = __ldg(xb1 + o); nx[u][2] = __ldg(xb2 + o); nx[u][3] = __ldg(xb3 + o);
                    const int it2 = it + 2 * NI + u < last_it ? it + 2 * NI + u : last_it;
                    i_nx[u] = p.list[part + it2 * nparts];
                }
                // A = 2^a = 2^n 2^f, n = rint(a) through the 1.5 * 2^52 trick (no conversion instructions), |f| <= 1/2; the
                // exponent is clamped to [-120, 120] (saturated scores; the clamped scalar path below takes A > 1e18)
                const double tm = a + 6755399441055744.0;
                int an_i = __double2loint(tm);
                an_i = an_i < -120 ? -120 : (an_i > 120 ? 120 : an_i);
                A[u] = ex2_approx((float)(a - (tm - 6755399441055744.0))) * __int_as_float((127 + an_i) << 23);
                risky_l = risky_l || A[u] > 1.0e18f;
            }
            float s1[NI], s0[NI];
            if (__any_sync(0xffffffffu, risky_l)) {
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
            // ---- link in place, rows parked for the turn-around (B is a multiple of NI: a pass never straddles a batch)
#pragma unroll
            for (int u = 0; u < NI; ++u) {
                if (it + u < my_n) {
                    double y = 0.0;
                    if (row_ok) {
                        if (p.link == DKS_LINK_LOGIT) y = fast_log_ratio(s1[u], s0[u], s_logtab) - lf1;
                        else y = (double)s1[u] * inv_n - f1;
                    }
                    sYw[lane * ystride + ((it + u) & bmask)] = y;
                }
            }
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

struct FusedConfig { int ni, warps, B; size_t smem; };

// picks (warps per CTA, batch) for a shape; returns false when the fused kernel does not apply.
// want_warps / want_B: 0 = default (tuning knobs, dks_set_option)
inline bool fused_config(int N, int G, int S_pad, int sm_count, int max_smem, int want_ni, int want_warps, int want_B,
                         FusedConfig* cfg) {
    if (G < 2 || G > 16 || N > MAXN) return false;                        // at most four nibble tables, 15 coefficients
    const int kpad = fused_kpad(G);
    // warps per CTA: as many as the shared memory holds (each brings its slice of Dm, its rows of P and its staging
    // tile), at most 20.  B = 16 unless B = 8 buys more warps.
    auto max_warps = [&](int b) {
        int w = 20;
        while (w > 0 && fused_smem_bytes(w, kpad, b, N) + 1024 > (size_t)max_smem) --w;
        return w;
    };
    int B = 16;
    if (want_B == 32 || want_B == 8) B = want_B;
    int warps = max_warps(B);
    if (want_B == 0 && max_warps(8) > warps) { B = 8; warps = max_warps(8); }
    if (want_warps > 0 && want_warps < warps) warps = want_warps;
    if (warps < 1) return false;
    if ((long long)sm_count * warps < S_pad / 32) return false;          // every row group needs a warp
    cfg->ni = (want_ni == 2 && fused_kpad(G) == 12) ? 2 : 1;          // two instances per pass over Dm (tuning knob)
    cfg->warps = warps; cfg->B = B;
    cfg->smem = fused_smem_bytes(warps, kpad, B, N);
    return true;
}

inline cudaError_t launch_explain_fused(const FusedParams& p, const FusedConfig& cfg, int grid, cudaStream_t stream) {
    const int kpad = fused_kpad(p.G);
    cudaError_t err = cudaSuccess;
#define DKS_FUSED_LAUNCH(NCT, KP, NW, NI)                                                                             \
    do {                                                                                                              \
        err = cudaFuncSetAttribute(explain_shared_fused_kernel<NCT, KP, NW, NI>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                   (int)cfg.smem);                                                                    \
        if (err == cudaSuccess)                                                                                       \
            explain_shared_fused_kernel<NCT, KP, NW, NI><<<grid, 32 * NW, cfg.smem, stream>>>(p, cfg.warps);          \
    } while (0)
    // background sizes with a compile-time specialisation (the chunk loop unrolls completely); everything else takes the
    // run-time version.  Block size: the smallest of 12 / 16 / 20 warps that holds cfg.warps.
    const int nw = cfg.warps > 16 ? 20 : (cfg.warps > 12 ? 16 : 12);
#define DKS_FUSED_NW(NCT, KP, NI)                                                                                     \
    do {                                                                                                              \
        if (nw == 12) DKS_FUSED_LAUNCH(NCT, KP, 12, NI);                                                              \
        else if (nw == 16) DKS_FUSED_LAUNCH(NCT, KP, 16, NI);                                                         \
        else DKS_FUSED_LAUNCH(NCT, KP, 20, NI);                                                                       \
    } while (0)
    if (kpad == 12 && cfg.ni == 2) {
        if (p.N == 100) DKS_FUSED_NW(100, 12, 2);
        else DKS_FUSED_NW(0, 12, 2);
    } else if (kpad == 12) {
        if (p.N == 100) DKS_FUSED_NW(100, 12, 1);
        else if (p.N == 128) DKS_FUSED_NW(128, 12, 1);
        else if (p.N == 64) DKS_FUSED_NW(64, 12, 1);
        else DKS_FUSED_NW(0, 12, 1);
    } else {
        if (p.N == 100) DKS_FUSED_NW(100, 16, 1);
        else DKS_FUSED_NW(0, 16, 1);
    }
#undef DKS_FUSED_NW
#undef DKS_FUSED_LAUNCH
    return err;
}

}  // namespace shared_path
}  // namespace dks
