// Fused coalition kernel on the Hopper tensor cores (wgmma, sm_90a), binary-logistic head.
//
// Per instance i and 128-coalition tile the masked-batch scores are one small dense contraction
//     T[s][j] = sum_k Z[s][k] * Delta_i[j][k],      Delta_i[j][k] = scale*(XW_i[v_k] - BW[j][v_k]),  k < M
//                                                   Delta_i[j][M] = scale*score_j   (Z[s][M] = 1)
// (scale = -kappa*log2 e, so exp(-kappa*score) = 2^T).  Z is 0/1 and exact in bf16; Delta is split into three bf16
// terms (hi/mid/lo, ~fp32-exact) and accumulated in fp32 registers by three wgmma (M=64, N=32, K=16) per 64-row half
// and 32-column block of the tile.
// Warpgroup roles of the persistent CTA (one per SM):
//   warpgroup 0           builders (one thread per tile row / background row): the instance's B operand (Delta splits)
//                         and each tile's A operand (Z bits expanded to bf16 through a 256-entry byte LUT, never read
//                         from HBM as a matrix) into shared memory, running up to NBUF tiles ahead;
//   warpgroups 1..N_CONS  consumers: tile g goes to consumer g % N_CONS, which issues the wgmma of each 64 x 32 block,
//                         waits for them and turns the fp32 scores into p1 = 1/(1+2^T) and the background-weighted sums
//                         (sum p1, sum p0) per coalition row -> link -> shared memory.  Four consumers keep enough
//                         independent MUFU chains in flight per SM sub-partition while another consumer waits on wgmma;
//   last warpgroup        WLS (float64), one instance behind: y = link(ey) - link(fnull) per row folded into E^T W y,
//                         per-instance normal matrix when the plan is not shared, triangular solves, phi.
// All hand-offs are mbarriers; no __syncthreads in the steady state.
#pragma once

#include <cuda_bf16.h>

#include "dks_kernels.cuh"

namespace dks {
namespace tc {

constexpr int TILE_S = 128;      // coalitions per A tile: two wgmma M = 64 halves
constexpr int KP = 16;           // K per split: up to 15 varying groups + the constant column
constexpr int NSPLIT = 3;        // bf16 hi/mid/lo
constexpr int MAX_NPAD = 128;    // background rows of one instance's B operand
constexpr int NBLK = 32;         // background columns per wgmma (N)
constexpr int N_CONS = 4;        // consumer warpgroups
constexpr int N_PROD_WARPS = 4, N_EPI_WARPS = 4 * N_CONS, N_WLS_WARPS = 4;
constexpr int NTHREADS = 32 * (N_PROD_WARPS + N_EPI_WARPS + N_WLS_WARPS);
constexpr int NBUF = 2 * N_CONS; // A-tile buffers: two per consumer
constexpr float T_CLAMP = 60.f;  // 2^t is clamped at 2^60 so the product of two (1 + 2^t) stays finite in fp32
constexpr uint32_t SPIN_LIMIT = 1u << 26;

// ---- PTX wrappers ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// bounded wait: a protocol bug must not hang the GPU -- flag the status word and trap instead
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int* status) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > SPIN_LIMIT) {
            status[0] = DKS_ERR_CUDA;
            status[1] = -77;
            __threadfence_system();
            asm volatile("trap;");
        }
    }
}
// TMA bulk copy global -> shared (1-D, cp.async.bulk), completion counted in bytes on an mbarrier
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// wgmma: the accumulator registers are in/out operands of every wrapper, so no access to them can be scheduled across
// the fence, the MMAs or the wait
__device__ __forceinline__ void wgmma_fence(float (&d)[16]) {
    asm volatile("wgmma.fence.sync.aligned;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
                   "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 :
                 : "memory");
}
// D (+)= A[smem] * B[smem], bf16 x bf16 -> fp32, M = 64, N = 32, K = 16, both operands K-major
__device__ __forceinline__ void wgmma_bf16_n32(float (&d)[16], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_commit_wait(float (&d)[16]) {
    asm volatile("wgmma.commit_group.sync.aligned;\n\twgmma.wait_group.sync.aligned 0;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
                   "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 :
                 : "memory");
}

// wgmma shared-memory matrix descriptor, K-major, no swizzle (canonical layout ((8,m),(T,2)):((1T,SBO),(1,LBO)):
// 8x16-byte core matrices; LBO = bytes between the two K-adjacent core matrices of one K=16 step, SBO = bytes
// between core matrices adjacent along M/N).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    return d;
}

// ---- shared memory carve-up ---------------------------------------------------------------------------------
constexpr int NBARS = 2 * NBUF + 9;   // a_full[NBUF], a_empty[NBUF], b_full[2], b_empty[2], inst_full[2], inst_empty[2], plan_ready
constexpr int BAR_BYTES = (NBARS * 8 + 127) / 128 * 128;
struct Smem {
    uint64_t* bars;
    int* vi;             // [16] varying position -> group (producer group only)
    double* chol;        // [15*15]
    double* rhs;         // [16]
    double* part;        // [N_WLS_WARPS][16] per-warp partial right-hand sides (int64 fixed point)
    double* ys;          // [2][S_cap] link(ey) - link(fnull) per coalition row, per instance parity
    float* wb;           // [MAX_NPAD] background weights
    uint64_t* zs;        // [S_cap] coalition words of the staged shared plan (TMA bulk copy)
    double* ws;          // [S_cap] its kernel weights
    LogTabEntry* logtab; // [64] table of fast_log_ratio
    uint4* lut;          // [256] byte -> eight bf16 (1.0 / 0.0)
    unsigned char* A;    // [NBUF][128*KP*2]
    unsigned char* B;    // [2][NSPLIT][Nb*KP*2]
};
__host__ __device__ inline size_t smem_bytes(int S_cap, int Nb) {
    return BAR_BYTES + 16 * sizeof(int) + (15 * 15 + 16 + N_WLS_WARPS * 16) * sizeof(double) +
           2 * (size_t)S_cap * sizeof(double) + 2 * ((size_t)S_cap + 2) * 8 + MAX_NPAD * sizeof(float) + DKS_LOGTAB_SIZE * 16 +
           256 * 16 + NBUF * (size_t)TILE_S * KP * 2 +
           2 * NSPLIT * (size_t)Nb * KP * 2 + 192;
}
__device__ inline Smem carve(unsigned char* base, int S_cap) {
    Smem s;
    s.bars = reinterpret_cast<uint64_t*>(base);
    s.vi = reinterpret_cast<int*>(base + BAR_BYTES);
    s.chol = reinterpret_cast<double*>(base + BAR_BYTES + 16 * sizeof(int));
    s.rhs = s.chol + 15 * 15;
    s.part = s.rhs + 16;
    s.ys = s.part + N_WLS_WARPS * 16;
    s.wb = reinterpret_cast<float*>(s.ys + 2 * (size_t)S_cap);
    unsigned char* p = reinterpret_cast<unsigned char*>(s.wb + MAX_NPAD);
    p = reinterpret_cast<unsigned char*>(((uintptr_t)p + 15) & ~(uintptr_t)15);
    const size_t plan_words = ((size_t)S_cap + 1) & ~(size_t)1;          // 16-byte multiples for the bulk copy
    s.zs = reinterpret_cast<uint64_t*>(p);
    s.ws = reinterpret_cast<double*>(p + plan_words * 8);
    p += 2 * plan_words * 8;
    s.logtab = reinterpret_cast<LogTabEntry*>(p);
    s.lut = reinterpret_cast<uint4*>(p + DKS_LOGTAB_SIZE * 16);
    p += DKS_LOGTAB_SIZE * 16 + 256 * 16;
    s.A = reinterpret_cast<unsigned char*>(((uintptr_t)p + 127) & ~(uintptr_t)127);   // MMA operands: 128-byte aligned
    s.B = s.A + NBUF * (size_t)TILE_S * KP * 2;
    return s;
}

struct TcParams {
    ExplainParams p;
    const double* BW;      // [N][G] grouped background contributions, float64 (R == 1)
    const double* scores;  // [N]
    int Nb;                // background rows of the B operand (N rounded up to NBLK)
    int Npad;              // columns of the debug dump (N rounded up to 16)
    float* dbg_T;          // optional [S_cap][Npad] dump of the scores of instance dbg_i
    int dbg_i;
    float* dbg_time;       // optional [6][256] clock64 timeline of CTA 0 (debug kernel variant only)
};

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}

// instances this CTA handles: i = blockIdx.x + q*gridDim.x; every role walks the same list
__device__ __forceinline__ int tiles_of(const ExplainParams& p, int i, int& M, int& S) {
    M = p.Mcnt[i];
    if (M < 2) { S = 0; return 0; }
    S = dks_effective_S(M, p.S_req);
    if (p.ext_z == nullptr) {
        PlanDev pd = p.plans[M];
        if (pd.z == nullptr || pd.S != S) { S = 0; return 0; }   // reported by the WLS warps
    }
    if (S > p.S_cap) { S = 0; return 0; }
    return (S + TILE_S - 1) / TILE_S;
}

// p1 = 1/(1+2^t) and p0 = 2^t/(1+2^t) (no cancellation) summed over background rows.  Two elements share one
// reciprocal: r = 1/((1+ua)(1+ub)), p1a = r(1+ub), p1b = r(1+ua)  -> 1.5 MUFU ops per element instead of 2.
__device__ __forceinline__ void consume_pair(float ta, float tb, float wa, float wb_, float& a1, float& a0) {
    ta = fminf(ta, T_CLAMP);
    tb = fminf(tb, T_CLAMP);
    const float ua = ex2_approx(ta), ub = ex2_approx(tb);
    const float da = 1.f + ua, db = 1.f + ub;
    const float r = rcp_approx(da * db);
    const float ra = r * db, rb = r * da;
    a1 = fmaf(wa, ra, a1);
    a1 = fmaf(wb_, rb, a1);
    a0 = fmaf(wa * ua, ra, a0);
    a0 = fmaf(wb_ * ub, rb, a0);
}

// Uniform background weights: four columns at a time.  With u = 2^t per column and the columns paired (0,2), (1,3):
// p1a + p1b = (2 + sm) / (1 + sm + q),  p0a + p0b = (sm + 2q) / (1 + sm + q),  sm = ua + ub, q = ua ub -- one
// reciprocal per pair, 6 MUFU per four columns.
__device__ __forceinline__ void consume_quad(float t0, float t1, float t2, float t3, f32x2& a1, f32x2& a0) {
    const f32x2 u = f2_pack(ex2_approx(fminf(t0, T_CLAMP)), ex2_approx(fminf(t1, T_CLAMP)));
    const f32x2 v = f2_pack(ex2_approx(fminf(t2, T_CLAMP)), ex2_approx(fminf(t3, T_CLAMP)));
    const f32x2 one2 = f2_pack(1.f, 1.f), two2 = f2_pack(2.f, 2.f);
    const f32x2 q = f2_mul(u, v), sm = f2_add(u, v);
    const f32x2 s1 = f2_add(sm, one2);
    float dlo, dhi;
    f2_unpack(f2_add(q, s1), dlo, dhi);
    const f32x2 r = f2_pack(rcp_approx(dlo), rcp_approx(dhi));
    a1 = f2_fma(r, f2_add(s1, one2), a1);
    a0 = f2_fma(r, f2_fma(two2, q, sm), a0);
}

// One accumulator row of a 64 x 32 block: v[2jj], v[2jj+1] hold columns 8jj + cq and 8jj + cq + 1.  `wb` points at the
// weight of column 0 of the block + cq; `full`: all 32 columns of the block are background rows, else `nleft` = background
// rows from column cq of the block on.
template <bool UW>
__device__ __forceinline__ void consume_row(const float (&v)[8], const float* __restrict__ wb, bool full, int nleft,
                                            float& acc1, float& acc0) {
    if (full) {
        if (UW) {
            f32x2 p1[2] = {f2_pack(0.f, 0.f), f2_pack(0.f, 0.f)}, p0[2] = {f2_pack(0.f, 0.f), f2_pack(0.f, 0.f)};
            consume_quad(v[0], v[1], v[2], v[3], p1[0], p0[0]);
            consume_quad(v[4], v[5], v[6], v[7], p1[1], p0[1]);
            float x0, x1, y0, y1;
            f2_unpack(f2_add(p1[0], p1[1]), x0, x1);
            f2_unpack(f2_add(p0[0], p0[1]), y0, y1);
            acc1 += x0 + x1;
            acc0 += y0 + y1;
            return;
        }
        float a1[2] = {0.f, 0.f}, a0[2] = {0.f, 0.f};
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) consume_pair(v[2 * jj], v[2 * jj + 1], wb[8 * jj], wb[8 * jj + 1], a1[jj & 1], a0[jj & 1]);
        acc1 += a1[0] + a1[1];
        acc0 += a0[0] + a0[1];
        return;
    }
    // last, partially filled block: weights come from shared memory (zero for the padding column of an odd pair)
    float a1 = 0.f, a0 = 0.f;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
        if (8 * jj < nleft) consume_pair(v[2 * jj], v[2 * jj + 1], wb[8 * jj], wb[8 * jj + 1], a1, a0);
    acc1 += a1;
    acc0 += a0;
}

template <bool UW, bool DBG>
__global__ void __launch_bounds__(NTHREADS, 1) explain_wgmma_kernel(TcParams tp) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const ExplainParams& p = tp.p;
    const int Nb = tp.Nb, N = p.N, G = p.G;
    Smem sm = carve(smem_raw, p.S_cap);
    uint64_t* a_full = sm.bars;
    uint64_t* a_empty = sm.bars + NBUF;
    uint64_t* b_full = sm.bars + 2 * NBUF;
    uint64_t* b_empty = sm.bars + 2 * NBUF + 2;
    uint64_t* inst_full = sm.bars + 2 * NBUF + 4;
    uint64_t* inst_empty = sm.bars + 2 * NBUF + 6;
    uint64_t* plan_ready = sm.bars + 2 * NBUF + 8;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t slab = (size_t)p.n * G;
    const int ninst = dks_inst_count(p);
    if ((int)blockIdx.x >= ninst) return;        // nothing for this CTA

    constexpr int PROD_THREADS = 32 * N_PROD_WARPS, CONS_THREADS = 32 * N_EPI_WARPS, WLS_THREADS = 32 * N_WLS_WARPS;
    if (threadIdx.x == 0) {
        for (int b = 0; b < NBUF; ++b) { mbar_init(&a_full[b], PROD_THREADS); mbar_init(&a_empty[b], 128); }
        for (int b = 0; b < 2; ++b) {
            mbar_init(&b_full[b], PROD_THREADS);
            mbar_init(&b_empty[b], CONS_THREADS);
            mbar_init(&inst_full[b], CONS_THREADS);
            mbar_init(&inst_empty[b], WLS_THREADS);
        }
        mbar_init(plan_ready, 1);
        fence_barrier_init();
    }
    // weights of the padded columns are zero; with uniform weights the sums stay unnormalised (weight 1)
    for (int j = threadIdx.x; j < MAX_NPAD; j += blockDim.x) sm.wb[j] = j < N ? (UW ? 1.f : p.wbf[j]) : 0.f;
    if (threadIdx.x < DKS_LOGTAB_SIZE) logtab_fill(sm.logtab, threadIdx.x);
    for (int b = threadIdx.x; b < 256; b += blockDim.x) {
        uint4 e;
        e.x = ((b & 1) ? 0x00003F80u : 0u) | ((b & 2) ? 0x3F800000u : 0u);
        e.y = ((b & 4) ? 0x00003F80u : 0u) | ((b & 8) ? 0x3F800000u : 0u);
        e.z = ((b & 16) ? 0x00003F80u : 0u) | ((b & 32) ? 0x3F800000u : 0u);
        e.w = ((b & 64) ? 0x00003F80u : 0u) | ((b & 128) ? 0x3F800000u : 0u);
        sm.lut[b] = e;
    }
    __syncthreads();

    // Stage the shared plan of this CTA's first instance (coalition words + weights) into shared memory with two TMA
    // bulk copies; builders and WLS warps read it from there instead of re-reading global memory every tile.
    // Instances with another M (rare) and per-instance plans keep reading global memory.
    int staged_M = -1;
    if (p.ext_z == nullptr) {
        for (int qi = blockIdx.x; qi < ninst && staged_M < 0; qi += gridDim.x) {
            int M_, S_;
            if (tiles_of(p, dks_inst_at(p, qi), M_, S_) > 0) staged_M = M_;
        }
        if (staged_M >= 0) {
            const uint32_t bytes = (uint32_t)((((size_t)p.plans[staged_M].S + 1) & ~(size_t)1) * 8);
            if (threadIdx.x == 0) {
                mbar_expect_tx(plan_ready, 2 * bytes);
                tma_load_1d(sm.zs, p.plans[staged_M].z, bytes, plan_ready);
                tma_load_1d(sm.ws, p.plans[staged_M].w, bytes, plan_ready);
            }
            mbar_wait(plan_ready, 0, p.status);
        }
    }

    const uint32_t a_bytes = TILE_S * KP * 2, b_split_bytes = (uint32_t)Nb * KP * 2;
    const long long t_start = clock64();
    auto stamp = [&](int ev, uint32_t g) {   // debug timeline: event ev of tile g of CTA 0, in cycles since start
        if (DBG && tp.dbg_time != nullptr && blockIdx.x == 0 && g < 256)
            tp.dbg_time[ev * 256 + g] = (float)(clock64() - t_start);
    };

    if (warp < N_PROD_WARPS) {
        // =================================== builders ===================================
        const int ptid = threadIdx.x;                 // 0..127: tile row (A) and background row (B) of this thread

        // B operand of the instance with ordinal o into slot o & 1: Delta splits, K-major core matrices [kc][j][8];
        // thread = row j.  The slot is free once the consumers are done with ordinal o - 2.
        auto build_B = [&](int i, int M, int o) {
            mbar_wait(&b_empty[o & 1], ((o >> 1) & 1) ^ 1, p.status);
            const uint64_t vm = p.vmask[i];
            unsigned char* Bq = sm.B + (size_t)(o & 1) * NSPLIT * b_split_bytes;
            named_bar_sync(2, PROD_THREADS);            // previous readers of sm.vi are done
            if (ptid < KP) {                            // thread k finds the k-th varying group
                int cnt = 0, gsel = 0;
                for (int gI = 0; gI < G; ++gI)
                    if ((vm >> gI) & 1ull) { if (cnt == ptid) gsel = gI; ++cnt; }
                sm.vi[ptid] = ptid < M ? gsel : 0;
            }
            named_bar_sync(2, PROD_THREADS);
            const int j = ptid;
            if (j < Nb) {
#pragma unroll
                for (int kc = 0; kc < 2; ++kc) {
                    float hi[8], mid[8], lo[8];
#pragma unroll
                    for (int k8 = 0; k8 < 8; ++k8) {
                        const int kk = kc * 8 + k8;
                        double v = 0.0;
                        if (j < N) {
                            const int gk = sm.vi[kk];
                            if (kk < M) v = p.scale * (p.XW[(size_t)i * G + gk] - tp.BW[(size_t)j * G + gk]);
                            else if (kk == M) v = p.scale * tp.scores[j];
                        }
                        float vf = (float)v;
                        float h = __bfloat162float(__float2bfloat16_rn(vf));
                        float r1 = vf - h;
                        float m = __bfloat162float(__float2bfloat16_rn(r1));
                        float r2 = (r1 - m) + (float)(v - (double)vf);
                        hi[k8] = h; mid[k8] = m; lo[k8] = r2;
                    }
                    uint4 wh, wm, wl;
                    wh.x = pack_bf16(hi[0], hi[1]); wh.y = pack_bf16(hi[2], hi[3]);
                    wh.z = pack_bf16(hi[4], hi[5]); wh.w = pack_bf16(hi[6], hi[7]);
                    wm.x = pack_bf16(mid[0], mid[1]); wm.y = pack_bf16(mid[2], mid[3]);
                    wm.z = pack_bf16(mid[4], mid[5]); wm.w = pack_bf16(mid[6], mid[7]);
                    wl.x = pack_bf16(lo[0], lo[1]); wl.y = pack_bf16(lo[2], lo[3]);
                    wl.z = pack_bf16(lo[4], lo[5]); wl.w = pack_bf16(lo[6], lo[7]);
                    const size_t off = (size_t)kc * Nb * 16 + (size_t)j * 16;
                    *reinterpret_cast<uint4*>(Bq + 0 * b_split_bytes + off) = wh;
                    *reinterpret_cast<uint4*>(Bq + 1 * b_split_bytes + off) = wm;
                    *reinterpret_cast<uint4*>(Bq + 2 * b_split_bytes + off) = wl;
                }
            }
            fence_proxy_async_smem();   // generic-proxy writes -> visible to the tensor core (async proxy)
            mbar_arrive(&b_full[o & 1]);
        };
        auto next_work = [&](int qi, int& Mn) {   // next instance of this CTA that has tiles (-1: none)
            for (int q2 = qi + gridDim.x; q2 < ninst; q2 += gridDim.x) {
                int S2;
                const int i2 = dks_inst_at(p, q2);
                if (tiles_of(p, i2, Mn, S2) > 0) return i2;
            }
            return -1;
        };

        uint32_t g = 0;   // global tile counter of this CTA
        int qb = 0;       // ordinal among the instances that have tiles (selects the B slot)
        int built_for = -1;
        for (int qi = blockIdx.x; qi < ninst; qi += gridDim.x) {
            const int i = dks_inst_at(p, qi);
            int M, S;
            const int T = tiles_of(p, i, M, S);
            if (T == 0) continue;
            const uint64_t* zp = p.ext_z ? p.ext_z + (size_t)i * p.ext_stride : (M == staged_M ? sm.zs : p.plans[M].z);
            if (built_for != i) build_B(i, M, qb);    // only the first instance; later ones are prefetched below
            const int t_prefetch = T > NBUF - 1 ? NBUF - 1 : T - 1;   // after this tile: build the next instance's B
            for (int t = 0; t < T; ++t, ++g) {
                const uint32_t buf = g % NBUF, u = g / NBUF;
                const int s = t * TILE_S + ptid;
                uint32_t zz = 0;
                if (s < S) zz = (uint32_t)(zp[s] & 0xFFFFull) | (1u << M);       // constant column carries score_j
                mbar_wait(&a_empty[buf], (u & 1) ^ 1, p.status);                 // consumer of tile g - NBUF is done
                unsigned char* Ab = sm.A + (size_t)buf * a_bytes;
                *reinterpret_cast<uint4*>(Ab + 0 * (TILE_S * 16) + ptid * 16) = sm.lut[zz & 0xFFu];
                *reinterpret_cast<uint4*>(Ab + 1 * (TILE_S * 16) + ptid * 16) = sm.lut[(zz >> 8) & 0xFFu];
                fence_proxy_async_smem();
                mbar_arrive(&a_full[buf]);
                if (ptid == 0) stamp(0, g);                               // A tile ready
                // prefetch: while this instance is in flight, build the next instance's B operand
                if (t == t_prefetch) {
                    int Mn;
                    int inext = next_work(qi, Mn);
                    if (inext >= 0) {
                        build_B(inext, Mn, qb + 1);
                        built_for = inext;
                    }
                }
            }
            ++qb;
        }
    } else if (warp < N_PROD_WARPS + N_EPI_WARPS) {
        // =================================== consumers ===================================
        const int cw = warp - N_PROD_WARPS;           // 0..N_EPI_WARPS-1
        const int cons = cw >> 2;                     // consumer warpgroup: tiles with g % N_CONS == cons
        const int r_lo = 16 * (cw & 3) + (lane >> 2); // accumulator rows r_lo and r_lo + 8 of each 64-row half
        const int cq = 2 * (lane & 3);                // accumulator columns 8jj + cq, 8jj + cq + 1 of each block
        const int nblk = (N + NBLK - 1) / NBLK;
        const double lf1 = p.linkfnull[1], f1 = p.fnull[1];
        const float inv_n = 1.0f / (float)N;
        const uint32_t a_base = smem_u32(sm.A), b_base = smem_u32(sm.B);

        uint32_t g = 0;
        int q = 0, qb = 0;
        for (int qi = blockIdx.x; qi < ninst; qi += gridDim.x, ++q) {
            const int i = dks_inst_at(p, qi);
            int M, S;
            const int T = tiles_of(p, i, M, S);
            double* ys = sm.ys + (size_t)(q & 1) * p.S_cap;
            bool waited = false;
            const int slot = qb & 1;
            if (T > 0) mbar_wait(&b_full[slot], (qb >> 1) & 1, p.status);     // B operand of this instance is in place
            for (int t = 0; t < T; ++t, ++g) {
                if ((int)(g % N_CONS) != cons) continue;
                const uint32_t buf = g % NBUF, u = g / NBUF;
                if ((cw & 3) == 0 && lane == 0) stamp(3, g);              // consumer starts waiting
                mbar_wait(&a_full[buf], u & 1, p.status);
                if ((cw & 3) == 0 && lane == 0) stamp(4, g);              // A tile seen
                float acc1[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, acc0[2][2] = {{0.f, 0.f}, {0.f, 0.f}};   // [half][row]
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint64_t ad = make_smem_desc(a_base + buf * a_bytes + h * 64 * 16, TILE_S * 16, 128);
                    for (int c = 0; c < nblk; ++c) {
                        float d[16];
#pragma unroll
                        for (int e = 0; e < 16; ++e) d[e] = 0.f;
                        wgmma_fence(d);
#pragma unroll
                        for (int sp = 0; sp < NSPLIT; ++sp) {
                            const uint32_t baddr = b_base + ((uint32_t)slot * NSPLIT + sp) * b_split_bytes + c * NBLK * 16;
                            wgmma_bf16_n32(d, ad, make_smem_desc(baddr, (uint32_t)Nb * 16, 128), sp > 0 ? 1u : 0u);
                        }
                        wgmma_commit_wait(d);
                        if (DBG && i == tp.dbg_i) {
#pragma unroll
                            for (int e = 0; e < 16; ++e) {
                                const int s = t * TILE_S + h * 64 + r_lo + ((e >> 1) & 1) * 8;
                                const int col = c * NBLK + (e >> 2) * 8 + cq + (e & 1);
                                if (s < p.S_cap && col < tp.Npad) tp.dbg_T[(size_t)s * tp.Npad + col] = d[e];
                            }
                        }
                        const float va[8] = {d[0], d[1], d[4], d[5], d[8], d[9], d[12], d[13]};
                        const float vb[8] = {d[2], d[3], d[6], d[7], d[10], d[11], d[14], d[15]};
                        const int col0 = c * NBLK + cq;
                        const bool full = (c + 1) * NBLK <= N;
                        consume_row<UW>(va, sm.wb + col0, full, N - col0, acc1[h][0], acc0[h][0]);
                        consume_row<UW>(vb, sm.wb + col0, full, N - col0, acc1[h][1], acc0[h][1]);
                    }
                }
                mbar_arrive(&a_empty[buf]);          // every wgmma reading A[buf] has completed
                if ((cw & 3) == 0 && lane == 0) stamp(5, g);              // tile drained
                // the four lanes of a quad hold the same rows: sum their column partials
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                        for (int o = 1; o < 4; o <<= 1) {
                            acc1[h][rr] += __shfl_xor_sync(0xffffffffu, acc1[h][rr], o);
                            acc0[h][rr] += __shfl_xor_sync(0xffffffffu, acc0[h][rr], o);
                        }
                if (!waited) {   // the row buffer of ordinal q-2 must have been consumed by the WLS warps
                    mbar_wait(&inst_empty[q & 1], ((q >> 1) & 1) ^ 1, p.status);
                    waited = true;
                }
                if ((lane & 3) == 0) {
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int rr = 0; rr < 2; ++rr) {
                            const int s = t * TILE_S + h * 64 + r_lo + rr * 8;
                            if (s < S) {
                                // link(ey) - link(fnull); with the logit link the normalisation of the sums cancels
                                double y;
                                if (p.link == DKS_LINK_LOGIT) y = fast_log_ratio(acc1[h][rr], acc0[h][rr], sm.logtab) - lf1;
                                else y = (double)(UW ? acc1[h][rr] * inv_n : acc1[h][rr]) - f1;
                                ys[s] = y;
                            }
                        }
                }
            }
            if (T > 0) {
                mbar_arrive(&b_empty[slot]);
                ++qb;
            }
            if (!waited) mbar_wait(&inst_empty[q & 1], ((q >> 1) & 1) ^ 1, p.status);
            mbar_arrive(&inst_full[q & 1]);          // release-arrive: publishes the rows written by this thread
        }
    } else {
        // =================================== WLS warpgroup (float64) ===================================
        // per row: y = link(ey) - link(fnull) folded into E^T W y; then the triangular solves and phi.  Runs one
        // instance behind the consumers.
        const int ww = warp - (N_PROD_WARPS + N_EPI_WARPS);                  // 0..3
        const int wtid = threadIdx.x - 32 * (N_PROD_WARPS + N_EPI_WARPS);     // 0..127
        int cachedM = -1;
        bool have_inverse = false;
        int q = 0;
        for (int qi = blockIdx.x; qi < ninst; qi += gridDim.x, ++q) {
            const int i = dks_inst_at(p, qi);
            int M, S;
            const int T = tiles_of(p, i, M, S);
            const int C = p.C;
            for (int idx = wtid; idx < C * G; idx += WLS_THREADS)
                p.phi[(size_t)(idx / G) * slab + (size_t)i * G + idx % G] = 0.0;
            if (T == 0) {
                mbar_wait(&inst_full[q & 1], (q >> 1) & 1, p.status);
                if (M == 1) {
                    if (wtid < C) {
                        int gI = __ffsll((long long)p.vmask[i]) - 1;
                        p.phi[(size_t)wtid * slab + (size_t)i * G + gI] = p.dlink[(size_t)i * C + wtid];
                    }
                } else if (M >= 2 && wtid == 0) {
                    int S0 = dks_effective_S(M, p.S_req);
                    bool missing = p.ext_z == nullptr && (p.plans[M].z == nullptr || p.plans[M].S != S0);
                    if (missing) { if (atomicCAS(&p.status[0], 0, DKS_ERR_PLAN_MISSING) == 0) p.status[1] = M; }
                    else { if (atomicCAS(&p.status[0], 0, DKS_ERR_INVALID) == 0) p.status[1] = i; }
                }
                mbar_arrive(&inst_empty[q & 1]);
                continue;
            }
            const int nA = M - 1, L = M - 1;
            const uint64_t* zp;
            const double* wp;
            // normal matrix / its Cholesky factor: shared plans bring a precomputed factor; per-instance plans are
            // factored here, overlapping the consumers' work on the same instance
            if (p.ext_z == nullptr) {
                zp = M == staged_M ? sm.zs : p.plans[M].z;
                wp = M == staged_M ? sm.ws : p.plans[M].w;
                const double* ainv = p.plans[M].ainv;        // inverse of E^T W E, computed once per plan
                if (M != cachedM) {
                    named_bar_sync(1, WLS_THREADS);
                    for (int idx = wtid; idx < nA * nA; idx += WLS_THREADS) sm.chol[idx] = ainv[idx];
                    cachedM = M;
                }
                have_inverse = true;
            } else {
                cachedM = -1;
                have_inverse = false;
                zp = p.ext_z + (size_t)i * p.ext_stride;
                wp = p.ext_w + (size_t)i * p.ext_stride;
                named_bar_sync(1, WLS_THREADS);
                if (p.ext_ainv != nullptr) {             // the plan came with the inverse of its normal matrix
                    const double* ainv = p.ext_ainv + (size_t)i * p.ext_fstride;
                    for (int idx = wtid; idx < nA * nA; idx += WLS_THREADS) sm.chol[idx] = ainv[idx];
                    have_inverse = true;
                } else {
                    wls_build_normal(zp, wp, S, M, sm.chol, ww, N_WLS_WARPS);
                    named_bar_sync(1, WLS_THREADS);
                    if (ww == 0) {
                        bool ok = wls_cholesky_warp(sm.chol, nA);
                        if (!ok && lane == 0) { if (atomicCAS(&p.status[0], 0, DKS_ERR_NUMERIC) == 0) p.status[1] = i; }
                    }
                }
            }
            const double delta = p.dlink[(size_t)i * C + 1];
            mbar_wait(&inst_full[q & 1], (q >> 1) & 1, p.status);
            const double* ys = sm.ys + (size_t)(q & 1) * p.S_cap;
            long long Tk[KP - 1];                    // fixed-point partial sums of E^T W y (exact integer adds)
#pragma unroll
            for (int k = 0; k < KP - 1; ++k) Tk[k] = 0;
            for (int s = wtid; s < S; s += WLS_THREADS) {
                const double y = ys[s];
                const uint64_t zrow = zp[s];
                const double wrow = wp[s];
                // fold the row into E^T W y:  e_k = z_k - z_L = (z_L ? -1 : 1) * z'_k with z' = z_L ? ~z : z
                const bool zl = (zrow >> L) & 1ull;
                const double v = wrow * (y - (zl ? delta : 0.0));
                const uint32_t zb = (uint32_t)(zl ? ~zrow : zrow);
                const long long vi = zl ? -to_fix(v) : to_fix(v);
#pragma unroll
                for (int k = 0; k < KP - 1; ++k)
                    if (k < nA && ((zb >> k) & 1u)) Tk[k] += vi;
            }
            long long* part_ll = reinterpret_cast<long long*>(sm.part);
#pragma unroll
            for (int k = 0; k < KP - 1; ++k)
                if (k < nA) {
                    const long long r = warp_sum_ll(Tk[k]);
                    if (lane == 0) part_ll[ww * 16 + k] = r;
                }
            named_bar_sync(1, WLS_THREADS);
            if (wtid < nA) {
                long long acc = 0;
                for (int e = 0; e < N_WLS_WARPS; ++e) acc += part_ll[e * 16 + wtid];
                sm.rhs[wtid] = from_fix(acc);
            }
            named_bar_sync(1, WLS_THREADS);
            if (have_inverse) {
                // beta = inv(E^T W E) (E^T W y): one thread per coefficient, then phi (both classes) by warp 0
                double beta = 0.0;
                if (ww == 0 && lane < nA) {
                    for (int l = 0; l < nA; ++l) beta = fma(sm.chol[lane * nA + l], sm.rhs[l], beta);
                }
                if (ww == 0) {
                    double sum = beta;                    // lanes >= nA hold 0
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                    // lane k < nA owns varying position k, lane nA the eliminated (last) one
                    double val = lane < nA ? beta : delta - sum;
                    if (fabs(val) < 1e-10) val = 0.0;
                    if (lane < M) {
                        const uint64_t vm = p.vmask[i];
                        int cnt = 0, gsel = 0;
                        for (int gI = 0; gI < G; ++gI)
                            if ((vm >> gI) & 1ull) { if (cnt == lane) gsel = gI; ++cnt; }
                        p.phi[slab + (size_t)i * G + gsel] = val;
                        p.phi[(size_t)i * G + gsel] = (val == 0.0) ? 0.0 : -val;
                    }
                }
            } else if (wtid == 0) {
                int vi[KP];
                {
                    const uint64_t vm = p.vmask[i];
                    int k = 0;
                    for (int gI = 0; gI < G; ++gI) if (((vm >> gI) & 1ull) && k < KP) vi[k++] = gI;
                }
                wls_solve_write(sm.chol, sm.rhs, M, delta, vi, p.phi + slab + (size_t)i * G, 1.0);
                double* phi0 = p.phi + (size_t)i * G;
                const double* phi1 = p.phi + slab + (size_t)i * G;
                for (int k = 0; k < M; ++k) { double v = phi1[vi[k]]; phi0[vi[k]] = (v == 0.0) ? 0.0 : -v; }
            }
            named_bar_sync(1, WLS_THREADS);
            mbar_arrive(&inst_empty[q & 1]);
        }
    }
}

}  // namespace tc

// ---- host glue --------------------------------------------------------------------------------------------------
inline int tc_npad(int N) { return (N + 15) / 16 * 16; }
inline int tc_nb(int N) { return (N + tc::NBLK - 1) / tc::NBLK * tc::NBLK; }

inline bool tc_supported(const dks_ctx* ctx, int S_cap) {
    if (!ctx->head.tc) return false;
    if (ctx->G > tc::KP - 1) return false;            // M + constant column must fit one K = 16 step
    if (ctx->N > tc::MAX_NPAD) return false;          // one B operand holds the whole background
    if ((long long)tc::smem_bytes(S_cap, tc_nb(ctx->N)) > (long long)ctx->max_smem_optin) return false;
    return true;
}

inline int tc_launch(dks_ctx* ctx, const ExplainParams& p, cudaStream_t stream) {
    tc::TcParams tp;
    tp.p = p;
    tp.BW = ctx->d_BW;
    tp.scores = ctx->d_scores;
    tp.Nb = tc_nb(ctx->N);
    tp.Npad = tc_npad(ctx->N);
    tp.dbg_T = ctx->dbg_T;
    tp.dbg_i = ctx->dbg_i;
    tp.dbg_time = ctx->dbg_time;
    size_t smem = tc::smem_bytes(p.S_cap, tp.Nb);
    void (*kern)(tc::TcParams) = nullptr;
    const bool dbg = tp.dbg_T != nullptr && tp.dbg_i >= 0;
    const bool uw = ctx->uniform_w;
    if (dbg) kern = uw ? tc::explain_wgmma_kernel<true, true> : tc::explain_wgmma_kernel<false, true>;
    else kern = uw ? tc::explain_wgmma_kernel<true, false> : tc::explain_wgmma_kernel<false, false>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return DKS_ERR_CUDA;
    int grid = ctx->sm_count < p.n ? ctx->sm_count : p.n;
    kern<<<grid, tc::NTHREADS, smem, stream>>>(tp);
    ctx->launches += 1;
    return DKS_OK;
}


}  // namespace dks
