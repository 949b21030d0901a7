// Device-side per-instance coalition plans (the sampling part of KernelExplainer.explain, SURVEY App. A.4 step 9).
//
// Upstream draws a fresh plan for every instance from an advancing MT19937 stream.  Here every instance gets its own
// plan from a counter-based generator, Philox4x32-10 keyed by the seed with counter (draw t, global row, block), so the
// plan of a row does not depend on batching, sharding or the number of GPUs.  The sequential semantics are upstream's:
//   draw t: subset size ~ p (sizes not fully enumerated), then a uniform subset of that size (Floyd's algorithm);
//   a mask seen before adds 1 to the weight of its first occurrence (and of its complement row);
//   a new mask takes the next row, followed by its complement when the size is "paired" and a row is left;
//   stop when the budget S is filled; sampled weights are rescaled to the mass the enumerated sizes left over.
// The enumerated prefix (deterministic per M) is copied from the shared plan of that M.  One CTA per instance: draws are
// produced in batches, first occurrences resolved with a shared-memory hash table (atomicMin on the draw index), row
// positions with a block prefix sum -- the result is independent of thread scheduling and of the batch sizes.
//
// The same CTA then prepares the instance's regression: E^T W E = (prefix part, precomputed per M) + scale * (integer
// co-occurrence counts of the sampled rows).  The counts come from the bit-transposed plan -- ballots turn 32 rows into
// one word per column, AND + popc count 32 rows per instruction, multiplicities enter through their bit planes -- and
// the matrix is Cholesky-factored and inverted here, so the explain kernels only do the mat-vec.
// tests/sampler_twin.py is the NumPy twin of the random stream; tests compare the plans bit for bit.
//
// Rows of W 64-bit words: W = 1 up to 64 groups, W = 2 for 65..128 (instances whose groups all vary).  The two-word form
// keys the hash table with 128-bit masks (16-byte shared-memory CAS), transposes four 32-bit words per row for the
// co-occurrence counts, and writes the normal matrix straight to global memory: a 127 x 127 float64 matrix does not fit
// next to the table (DESIGN.md §6.1).  factor_wide_plans_kernel then inverts it in place, one CTA per instance.
#pragma once

#include "dks_common.cuh"
#include "dks_kernels.cuh"

namespace dks {
namespace sampler {

constexpr int THREADS = 256;
constexpr int NWARPS = THREADS / 32;
constexpr int DRAWS_PER_THREAD = 4;
constexpr int BATCH = THREADS * DRAWS_PER_THREAD;
constexpr int MAX_SAMPLED = 4096;          // rows the sampled part of a plan may have (multiplicities stay < 2^15)
constexpr int MAX_SIZES = 64;              // sampled subset sizes (DksSamplingInfo::cdf): M <= 128 has at most 63

using SamplingInfo = ::DksSamplingInfo;

__device__ __forceinline__ void philox4x32_10(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                              uint32_t (&out)[4]) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

__device__ __forceinline__ uint32_t hash_mask(uint64_t m) {
    m ^= m >> 33; m *= 0xff51afd7ed558ccdull; m ^= m >> 33; m *= 0xc4ceb9fe1a85ec53ull; m ^= m >> 33;
    return (uint32_t)m;
}

// a coalition mask of W words (W = 1 or 2) held in registers: bit tests and sets never index the array dynamically
template <int W> struct RowMask { uint64_t w[W]; };
template <int W> __device__ __forceinline__ bool mask_bit(const RowMask<W>& m, int b) {
    if constexpr (W == 1) return (m.w[0] >> b) & 1ull;
    else return ((b < 64 ? m.w[0] : m.w[1]) >> (b & 63)) & 1ull;
}
template <int W> __device__ __forceinline__ void mask_set(RowMask<W>& m, int b) {
    if constexpr (W == 1) m.w[0] |= 1ull << b;
    else { if (b < 64) m.w[0] |= 1ull << b; else m.w[1] |= 1ull << (b - 64); }
}
// hash-table key of the two-word rows: 16-byte shared-memory CAS (sm_90), all-zero = empty slot (a mask is never empty)
struct __align__(16) Key2 { unsigned long long lo, hi; };

// 32 x 32 bit-matrix transpose across the lanes of a warp (5 butterfly stages).  With x_r the word of lane r, lane i ends
// up with bit p = bit (31 - i) of x_(31-p): column c of the block sits in lane 31 - c, row r at bit 31 - r.
__device__ __forceinline__ uint32_t bit_transpose32(uint32_t x, int lane) {
    uint32_t m = 0x0000FFFFu;
#pragma unroll
    for (int j = 16; j != 0; j >>= 1) {
        const uint32_t other = __shfl_xor_sync(0xffffffffu, x, j);
        if (lane & j) x ^= ((other ^ (x >> j)) & m) << j;       // upper lane of the pair: takes the partner's low block
        else x ^= (x ^ (other >> j)) & m;                         // lower lane: takes the partner's high block
        m ^= m << (j >> 1);
    }
    return x;
}

struct SamplerParams {
    int n, G, S_req, stride;
    int table_cap;                  // hash table slots (power of two >= 2 * max_left, >= 256)
    int max_left;                   // most sampled rows any plan of this launch can have (multiple of 32)
    int fstride;                    // doubles per instance in out_chol / out_ainv
    uint64_t seed;
    long long row_offset;           // global index of row 0 of this call
    const int* Mcnt;
    const PlanDev* plans;           // shared plans: source of the enumerated prefix
    const SamplingInfo* info;       // [DKS_MAX_GROUPS + 1]
    const double* const* afix;      // [DKS_MAX_GROUPS + 1] normal matrix of the enumerated prefix
    uint64_t* out_z;                // [n][stride][W]
    double* out_w;                  // [n][stride]
    double* out_chol;               // [n][fstride] E^T W E on exit (factored / inverted by the next kernel)
    double* out_ainv;               // [n][fstride] its inverse (one-word rows)
    int* status;
};

// W = 1: hash table (8-byte keys) + row slots + the staged normal matrix and its scratch; W = 2: 16-byte keys, no staging
inline size_t smem_bytes(int table_cap, int max_left, int G, int W = 1) {
    const size_t nA = G > 1 ? G - 1 : 1;
    return (size_t)table_cap * (8 * W + 4 + 4) + (size_t)max_left * 4 + (W == 1 ? 2 * nA * nA * sizeof(double) : 0);
}

template <int W>
__global__ void __launch_bounds__(THREADS) sample_plans_kernel(SamplerParams p) {
    extern __shared__ __align__(16) unsigned char smraw[];
    const int cap = p.table_cap;
    uint64_t* tkey = reinterpret_cast<uint64_t*>(smraw);                 // [cap][W]
    uint32_t* tfirst = reinterpret_cast<uint32_t*>(tkey + (size_t)cap * W);   // [cap] first draw index
    uint32_t* tcount = tfirst + cap;                                      // [cap] multiplicity among counted draws
    uint32_t* rowslot = tcount + cap;                                     // [max_left] table slot of each sampled row
    double* Abuf = reinterpret_cast<double*>(rowslot + p.max_left);       // W = 1: [2][nA*nA] normal matrix + scratch
    uint32_t* colbits = reinterpret_cast<uint32_t*>(tkey);                // aliases tkey once the draws are done
    __shared__ uint32_t s_warp[NWARPS];
    __shared__ uint32_t s_carry, s_maxcnt;
    __shared__ double s_red[NWARPS];
    __shared__ double s_cdf[MAX_SIZES];
    const int tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;

    for (int i = blockIdx.x; i < p.n; i += gridDim.x) {
        const int M = p.Mcnt[i];
        uint64_t* oz = p.out_z + (size_t)i * p.stride * W;
        double* ow = p.out_w + (size_t)i * p.stride;
        if (M < 2) continue;
        if (W == 2 && M != p.G) continue;          // two-word rows: instances whose groups all vary (the rest are flagged)
        const int S = dks_effective_S(M, p.S_req);
        const PlanDev pd = p.plans[M];
        if (pd.z == nullptr || pd.S != S || S > p.stride || p.afix[M] == nullptr) {
            if (tid == 0) { if (atomicCAS(&p.status[0], 0, DKS_ERR_PLAN_MISSING) == 0) p.status[1] = M; }
            for (int s = tid; s < p.stride * W; s += THREADS) oz[s] = 0ull;
            for (int s = tid; s < p.stride; s += THREADS) ow[s] = 0.0;
            continue;
        }
        const SamplingInfo& inf = p.info[M];
        const int nfixed = inf.nfixed;
        const int left0 = inf.ncdf > 0 ? S - nfixed : 0;
        if (left0 > p.max_left) {
            if (tid == 0) { if (atomicCAS(&p.status[0], 0, DKS_ERR_UNSUPPORTED) == 0) p.status[1] = M; }
            for (int s = tid; s < p.stride * W; s += THREADS) oz[s] = 0ull;
            for (int s = tid; s < p.stride; s += THREADS) ow[s] = 0.0;
            continue;
        }
        // enumerated prefix (deterministic per M); the rest starts empty
        for (int s = tid; s < S * W; s += THREADS) oz[s] = s < nfixed * W ? pd.z[s] : 0ull;
        for (int s = tid; s < S; s += THREADS) ow[s] = s < nfixed ? pd.w[s] : 0.0;
        RowMask<W> fullmask;                    // the M-bit full mask (complements are taken against it)
        fullmask.w[0] = M >= 64 ? ~0ull : ((1ull << M) - 1ull);
        if constexpr (W == 2) fullmask.w[1] = M >= 128 ? ~0ull : ((1ull << (M - 64)) - 1ull);
        if (tid < MAX_SIZES) s_cdf[tid] = tid < inf.ncdf ? inf.cdf[tid] : 2.0;
        const int ncdf = inf.ncdf, n_full = inf.n_full, n_paired = inf.n_paired;
        uint32_t filled = 0u;
        double scale = 0.0;
        __syncthreads();
        if (left0 > 0) {
            for (int h = tid; h < cap * W; h += THREADS) tkey[h] = 0ull;
            for (int h = tid; h < cap; h += THREADS) { tfirst[h] = 0xFFFFFFFFu; tcount[h] = 0u; }
            if (tid == 0) s_carry = 0u;
            __syncthreads();

            const uint64_t grow = (uint64_t)(p.row_offset + i);
            const uint32_t k0 = (uint32_t)p.seed, k1 = (uint32_t)(p.seed >> 32);
            const uint32_t ndraws = 4u * (uint32_t)left0;        // upstream draws 4 * samples_left size picks at most
            uint32_t t0 = 0u;
            while (t0 < ndraws) {
                // draws of this batch: about what the rows still missing need (a draw yields up to two rows)
                const uint32_t missing = (uint32_t)left0 - s_carry;
                uint32_t bsz = missing - missing / 3u + 32u;
                if (bsz > (uint32_t)BATCH) bsz = BATCH;
                const uint32_t tend = min(ndraws, t0 + bsz);
                const uint32_t dpt = (tend - t0 + THREADS - 1u) / THREADS;     // draws per thread in this batch (<= 4)
                RowMask<W> mask[DRAWS_PER_THREAD];
                uint32_t slot[DRAWS_PER_THREAD];
                bool paired[DRAWS_PER_THREAD], valid[DRAWS_PER_THREAD];
                // ---- 1. generate this thread's draws (consecutive t) and register first occurrences
#pragma unroll
                for (int j = 0; j < DRAWS_PER_THREAD; ++j) {
                    const uint32_t t = t0 + (uint32_t)tid * dpt + j;
                    valid[j] = (uint32_t)j < dpt && t < tend;
#pragma unroll
                    for (int q = 0; q < W; ++q) mask[j].w[q] = 0ull;
                    slot[j] = 0u; paired[j] = false;
                    if (!valid[j]) continue;
                    uint32_t rnd[4];
                    philox4x32_10(k0, k1, t, (uint32_t)grow, (uint32_t)(grow >> 32), 0u, rnd);
                    const double u = ((double)rnd[0] + 0.5) * 2.3283064365386963e-10;     // (r + 1/2) / 2^32
                    int idx = 0;
                    while (idx < ncdf - 1 && u >= s_cdf[idx]) ++idx;
                    const int size = idx + n_full + 1;
                    paired[j] = size <= n_paired;
                    // uniform subset of `size` of the M positions (Floyd): for j2 = M-size .. M-1 pick in [0, j2]
                    RowMask<W> mk;
#pragma unroll
                    for (int q = 0; q < W; ++q) mk.w[q] = 0ull;
                    int have = 1;                                     // rnd[1..3] are still unused
                    uint32_t blockno = 0u;
                    for (int j2 = M - size; j2 < M; ++j2) {
                        if (have == 4) {
                            ++blockno;
                            philox4x32_10(k0, k1, t, (uint32_t)grow, (uint32_t)(grow >> 32), blockno, rnd);
                            have = 0;
                        }
                        const uint32_t r32 = have == 0 ? rnd[0] : have == 1 ? rnd[1] : have == 2 ? rnd[2] : rnd[3];
                        ++have;
                        const int pick = (int)(((uint64_t)r32 * (uint64_t)(j2 + 1)) >> 32);
                        const int bit = mask_bit(mk, pick) ? j2 : pick;
                        mask_set(mk, bit);
                    }
                    mask[j] = mk;
                    if constexpr (W == 1) {
                        uint32_t h = hash_mask(mk.w[0]) & (uint32_t)(cap - 1);
                        while (true) {
                            const unsigned long long old =
                                atomicCAS(reinterpret_cast<unsigned long long*>(&tkey[h]), 0ull, (unsigned long long)mk.w[0]);
                            if (old == 0ull || old == (unsigned long long)mk.w[0]) break;
                            h = (h + 1) & (uint32_t)(cap - 1);
                        }
                        slot[j] = h;
                    } else {
                        uint32_t h = hash_mask(mk.w[0] ^ (mk.w[1] * 0x9E3779B97F4A7C15ull)) & (uint32_t)(cap - 1);
                        Key2* tk2 = reinterpret_cast<Key2*>(tkey);
                        const Key2 want{mk.w[0], mk.w[1]};
                        while (true) {
                            const Key2 old = atomicCAS(&tk2[h], Key2{0ull, 0ull}, want);
                            if ((old.lo == 0ull && old.hi == 0ull) || (old.lo == want.lo && old.hi == want.hi)) break;
                            h = (h + 1) & (uint32_t)(cap - 1);
                        }
                        slot[j] = h;
                    }
                    const uint32_t h = slot[j];
                    atomicMin(&tfirst[h], t);
                }
                __syncthreads();
                // ---- 2. rows each draw would create, exclusive prefix over the batch in draw order
                uint32_t rows[DRAWS_PER_THREAD], local = 0u;
#pragma unroll
                for (int j = 0; j < DRAWS_PER_THREAD; ++j) {
                    const uint32_t t = t0 + (uint32_t)tid * dpt + j;
                    const bool fresh = valid[j] && tfirst[slot[j]] == t;
                    rows[j] = fresh ? (paired[j] ? 2u : 1u) : 0u;
                    local += rows[j];
                }
                uint32_t incl = local;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += v;
                }
                if (lane == 31) s_warp[wib] = incl;
                __syncthreads();
                uint32_t warp_off = 0u, total = 0u;
#pragma unroll
                for (int wq = 0; wq < NWARPS; ++wq) { if (wq < wib) warp_off += s_warp[wq]; total += s_warp[wq]; }
                const uint32_t carry = s_carry;
                uint32_t before = carry + warp_off + incl - local;    // rows created by earlier draws
                // ---- 3. draws made while the budget was not yet full count; new masks among them take rows
#pragma unroll
                for (int j = 0; j < DRAWS_PER_THREAD; ++j) {
                    if (valid[j] && before < (uint32_t)left0) {
                        atomicAdd(&tcount[slot[j]], 1u);
                        if (rows[j] > 0u) {
#pragma unroll
                            for (int q = 0; q < W; ++q) oz[(size_t)(nfixed + before) * W + q] = mask[j].w[q];
                            rowslot[before] = slot[j];
                            if (rows[j] == 2u && before + 1u < (uint32_t)left0) {
#pragma unroll
                                for (int q = 0; q < W; ++q)
                                    oz[(size_t)(nfixed + before + 1u) * W + q] = mask[j].w[q] ^ fullmask.w[q];
                                rowslot[before + 1u] = slot[j];
                            }
                        }
                    }
                    before += rows[j];
                }
                __syncthreads();
                if (tid == 0) s_carry = carry + total;
                __syncthreads();
                t0 = tend;
                if (carry + total >= (uint32_t)left0) break;
            }
            // ---- 4. weights: multiplicity of the row's mask, rescaled to the mass left for the sampled sizes
            filled = min(s_carry, (uint32_t)left0);
            double part = 0.0;
            uint32_t mx = 0u;
            for (uint32_t r = tid; r < filled; r += THREADS) {
                const uint32_t c = tcount[rowslot[r]];
                part += (double)c;
                mx = max(mx, c);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                part += __shfl_xor_sync(0xffffffffu, part, o);
                mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            }
            if (lane == 0) { s_red[wib] = part; s_warp[wib] = mx; }
            __syncthreads();
            double totalw = 0.0;
            uint32_t maxcnt = 0u;
#pragma unroll
            for (int wq = 0; wq < NWARPS; ++wq) { totalw += s_red[wq]; maxcnt = max(maxcnt, s_warp[wq]); }
            scale = totalw > 0.0 ? inf.weight_left / totalw : 0.0;
            for (uint32_t r = tid; r < filled; r += THREADS) ow[nfixed + r] = (double)tcount[rowslot[r]] * scale;
            if (tid == 0) s_maxcnt = maxcnt;
            __syncthreads();
        }

        // ---- 5. E^T W E of the instance: prefix part + scale * integer co-occurrence counts of the sampled rows.
        // e_k = z_k - z_L, and e_k e_l = [bits k and l set in z'] with z' = z_L ? ~z : z.  Each warp transposes 32 rows
        // at a time (bit_transpose32: afterwards lane 31-c holds column c of the 32 x 32 bit block, rows in a fixed
        // permuted bit order that is the same for every word transposed), so a column pair is counted 32 rows per popc.
        const int nA = M - 1, L = M - 1;
        const int ngroups = ((int)filled + 31) / 32;
        const int cstride = ngroups | 1;                                // odd word stride: conflict-free column reads
        const int nplanes = filled ? 32 - __clz(s_maxcnt) : 0;
        uint32_t* planes = colbits + (size_t)nA * cstride;            // [nplanes][cstride] bit planes of the multiplicity
        int* Aint = reinterpret_cast<int*>(tfirst);                    // [npairs] (first-occurrence indices are dead)
        const int npairs = nA * (nA + 1) / 2;
        for (int pr = tid; pr < npairs; pr += THREADS) Aint[pr] = 0;
        for (int g = wib; g < ngroups; g += NWARPS) {                // the hash keys are dead: colbits may overwrite them
            const uint32_t r = (uint32_t)g * 32u + lane;
            RowMask<W> zr;
#pragma unroll
            for (int q = 0; q < W; ++q) zr.w[q] = 0ull;
            uint32_t cnt = 0u;
            if (r < filled) {
#pragma unroll
                for (int q = 0; q < W; ++q) zr.w[q] = oz[(size_t)(nfixed + r) * W + q];
                if (mask_bit(zr, L)) {
#pragma unroll
                    for (int q = 0; q < W; ++q) zr.w[q] = ~zr.w[q];
                }
                cnt = tcount[rowslot[r]];
            }
            const int c = 31 - lane;                                  // the column this lane holds after a transpose
#pragma unroll
            for (int hw = 0; hw < 2 * W; ++hw) {                      // 32-bit halves of the row words: columns 32 hw + c
                if (32 * hw < nA) {
                    const uint32_t part = (uint32_t)(zr.w[hw >> 1] >> (32 * (hw & 1)));
                    const uint32_t tb = bit_transpose32(part, lane);
                    if (32 * hw + c < nA) colbits[(size_t)(32 * hw + c) * cstride + g] = tb;
                }
            }
            const uint32_t pl = bit_transpose32(cnt, lane);
            if (c < nplanes) planes[(size_t)c * cstride + g] = pl;
        }
        __syncthreads();
        {
            // work item = (column pair, slice of the row groups); slices keep all threads busy when pairs are few
            int nsl = THREADS / npairs;
            if (nsl < 1) nsl = 1;
            if (nsl > ngroups) nsl = ngroups > 0 ? ngroups : 1;
            const int per = (ngroups + nsl - 1) / nsl;
            for (int item = tid; item < npairs * nsl; item += THREADS) {
                const int pr = item / nsl, sl = item - pr * nsl;
                int k = (int)((sqrtf(8.0f * (float)pr + 1.0f) - 1.0f) * 0.5f);
                while (k * (k + 1) / 2 > pr) --k;
                while ((k + 1) * (k + 2) / 2 <= pr) ++k;
                const int l = pr - k * (k + 1) / 2;                  // pr = k(k+1)/2 + l, l <= k
                const uint32_t* ck = colbits + (size_t)k * cstride;
                const uint32_t* cl = colbits + (size_t)l * cstride;
                const int g1 = min(ngroups, (sl + 1) * per);
                uint32_t acc = 0u;
                for (int g = sl * per; g < g1; ++g) {
                    const uint32_t both = ck[g] & cl[g];
                    for (int b2 = 0; b2 < nplanes; ++b2) acc += (uint32_t)__popc(both & planes[(size_t)b2 * cstride + g]) << b2;
                }
                if (acc) atomicAdd(&Aint[pr], (int)acc);
            }
        }
        __syncthreads();
        const double* afix = p.afix[M];
        // the matrix goes out unfactored: factor_plans_kernel (one warp per instance) or factor_wide_plans_kernel does the
        // serial part.  One-word rows stage it in shared memory for a coalesced copy; two-word rows write it directly.
        double* Aout = p.out_chol + (size_t)i * p.fstride;
        double* Adst = W == 1 ? Abuf : Aout;
        for (int pr = tid; pr < npairs; pr += THREADS) {
            int k = (int)((sqrtf(8.0f * (float)pr + 1.0f) - 1.0f) * 0.5f);
            while (k * (k + 1) / 2 > pr) --k;
            while ((k + 1) * (k + 2) / 2 <= pr) ++k;
            const int l = pr - k * (k + 1) / 2;
            const double v = afix[k * nA + l] + scale * (double)Aint[pr];
            Adst[k * nA + l] = v;
            Adst[l * nA + k] = v;
        }
        __syncthreads();
        if constexpr (W == 1) {
            for (int idx = tid; idx < nA * nA; idx += THREADS) Aout[idx] = Abuf[idx];
            __syncthreads();
        }
    }
}

// Cholesky factor and inverse of every instance's normal matrix, one warp per instance (the chains of square roots and
// divisions are serial: many instances side by side hide their latency).  chol holds the matrix on entry.
constexpr int FACTOR_WARPS = 8;
__global__ void __launch_bounds__(FACTOR_WARPS * 32) factor_plans_kernel(int n, const int* __restrict__ Mcnt, int fstride,
                                                                         double* __restrict__ chol, double* __restrict__ ainv,
                                                                         int nAmax, int* __restrict__ status) {
    extern __shared__ double fsm[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    double* A = fsm + (size_t)wib * 2 * nAmax * nAmax;       // [nA*nA] matrix, then nA*nA of scratch
    const int nw = blockDim.x >> 5;
    for (int i = blockIdx.x * nw + wib; i < n; i += gridDim.x * nw) {
        const int M = Mcnt[i];
        if (M < 2) continue;
        const int nA = M - 1;
        double* ci = chol + (size_t)i * fstride;
        double* ai = ainv + (size_t)i * fstride;
        for (int idx = lane; idx < nA * nA; idx += 32) A[idx] = ci[idx];
        __syncwarp();
        const bool ok = wls_cholesky_warp(A, nA);
        if (!ok && lane == 0) { if (atomicCAS(&status[0], 0, DKS_ERR_NUMERIC) == 0) status[1] = i; }
        __syncwarp();
        for (int idx = lane; idx < nA * nA; idx += 32) ci[idx] = A[idx];
        for (int c = lane; c < nA; c += 32) {               // column c of the inverse solves L L^T x = e_c
            double* x = A + nA * nA + c * nA;
            for (int r = 0; r < nA; ++r) {
                double v = (r == c) ? 1.0 : 0.0;
                for (int k = 0; k < r; ++k) v -= A[r * nA + k] * x[k];
                x[r] = v / A[r * nA + r];
            }
            for (int r = nA - 1; r >= 0; --r) {
                double v = x[r];
                for (int k = r + 1; k < nA; ++k) v -= A[k * nA + r] * x[k];
                x[r] = v / A[r * nA + r];
            }
            for (int r = 0; r < nA; ++r) ai[r * nA + c] = x[r];
        }
        __syncwarp();
    }
}

// Two-word rows (nA <= 127): the inverse of every instance's normal matrix, in place, one CTA per instance.  The explain
// kernel multiplies by the inverse (what upstream's np.linalg.inv gives) and needs no factor, so only one nA x nA buffer
// per instance exists.  Gauss-Jordan elimination without pivoting (the matrix is symmetric positive definite: every pivot
// is a Schur-complement diagonal, > 0 exactly when the matrix is definite); the matrix sits in shared memory and each of
// the nA steps updates all of it in parallel.
constexpr int WIDE_FACTOR_THREADS = 512;
inline size_t wide_factor_smem(int nA) { return sizeof(double) * ((size_t)nA * nA + 2 * (size_t)nA); }

__global__ void __launch_bounds__(WIDE_FACTOR_THREADS) factor_wide_plans_kernel(int n, const int* __restrict__ Mcnt, int G,
                                                                                 int fstride, double* __restrict__ amat,
                                                                                 int* __restrict__ status) {
    extern __shared__ double wsm[];
    const int tid = threadIdx.x;
    __shared__ int s_ok;
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        if (Mcnt[i] != G) continue;
        const int nA = G - 1;
        double* A = wsm;                        // [nA][nA]
        double* colk = A + (size_t)nA * nA;     // [nA] column k before step k
        double* rowk = colk + nA;               // [nA] row k after step k
        double* gi = amat + (size_t)i * fstride;
        __syncthreads();
        for (int idx = tid; idx < nA * nA; idx += blockDim.x) A[idx] = gi[idx];
        if (tid == 0) s_ok = 1;
        __syncthreads();
        for (int k = 0; k < nA; ++k) {
            const double piv = A[k * nA + k];
            if (!(piv > 0.0)) { if (tid == 0) s_ok = 0; }
            const double ip = 1.0 / piv;
            for (int r = tid; r < nA; r += blockDim.x) {
                colk[r] = A[r * nA + k];
                rowk[r] = r == k ? ip : A[k * nA + r] * ip;
            }
            __syncthreads();
            for (int r = tid >> 5; r < nA; r += blockDim.x >> 5) {        // a warp per row: no index division
                const double cr = colk[r];
                for (int c = tid & 31; c < nA; c += 32) {
                    const int idx = r * nA + c;
                    if (r == k) A[idx] = rowk[c];
                    else A[idx] = (c == k ? 0.0 : A[idx]) - cr * rowk[c];
                }
            }
            __syncthreads();
        }
        if (s_ok == 0 && tid == 0) { if (atomicCAS(&status[0], 0, DKS_ERR_NUMERIC) == 0) status[1] = i; }
        for (int idx = tid; idx < nA * nA; idx += blockDim.x) gi[idx] = A[idx];
    }
}

}  // namespace sampler
}  // namespace dks
