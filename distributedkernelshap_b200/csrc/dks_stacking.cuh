// Stacking ensembles on the device (DESIGN.md §5.0.20): f(x) = head(W m(x) + b + W_pass x) over K members (tree ensembles,
// kernel machines, MLPs, neighbour models; dks_set_stacking), m(x) [F] the members' kept outputs in member order and W_pass
// the passthrough columns' weights.  The final estimator applies to the members' outputs of each masked row, so the
// background mean ey(s) = sum_j w_j f(z_s ? x : bg_j) needs every member's output on every (s, j): each member's explain
// kernel, in its ROWS instantiation, stores them to one workspace ws [n][F][j1 - j0][S_cap] for a chunk j0 <= j < j1 of the
// background (members in order, on one stream); stacking_reduce_kernel then applies the final estimator per row and adds
// w_j f into ey [n][C][S_cap], the chain continuing across chunks; explain_ensemble_tail_kernel takes the link and the solve
// once.
#pragma once

#include "dks_kernels.cuh"

namespace dks {
namespace stack {

constexpr int THREADS = 256;
constexpr int MAX_F = 128;       // meta columns: DKS_ENS_MAX_MEMBERS x DKS_ENS_MAX_OUT

constexpr int MO = DKS_ENS_MAX_OUT;

// the head's C outputs of the R scores r: identity, [1 - expit(r), expit(r)] (neither half by cancellation), or softmax.
// r and o [MO] are indexed at compile time only, so they stay in registers.
__device__ __forceinline__ void stack_head(const double (&r)[MO], int R, int head, double (&o)[MO]) {
    if (head == DKS_STACK_HEAD_SIGMOID) {
        const double e = exp(-fabs(r[0]));
        const double big = 1.0 / (1.0 + e), small = e / (1.0 + e);
        o[1] = r[0] >= 0 ? big : small;
        o[0] = r[0] >= 0 ? small : big;
    } else if (head == DKS_STACK_HEAD_SOFTMAX) {
        double m = r[0];
#pragma unroll
        for (int q = 1; q < MO; ++q) if (q < R) m = fmax(m, r[q]);
        double sum = 0;
#pragma unroll
        for (int q = 0; q < MO; ++q) if (q < R) { o[q] = exp(r[q] - m); sum += o[q]; }
#pragma unroll
        for (int q = 0; q < MO; ++q) o[q] /= sum;
    } else {
#pragma unroll
        for (int q = 0; q < MO; ++q) o[q] = r[q];
    }
}

// f(x) [n][C] from the members' outputs out_k [K][n][C_k] (members packed in order) and the rows X [n][D] the members read
// (passthrough) and, with dlink, link(f(x)) - link(fnull) for stage 1.  A row a member refused is already reported
// (DKS_ERR_DOMAIN) by that member's predict kernel, which runs first.
__global__ void stacking_predict_kernel(const double* __restrict__ outk, StackDev sd, const double* __restrict__ X, int n,
                                        int link, const double* __restrict__ linkfnull, double* __restrict__ out,
                                        double* __restrict__ dlink, int* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double r[MO], o[MO];
#pragma unroll
    for (int q = 0; q < MO; ++q) r[q] = q < sd.R ? sd.b[q] : 0.0;
    size_t off = 0;
    for (int k = 0, f = 0; k < sd.K; ++k) {
        const double* mk = outk + off + (size_t)i * sd.ck[k] + sd.cfirst[k];
        for (int c = 0; c < sd.ccount[k]; ++c, ++f) {
            const double m = mk[c];
#pragma unroll
            for (int q = 0; q < MO; ++q) if (q < sd.R) r[q] = fma(sd.W[(size_t)q * sd.F + f], m, r[q]);
        }
        off += (size_t)n * sd.ck[k];
    }
    if (sd.Wp != nullptr)
#pragma unroll
        for (int q = 0; q < MO; ++q) {
            if (q >= sd.R) continue;
            double t = 0.0;
            for (int c = 0; c < sd.D; ++c) t = fma(sd.Wp[(size_t)q * sd.D + c], X[(size_t)i * sd.D + c], t);
            r[q] += t;
        }
    stack_head(r, sd.R, sd.head, o);
    predict_epilogue(o, sd.C, i, link, linkfnull, out, dlink, status, false);
}

// passthrough tables: T[row][g][r] = sum over the columns c of group g (CSR goff / gcols over the D columns the members read)
// of W_pass[r][c] rows[row][c], and with tot, tot[row][r] = the sum over every column.  Stage 1 forms XWg of the instances,
// dks_fit BWg and BWtot of the background.
__global__ void stacking_pass_kernel(const double* __restrict__ rows, int nrows, int G, const int* __restrict__ goff,
                                     const int* __restrict__ gcols, StackDev sd, double* __restrict__ T,
                                     double* __restrict__ tot) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)nrows * sd.R) return;
    const int row = (int)(idx / sd.R), q = (int)(idx - (long long)row * sd.R);
    const double* x = rows + (size_t)row * sd.D;
    const double* w = sd.Wp + (size_t)q * sd.D;
    for (int g = 0; g < G; ++g) {
        double t = 0.0;
        for (int e = goff[g]; e < goff[g + 1]; ++e) t = fma(w[gcols[e]], x[gcols[e]], t);
        T[((size_t)row * G + g) * sd.R + q] = t;
    }
    if (tot != nullptr) {
        double t = 0.0;
        for (int c = 0; c < sd.D; ++c) t = fma(w[c], x[c], t);
        tot[(size_t)row * sd.R + q] = t;
    }
}

// One CTA per instance (grid-stride) over the list the members ran on, threads over coalitions.  For every background row j
// of the chunk with w_j != 0: the F meta values of (s, j) from ws (coalesced along s), the scores b + W m in meta-column
// order, plus the passthrough BWtot[j] + sum over the varying positions k in s of XWg[i][vi[k]] - BWg[j][vi[k]] (a group
// that does not vary takes bg_j's value in every row and in x alike, so it never enters), the head, and
// ey[c][s] = fma(w_j, f_c, ey[c][s]).  `first`: the chain starts from zero, else it continues from ey.  Instances with
// M <= 1, a missing plan or a refused f(x) are left to explain_ensemble_tail_kernel.  Every sum runs in a fixed order: ey
// depends neither on the grid nor on where the chunks split the background.
__global__ void __launch_bounds__(THREADS) stacking_reduce_kernel(ExplainParams p, StackDev sd, const double* __restrict__ ws,
                                                                  int j0, int j1, const double* __restrict__ XWg,
                                                                  const double* __restrict__ BWg,
                                                                  const double* __restrict__ BWtot, double* __restrict__ ey,
                                                                  int first) {
    __shared__ double Ws[DKS_ENS_MAX_OUT * MAX_F];
    __shared__ double bs[DKS_ENS_MAX_OUT];
    __shared__ int vi[64];
    const int tid = threadIdx.x;
    const int G = p.G, C = sd.C, R = sd.R, F = sd.F;
    const bool pass = sd.Wp != nullptr;
    const size_t nj = (size_t)(j1 - j0);
    for (int idx = tid; idx < R * F; idx += blockDim.x) Ws[(idx / F) * MAX_F + idx % F] = sd.W[idx];
    if (tid < MO) bs[tid] = tid < R ? sd.b[tid] : 0.0;

    const int ninst = dks_inst_count(p);
    for (int qi = blockIdx.x; qi < ninst; qi += gridDim.x) {
        const int i = dks_inst_at(p, qi);
        const int M = p.Mcnt[i];
        const uint64_t vm = p.vmask[i];
        __syncthreads();  // previous instance done with vi (and, the first time, W and b staged)
        if (M <= 1) continue;
        bool fx_bad = false;
        for (int c = 0; c < C; ++c) fx_bad |= !isfinite(p.dlink[(size_t)i * C + c]);
        if (fx_bad) continue;
        InstPlan pl;
        if (!inst_plan(p, i, M, pl)) continue;
        varying_positions(vm, G, vi);
        __syncthreads();
        const int S = pl.S;
        double* e = ey + (size_t)i * C * p.S_cap;
        const double* xw = pass ? XWg + (size_t)i * G * R : nullptr;
        for (int s = tid; s < S; s += blockDim.x) {
            const uint64_t z = pl.z[s];
            double acc[MO];
#pragma unroll
            for (int c = 0; c < MO; ++c) acc[c] = (first || c >= C) ? 0.0 : e[(size_t)c * p.S_cap + s];
            for (int j = j0; j < j1; ++j) {
                const double wj = p.wbg[j];
                if (wj == 0.0) continue;
                double r[MO], o[MO];
#pragma unroll
                for (int q = 0; q < MO; ++q) r[q] = bs[q];
                const double* m = ws + ((size_t)i * F * nj + (size_t)(j - j0)) * p.S_cap + s;
                for (int f = 0; f < F; ++f) {
                    const double v = m[(size_t)f * nj * p.S_cap];
#pragma unroll
                    for (int q = 0; q < MO; ++q) if (q < R) r[q] = fma(Ws[q * MAX_F + f], v, r[q]);
                }
                if (pass) {
                    const double* bw = BWg + (size_t)j * G * R;
#pragma unroll
                    for (int q = 0; q < MO; ++q) {
                        if (q >= R) continue;
                        double t = BWtot[(size_t)j * R + q];
                        for (int k = 0; k < M; ++k)
                            if ((z >> k) & 1ull) t += xw[(size_t)vi[k] * R + q] - bw[(size_t)vi[k] * R + q];
                        r[q] += t;
                    }
                }
                stack_head(r, R, sd.head, o);
#pragma unroll
                for (int c = 0; c < MO; ++c) if (c < C) acc[c] = fma(wj, o[c], acc[c]);
            }
#pragma unroll
            for (int c = 0; c < MO; ++c) if (c < C) e[(size_t)c * p.S_cap + s] = acc[c];
        }
    }
}

}  // namespace stack
}  // namespace dks
