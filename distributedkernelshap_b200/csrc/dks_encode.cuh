// Column encodings (dks_set_column_encoding, DESIGN.md §5.0.13, §5.0.16): a tree ensemble, kernel machine, MLP or neighbour
// model behind a scikit-learn Pipeline of per-column steps reads encoded columns, each an exact program over one raw column.  encode_kernel replays the programs on
// raw rows, bit for bit what pipe[:-1].transform gives: the scalers' arithmetic is rounded op by op (__d*_rn: nvcc would
// otherwise contract x * s + o into one fused multiply-add, which numpy does not), the clip keeps NaN as np.clip does, and
// the lookups are exact binary searches over float64 keys.
#pragma once

#include "dks_common.cuh"

namespace dks {
namespace enc {

__host__ __device__ inline double rn_sub(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
__host__ __device__ inline double rn_div(double a, double b) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}
__host__ __device__ inline double rn_mul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ inline double rn_add(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}

// the program of one encoded column (ops [first, first + count)) on the raw value v; *refused is set where a lookup refuses
// the value (its NaN or unknown output is then returned)
__host__ __device__ inline double encode_value(const EncodingDev& e, int first, int count, double v, bool* refused) {
    for (int k = first; k < first + count; ++k) {
        const int* op = e.ops + 4 * (size_t)k;
        const double c0 = e.opv[2 * (size_t)k], c1 = e.opv[2 * (size_t)k + 1];
        switch (op[0]) {
        case DKS_ENC_OP_SUB: v = rn_sub(v, c0); break;
        case DKS_ENC_OP_DIV: v = rn_div(v, c0); break;
        case DKS_ENC_OP_MUL: v = rn_mul(v, c0); break;
        case DKS_ENC_OP_ADD: v = rn_add(v, c0); break;
        case DKS_ENC_OP_CLIP: v = v < c0 ? c0 : (v > c1 ? c1 : v); break;   // np.clip: a NaN compares false and stays
        case DKS_ENC_OP_NANFILL: if (v != v) v = c0; break;
        case DKS_ENC_OP_ISNAN: v = (v != v) ? 1.0 : 0.0; break;
        case DKS_ENC_OP_PIECES:
        case DKS_ENC_OP_TABLE: {
            const int m = op[2];
            const double* t = e.tab + op[3];       // keys [m], outputs [m + 1], NaN output
            if (v != v) {
                if (op[1] & DKS_ENC_NAN_ERROR) *refused = true;
                v = t[2 * m + 1];
                break;
            }
            int lo = 0, hi = m;
            if (op[0] == DKS_ENC_OP_PIECES) {
                // numpy searchsorted(side='right'): the number of edges <= v
                while (lo < hi) { const int mid = (lo + hi) >> 1; if (t[mid] <= v) lo = mid + 1; else hi = mid; }
                v = t[m + lo];
            } else {
                while (lo < hi) { const int mid = (lo + hi) >> 1; if (t[mid] < v) lo = mid + 1; else hi = mid; }
                if (lo < m && t[lo] == v) {
                    v = t[m + lo];
                } else {
                    if (op[1] & DKS_ENC_UNKNOWN_ERROR) *refused = true;
                    v = t[2 * m];
                }
            }
            break;
        }
        }
    }
    return v;
}

// Xe [n][E] from raw rows X [n][D]: one thread per (row, encoded column), grid-stride.  A refused value is reported as
// DKS_ERR_DOMAIN with its row.
__global__ void encode_kernel(const double* __restrict__ X, int n, int D, EncodingDev e, double* __restrict__ Xe,
                              int* __restrict__ status) {
    const long long total = (long long)n * e.E;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(idx / e.E), c = (int)(idx - (long long)i * e.E);
        const int* h = e.hdr + 3 * (size_t)c;
        bool refused = false;
        Xe[idx] = encode_value(e, h[1], h[2], X[(size_t)i * D + h[0]], &refused);
        if (refused && atomicCAS(&status[0], 0, DKS_ERR_DOMAIN) == 0) status[1] = i;
    }
}

// encode_kernel for the models that sum over their columns (kernel machines, MLPs, neighbour models; DESIGN.md §5.0.16): a
// raw infinity that any encoded column reads is refused as well.  Every scikit-learn transformer refuses one, and so do
// these estimators when a column passes through to them.
__global__ void encode_finite_kernel(const double* __restrict__ X, int n, int D, EncodingDev e, double* __restrict__ Xe,
                                     int* __restrict__ status) {
    const long long total = (long long)n * e.E;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(idx / e.E), c = (int)(idx - (long long)i * e.E);
        const int* h = e.hdr + 3 * (size_t)c;
        const double x = X[(size_t)i * D + h[0]];
        bool refused = isinf(x);
        Xe[idx] = encode_value(e, h[1], h[2], x, &refused);
        if (refused && atomicCAS(&status[0], 0, DKS_ERR_DOMAIN) == 0) status[1] = i;
    }
}

}  // namespace enc
}  // namespace dks
