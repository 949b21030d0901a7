// Link arithmetic shared by the solve kernels: ln(a1) - ln(a0) of two positive float32 sums around a 64-entry table.
// Plain C++ apart from the bit casts, so the host-side emulation of the simple kernels (tests/emu) compiles it too.
#pragma once

namespace dks {

// ---- cheap link arithmetic.  f32<->f64 conversions run at 16 lanes/clk/SM (they share the XU pipe with MUFU) and a
// float64 division + log() is a ~110-instruction dependent chain.  So the per-row log is evaluated in fp32 around a 64-entry table with two float64 ops at the end.
//
// ln(a1) - ln(a0) for positive float32 sums.  a = 2^e * m, m in [1,2) = c_k (1 + r) with c_k = 1 + (k + 1/2)/64 the centre
// of the k-th of 64 mantissa intervals, |r| <= 2^-7.  r = m/c_k - 1 is formed with a two-float reciprocal
// (fmaf(m, rc_hi, -1) + m*rc_lo: abs error ~5e-10) and ln(1+r) = r - r^2/2 + r^3/3 - r^4/4 + r^5/5 in fp32 (abs error
// ~1e-9); only e*ln2 + ln c_k (table, float64) is combined in float64.  Total abs error ~2e-9.
#define DKS_LOGTAB_SIZE 64
struct LogTabEntry { float rc_hi, rc_lo; double lnc; };
__device__ __forceinline__ void logtab_fill(LogTabEntry* tab, int k) {
    const double c = 1.0 + ((double)k + 0.5) / 64.0;
    const double rc = 1.0 / c;
    LogTabEntry e;
    e.rc_hi = (float)rc;
    e.rc_lo = (float)(rc - (double)e.rc_hi);
    e.lnc = log(c);
    tab[k] = e;
}
__device__ __forceinline__ double fast_log_ratio(float a1, float a0, const LogTabEntry* __restrict__ tab) {
    const int b1 = __float_as_int(a1), b0 = __float_as_int(a0);
    const LogTabEntry t1 = tab[(b1 >> 17) & 63], t0 = tab[(b0 >> 17) & 63];
    const float m1 = __int_as_float((b1 & 0x007FFFFF) | 0x3F800000), m0 = __int_as_float((b0 & 0x007FFFFF) | 0x3F800000);
    const float r1 = fmaf(m1, t1.rc_hi, -1.f) + m1 * t1.rc_lo, r0 = fmaf(m0, t0.rc_hi, -1.f) + m0 * t0.rc_lo;
    const float p1 = r1 * (1.f + r1 * (-0.5f + r1 * (0.33333334f + r1 * (-0.25f + r1 * 0.2f))));
    const float p0 = r0 * (1.f + r0 * (-0.5f + r0 * (0.33333334f + r0 * (-0.25f + r0 * 0.2f))));
    const int de = (b1 >> 23) - (b0 >> 23);
    return fma((double)de, 0.6931471805599453094, t1.lnc - t0.lnc) + (double)(p1 - p0);
}

}  // namespace dks
