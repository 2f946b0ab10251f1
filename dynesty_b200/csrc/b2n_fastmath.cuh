// b2n_fastmath.cuh -- BRANCH-FREE double-precision log / sqrt / sin-cos for the restricted argument ranges
// of the Box-Muller draws (B2N-RNG v1, oracle/philox.py):
//     lg = log(U0),  U0 in [2^-53, 1)          rad = sqrt(-2 lg)          (sin, cos)(2 pi U1),  U1 in (0, 1)
// Why: libdevice's log / sqrt / sincospi are < 1 ulp but contain slow-path branches (denormals, huge
// arguments); ptxas therefore keeps two draws of one warp in separate basic blocks and their dependency chains
// cannot overlap.  These versions have no control flow at all, so several draws written
// side by side interleave.  Algorithms: fdlibm / FreeBSD msun e_log.c, k_sin.c, k_cos.c (Sun Microsystems,
// public algorithms restated; polynomial coefficients are the published minimax constants), with the
// divisions and square roots replaced by approximate-reciprocal + Newton steps.
// Accuracy (tests/test_fastmath_host.py, 4e6 random arguments against long-double libm): <= 1.5 ulp.
//
// The file compiles for the host as well (B2N_HD), which is how the accuracy test runs without a GPU; on the
// host the hardware approximations are emulated by rounding an exact result to float precision first.
#pragma once
#ifndef __CUDACC_RTC__
#include <stdint.h>
#include <string.h>
#include <math.h>
#endif

#ifdef __CUDACC__
#define B2N_HD __host__ __device__ __forceinline__
#else
#define B2N_HD static inline
#endif

// The polynomial coefficients are read from constant memory on the device: an FP64 instruction takes a constant-bank
// operand for free, while a 64-bit literal costs two register moves each time it is used.  One list feeds the device table and the host values.
#define B2N_FM_CONSTS(X)                                                                                          \
    X(LN2_HI, 6.93147180369123816490e-01) X(LN2_LO, 1.90821492927058770002e-10)                                   \
    X(LG1, 6.666666666666735130e-01) X(LG2, 3.999999999940941908e-01) X(LG3, 2.857142874366239149e-01)            \
    X(LG4, 2.222219843214978396e-01) X(LG5, 1.818357216161805012e-01) X(LG6, 1.531383769920937332e-01)            \
    X(LG7, 1.479819860511658591e-01)                                                                              \
    X(PI_HI, 3.14159265358979311600e+00) X(PI_LO, 1.22464679914735317723e-16)                                     \
    X(S1, -1.66666666666666324348e-01) X(S2, 8.33333333332248946124e-03) X(S3, -1.98412698298579493134e-04)       \
    X(S4, 2.75573137070700676789e-06) X(S5, -2.50507602534068634195e-08) X(S6, 1.58969099521155010221e-10)        \
    X(C1, 4.16666666666666019037e-02) X(C2, -1.38888888888741095749e-03) X(C3, 2.48015872894767294178e-05)        \
    X(C4, -2.75573143513906633035e-07) X(C5, 2.08757232129817482790e-09) X(C6, -1.13596475577881948265e-11)
#define B2N_FM_ENUM(name, val) B2N_FMK_##name,
enum { B2N_FM_CONSTS(B2N_FM_ENUM) B2N_FMK_COUNT };
#define B2N_FM_VAL(name, val) val,
#ifdef __CUDACC__
__constant__ double b2n_fmk_dev[B2N_FMK_COUNT] = {B2N_FM_CONSTS(B2N_FM_VAL)};
#endif
static const double b2n_fmk_host[B2N_FMK_COUNT] = {B2N_FM_CONSTS(B2N_FM_VAL)};
#if defined(__CUDA_ARCH__)
#define B2N_FMK(name) b2n_fmk_dev[B2N_FMK_##name]
#else
#define B2N_FMK(name) b2n_fmk_host[B2N_FMK_##name]
#endif

B2N_HD double b2n_rcp_seed(double d) {        // ~20-bit reciprocal estimate
#if defined(__CUDA_ARCH__)
    double y;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
    return y;
#else
    return (double)(float)(1.0 / d);
#endif
}
B2N_HD double b2n_rsqrt_seed(double a) {      // ~20-bit reciprocal square root estimate
#if defined(__CUDA_ARCH__)
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(a));
    return y;
#else
    return (double)(float)(1.0 / sqrt(a));
#endif
}

// n / d for normal, finite operands far from overflow: two Newton steps on the reciprocal, one residual
// correction of the quotient (error <= 1 ulp)
B2N_HD double b2n_div(double n, double d) {
    double y = b2n_rcp_seed(d);
    double e = fma(-d, y, 1.0);
    y = fma(y, e, y);
    e = fma(-d, y, 1.0);
    y = fma(y, e, y);
    double q = n * y;
    const double r = fma(-d, q, n);
    return fma(r, y, q);
}

// sqrt(a) for normal positive a: coupled Newton iteration on g ~ sqrt(a), h ~ 1/(2 sqrt(a)), final residual step
B2N_HD double b2n_sqrt(double a) {
    const double y = b2n_rsqrt_seed(a);
    double g = a * y, h = 0.5 * y;
    double r = fma(-h, g, 0.5);
    g = fma(g, r, g);
    h = fma(h, r, h);
    r = fma(-h, g, 0.5);
    g = fma(g, r, g);
    h = fma(h, r, h);
    const double d = fma(-g, g, a);
    return fma(d, h, g);
}

// log(x) for normal positive x (fdlibm e_log.c without its special cases)
B2N_HD double b2n_log(double x) {
    const double ln2_hi = B2N_FMK(LN2_HI), ln2_lo = B2N_FMK(LN2_LO);
    const double Lg1 = B2N_FMK(LG1), Lg2 = B2N_FMK(LG2), Lg3 = B2N_FMK(LG3), Lg4 = B2N_FMK(LG4), Lg5 = B2N_FMK(LG5),
                 Lg6 = B2N_FMK(LG6), Lg7 = B2N_FMK(LG7);
    uint64_t bits;
#if defined(__CUDA_ARCH__)
    bits = (uint64_t)__double_as_longlong(x);
#else
    memcpy(&bits, &x, 8);
#endif
    uint32_t hx = (uint32_t)(bits >> 32);
    const uint32_t lx = (uint32_t)bits;
    int k = (int)(hx >> 20) - 1023;
    hx &= 0x000fffffu;
    const uint32_t i = (hx + 0x95f64u) & 0x100000u;          // mantissa >= sqrt(2): halve it, k += 1
    hx |= (i ^ 0x3ff00000u);
    k += (int)(i >> 20);
    const uint64_t mb = ((uint64_t)hx << 32) | lx;
    double m;
#if defined(__CUDA_ARCH__)
    m = __longlong_as_double((long long)mb);
#else
    memcpy(&m, &mb, 8);
#endif
    const double f = m - 1.0;
    const double s = b2n_div(f, 2.0 + f);
    const double dk = (double)k;
    const double z = s * s, w = z * z;
    const double t1 = w * fma(w, fma(w, Lg6, Lg4), Lg2);
    const double t2 = z * fma(w, fma(w, fma(w, Lg7, Lg5), Lg3), Lg1);
    const double R = t2 + t1;
    const double hfsq = 0.5 * f * f;
    return dk * ln2_hi - ((hfsq - fma(s, hfsq + R, dk * ln2_lo)) - f);
}

// (sin, cos)(2 pi u) for u in [0, 1): exact reduction t = 2u = q/2 + r, |r| <= 1/4, then x = pi r in
// double-double and the FreeBSD k_sin / k_cos kernels on |x| <= pi/4, quadrant by selects
B2N_HD void b2n_sincos2pi(double u, double* sn, double* cs) {
    const double PI_HI = B2N_FMK(PI_HI), PI_LO = B2N_FMK(PI_LO);
    const double t = u + u;
    const double qd = rint(t + t);                 // 0 .. 4
    const double r = fma(-0.5, qd, t);             // exact
    const double x = r * PI_HI;
    const double y = fma(r, PI_HI, -x) + r * PI_LO;
    const double z = x * x;
    // k_sin(x, y, 1)
    const double S1 = B2N_FMK(S1), S2 = B2N_FMK(S2), S3 = B2N_FMK(S3), S4 = B2N_FMK(S4), S5 = B2N_FMK(S5), S6 = B2N_FMK(S6);
    const double w = z * z;
    const double rs = S2 + z * (S3 + z * S4) + z * w * (S5 + z * S6);
    const double v = z * x;
    const double S = x - ((z * (0.5 * y - v * rs) - y) - v * S1);
    // k_cos(x, y)
    const double C1 = B2N_FMK(C1), C2 = B2N_FMK(C2), C3 = B2N_FMK(C3), C4 = B2N_FMK(C4), C5 = B2N_FMK(C5), C6 = B2N_FMK(C6);
    const double rc = z * (C1 + z * (C2 + z * C3)) + (w * w) * (C4 + z * (C5 + z * C6));
    const double hz = 0.5 * z, wc = 1.0 - hz;
    const double Cc = wc + (((1.0 - wc) - hz) + (z * rc - x * y));
    const int q = (int)qd & 3;
    const bool swap = (q & 1) != 0;
    const double s0 = swap ? Cc : S, c0 = swap ? S : Cc;
    *sn = (q == 2 || q == 3) ? -s0 : s0;           // q: 0 (S, C)  1 (C, -S)  2 (-S, -C)  3 (-C, S)
    *cs = (q == 1 || q == 2) ? -c0 : c0;
}
