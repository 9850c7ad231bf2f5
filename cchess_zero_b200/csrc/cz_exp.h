/* cz_exp: exp(x) in double precision for x <= 0, written with + - * / and integer conversions only, so that the library (nvcc,
 * --fmad=false) and the test specification (a C compiler, -ffp-contract=off) compute the same bits.  CUDA's exp() and the C
 * library's exp() are each accurate to about an ulp, but they are not the same function and differ in the last bit on some inputs.
 *
 *   x = k ln2 + r, k = round(x / ln2), |r| <= ln2 / 2; r is formed with ln2 split in two parts (Cody-Waite), the first of which has
 *   32 trailing zero bits, so k * CZ_LN2_HI is exact for |k| < 2^21;
 *   exp(r) = 1 + r + r^2 (1/2 + r (1/6 + ...)), the Taylor series to r^14 (truncation below 2^-60 of the result) in Horner form,
 *   with the leading 1 + r added last;
 *   exp(x) = exp(r) * 2^k, 2^k formed by squaring 1/2 (exact).  Below 2^-1022 the result is scaled in two steps, the first exact,
 *   so the one rounding is that of the final product (subnormal results).
 *
 * Special values: cz_exp(0) = 1, cz_exp(-inf) = 0, cz_exp(NaN) = NaN; x < -746 gives 0 (exp(x) < 2^-1076 rounds to 0).  x > 0 is
 * outside the domain (the softmax priors subtract the maximum first) and is evaluated as x = 0. */
#ifndef CZ_EXP_H
#define CZ_EXP_H

#ifdef __CUDACC__
#define CZ_EXP_FN static __host__ __device__ __forceinline__
#else
#define CZ_EXP_FN static inline
#endif

#define CZ_LN2_HI 6.93147180369123816490e-01  /* 0x3fe62e42fee00000 */
#define CZ_LN2_LO 1.90821492927058770002e-10  /* 0x3dea39ef35793c76: ln2 - CZ_LN2_HI */
#define CZ_INV_LN2 1.44269504088896338700e+00

CZ_EXP_FN double cz_exp(double x) {
    if (x != x) return x;                 /* NaN */
    if (x < -746.0) return 0.0;           /* -inf included */
    if (x > 0.0) x = 0.0;                 /* outside the domain: clamped, exp(0) = 1 */
    const int k = -(int)(0.5 - x * CZ_INV_LN2);            /* round(x / ln2), x <= 0 */
    const double kd = (double)k;
    const double r = (x - kd * CZ_LN2_HI) - kd * CZ_LN2_LO;
    double q = 1.0 / 87178291200.0;                        /* 1/14! */
    q = 1.0 / 6227020800.0 + r * q;                        /* 1/13! */
    q = 1.0 / 479001600.0 + r * q;
    q = 1.0 / 39916800.0 + r * q;
    q = 1.0 / 3628800.0 + r * q;
    q = 1.0 / 362880.0 + r * q;
    q = 1.0 / 40320.0 + r * q;
    q = 1.0 / 5040.0 + r * q;
    q = 1.0 / 720.0 + r * q;
    q = 1.0 / 120.0 + r * q;
    q = 1.0 / 24.0 + r * q;
    q = 1.0 / 6.0 + r * q;
    q = 0.5 + r * q;
    double p = 1.0 + (r + (r * r) * q);
    int n = -k;                                            /* 0 <= n <= 1077 */
    if (n > 1022) { p = p * (1.0 / 340282366920938463463374607431768211456.0); n -= 128; }   /* * 2^-128, exact */
    double s = 1.0, b = 0.5;
    while (n) {                                            /* s = 2^-n, exact */
        if (n & 1) s = s * b;
        b = b * b;
        n >>= 1;
    }
    return p * s;
}

#undef CZ_EXP_FN
#endif
