/*
 * vdl2_fastmath.cuh — (float)atan2((double)im, (double)re) and hypotf(re, im) of a decimated sample without the
 * general-purpose libm routines.
 *
 * The reference obtains a sample's phase as `atan2(im, re)` in double and narrows it to float on store
 * (src/demod.c:232,256).  What the demodulator consumes is therefore fl32(atan2(im, re)): any evaluation of
 * atan2 whose error is far below half a float ulp yields the same float, unless the true value lies within that
 * error of a float rounding boundary (a midpoint between two floats).  vdl2_phase_fast evaluates atan2 in
 * double with a short argument reduction (9 break points k/8, one division, a degree-5 polynomial in t^2:
 * ~22 FP64 operations instead of the ~65 of the libdevice routine) and reports, Ziv style, whether its result
 * is too close to a rounding boundary to be trusted; the caller then falls back to the full routine (about one
 * sample in a million; on the device vdl2_atan2_cr below).  The float returned without the fall-back flag is the
 * correctly rounded one, which away from a rounding boundary is also the narrowed correctly rounded double.
 *
 * Error budget (relative to the final result r; the guard used is 2^-44, 16x the bound):
 *   t = num/den      num, den exact in double (|c| <= 1 has 4 significant bits, the floats 24);
 *                    one Newton step on a >= 2^-18 reciprocal seed leaves |1 - den r| <= 2^-36, and the correction
 *                    t += r (num - den t) squares that: |dt/t| <= 2^-51 (rounding of the last fma dominates)
 *   atan(t)          |t| <= 1/16 (+2^-20 slack from the approximate selection of k); the series is cut after
 *                    t^11/11: truncation <= t^12/13 <= 2^-51.7 relative to t; evaluation error <= 2^-51
 *   A_k + atan(t)    table entry rounded to nearest: 2^-54 absolute (values < 1), sum 2^-53 relative
 *   pi/2 - r, pi - r two-term constants (hi + lo), no cancellation (r <= pi/4 resp. pi/2): 2^-52 relative
 *   total            < 2^-48 relative to |r| >= ~1e-30 (smaller results and non-finite inputs take the slow path)
 */
#ifndef VDL2_FASTMATH_CUH
#define VDL2_FASTMATH_CUH
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define VDL2_FM_HD __host__ __device__ __forceinline__
#else
#define VDL2_FM_HD static inline
#endif

/* {atan(k/8), k/8} for k = 0..8, atan correctly rounded to double (generated with mpmath at 200 bits) */
#define VDL2_ATAN_TABLE_INIT { \
	0.0, 0.0, \
	0x1.fd5ba9aac2f6ep-4, 0.125, \
	0x1.f5b75f92c80ddp-3, 0.25, \
	0x1.6f61941e4def1p-2, 0.375, \
	0x1.dac670561bb4fp-2, 0.5, \
	0x1.1e00babdefeb4p-1, 0.625, \
	0x1.4978fa3269ee1p-1, 0.75, \
	0x1.700a7c5784634p-1, 0.875, \
	0x1.921fb54442d18p-1, 1.0 }
#define VDL2_ATAN_TABLE_DOUBLES 18

#define VDL2_PI_HI 0x1.921fb54442d18p+1
#define VDL2_PI_LO 0x1.1a62633145c07p-53
#define VDL2_PIO2_HI 0x1.921fb54442d18p+0
#define VDL2_PIO2_LO 0x1.1a62633145c07p-54

/* polynomial and folding constants; on the device they sit in constant memory so that they reach the FP64 pipe as
 * constant-bank operands instead of being assembled from two 32-bit immediates each */
#define VDL2_FM_C0 -0x1.745d1745d1746p-4   /* -1/11 */
#define VDL2_FM_C1 0x1.c71c71c71c71cp-4    /*  1/9  */
#define VDL2_FM_C2 -0x1.2492492492492p-3   /* -1/7  */
#define VDL2_FM_C3 0x1.999999999999ap-3    /*  1/5  */
#define VDL2_FM_C4 -0x1.5555555555555p-2   /* -1/3  */
#if defined(__CUDACC__)
static __constant__ double c_vdl2_fm[9] = { VDL2_FM_C0, VDL2_FM_C1, VDL2_FM_C2, VDL2_FM_C3, VDL2_FM_C4, VDL2_PIO2_HI, VDL2_PIO2_LO, VDL2_PI_HI, VDL2_PI_LO };
#endif
#if defined(__CUDA_ARCH__)
#define VDL2_FM_K(i, v) c_vdl2_fm[i]
#else
#define VDL2_FM_K(i, v) (v)
#endif

VDL2_FM_HD double vdl2_fm_rcp_seed(double d) {
#if defined(__CUDA_ARCH__)
	double r;
	asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));      /* MUFU.RCP64H: ~20 good bits */
	return r;
#else
	return (double)(1.0f / (float)d);                          /* any seed good to 2^-18 gives the same bounds */
#endif
}

VDL2_FM_HD double vdl2_fm_fma(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
	return __fma_rn(a, b, c);
#else
	return fma(a, b, c);
#endif
}

/* Returns fl32(atan2(im, re)) and clears *slow, or sets *slow when the caller must use the full routine:
 * non-finite / zero / extreme inputs, or a result within 2^-44 (relative) of a float rounding boundary.
 * `tab` points at VDL2_ATAN_TABLE_DOUBLES doubles initialised with VDL2_ATAN_TABLE_INIT (shared memory on the device). */
VDL2_FM_HD float vdl2_phase_fast(float re, float im, const double *tab, int *slow) {
	const float ax = fabsf(re), ay = fabsf(im);
	const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
	/* comparisons are false for NaN (fmaxf/fminf drop a NaN operand, so both components are tested); zero, infinite
	 * or extreme magnitudes and component ratios below 1e-6 (other than an exact zero) leave the fast path */
	if(!(ax <= 1.0e30f && ay <= 1.0e30f && mx >= 1.0e-30f && (mn >= mx * 1.0e-6f || mn == 0.0f))) { *slow = 1; return 0.0f; }
	/* break point: k = round(8 * mn/mx) from an approximate quotient (any neighbour would do) */
#if defined(__CUDA_ARCH__)
	const float q = __fdividef(mn, mx);                      /* MUFU.RCP + FMUL: approximate is enough here */
	const uint32_t k = __float_as_uint(__fmaf_rn(q, 8.0f, 12582912.0f)) & 15u;
#else
	const float q = mn / mx;
	float kf = q * 8.0f + 12582912.0f;
	uint32_t kb; memcpy(&kb, &kf, 4);
	const uint32_t k = kb & 15u;
#endif
	const double A = tab[2 * k], c = tab[2 * k + 1];
	const double dmx = (double)mx, dmn = (double)mn;
	const double num = vdl2_fm_fma(-c, dmx, dmn);          /* exact */
	const double den = vdl2_fm_fma(c, dmn, dmx);           /* exact */
#ifdef VDL2_FM_RCP_SEED_OVERRIDE
	double r = VDL2_FM_RCP_SEED_OVERRIDE(den);        /* tools/check_fastmath.cpp: a deliberately perturbed seed */
#else
	double r = vdl2_fm_rcp_seed(den);
#endif
	r = vdl2_fm_fma(r, vdl2_fm_fma(-den, r, 1.0), r);      /* one Newton step: |1 - den r| <= 2^-36 */
	double t = num * r;
	t = vdl2_fm_fma(vdl2_fm_fma(-den, t, num), r, t);       /* one correction: t within an ulp of num/den */
	const double s = t * t;
	double p = VDL2_FM_K(0, VDL2_FM_C0);
	p = vdl2_fm_fma(p, s, VDL2_FM_K(1, VDL2_FM_C1));
	p = vdl2_fm_fma(p, s, VDL2_FM_K(2, VDL2_FM_C2));
	p = vdl2_fm_fma(p, s, VDL2_FM_K(3, VDL2_FM_C3));
	p = vdl2_fm_fma(p, s, VDL2_FM_K(4, VDL2_FM_C4));
	double a = A + vdl2_fm_fma(t * s, p, t);
	if(ay > ax) a = (VDL2_FM_K(5, VDL2_PIO2_HI) - a) + VDL2_FM_K(6, VDL2_PIO2_LO);
	if(re < 0.0f) a = (VDL2_FM_K(7, VDL2_PI_HI) - a) + VDL2_FM_K(8, VDL2_PI_LO);
	/* distance of the double from the nearest float rounding boundary: the 29 bits the narrowing drops */
	uint64_t bits;
#if defined(__CUDA_ARCH__)
	bits = (uint64_t)__double_as_longlong(a);
#else
	memcpy(&bits, &a, 8);
#endif
	const uint32_t drop = (uint32_t)bits & 0x1FFFFFFFu;
	const uint32_t dist = drop > 0x10000000u ? drop - 0x10000000u : 0x10000000u - drop;
	/* 2^-44 relative = 2^8..2^9 units of the last double bit.  a == 0 (im == 0, re > 0) is exact. */
	*slow = (dist < 512u && a != 0.0) ? 1 : 0;
	float f = (float)a;
#if defined(__CUDA_ARCH__)
	return __uint_as_float(__float_as_uint(f) | (__float_as_uint(im) & 0x80000000u));
#else
	return copysignf(f, im);
#endif
}

/* The same evaluation as straight-line code (no early exit): the range test only feeds the *slow flag, so the whole
 * routine can be scheduled into the middle of another instruction stream (K1 interleaves it with the filter
 * recurrence of the next decimation group).  Out-of-range inputs run through the arithmetic harmlessly (the result
 * is discarded by the caller when *slow is set; the table index is clamped).  An exact zero sample, which the
 * early-exit version hands to the slow path, is answered here: atan2(+-0, +0) = +-0, atan2(+-0, -0) = +-pi. */
VDL2_FM_HD float vdl2_phase_fast_nb(float re, float im, const double *tab, int *slow) {
	const float ax = fabsf(re), ay = fabsf(im);
	const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
	const bool in_range = ax <= 1.0e30f && ay <= 1.0e30f && mx >= 1.0e-30f && (mn >= mx * 1.0e-6f || mn == 0.0f);
	const bool zero = ax == 0.0f && ay == 0.0f;
#if defined(__CUDA_ARCH__)
	const float q = __fdividef(mn, mx);
	uint32_t k = __float_as_uint(__fmaf_rn(q, 8.0f, 12582912.0f)) & 15u;
#else
	const float q = mn / mx;
	float kf = q * 8.0f + 12582912.0f;
	uint32_t kb; memcpy(&kb, &kf, 4);
	uint32_t k = kb & 15u;
#endif
	k = k > 8u ? 8u : k;
	const double A = tab[2 * k], c = tab[2 * k + 1];
	const double dmx = (double)mx, dmn = (double)mn;
	const double num = vdl2_fm_fma(-c, dmx, dmn);
	const double den = vdl2_fm_fma(c, dmn, dmx);
#ifdef VDL2_FM_RCP_SEED_OVERRIDE
	double r = VDL2_FM_RCP_SEED_OVERRIDE(den);
#else
	double r = vdl2_fm_rcp_seed(den);
#endif
	r = vdl2_fm_fma(r, vdl2_fm_fma(-den, r, 1.0), r);
	double t = num * r;
	t = vdl2_fm_fma(vdl2_fm_fma(-den, t, num), r, t);
	const double s = t * t;
	double p = VDL2_FM_K(0, VDL2_FM_C0);
	p = vdl2_fm_fma(p, s, VDL2_FM_K(1, VDL2_FM_C1));
	p = vdl2_fm_fma(p, s, VDL2_FM_K(2, VDL2_FM_C2));
	p = vdl2_fm_fma(p, s, VDL2_FM_K(3, VDL2_FM_C3));
	p = vdl2_fm_fma(p, s, VDL2_FM_K(4, VDL2_FM_C4));
	double a = A + vdl2_fm_fma(t * s, p, t);
	const double a1 = (VDL2_FM_K(5, VDL2_PIO2_HI) - a) + VDL2_FM_K(6, VDL2_PIO2_LO);
	a = ay > ax ? a1 : a;
	const double a2 = (VDL2_FM_K(7, VDL2_PI_HI) - a) + VDL2_FM_K(8, VDL2_PI_LO);
	a = re < 0.0f ? a2 : a;
	uint64_t bits;
#if defined(__CUDA_ARCH__)
	bits = (uint64_t)__double_as_longlong(a);
#else
	memcpy(&bits, &a, 8);
#endif
	const uint32_t drop = (uint32_t)bits & 0x1FFFFFFFu;
	const uint32_t dist = drop > 0x10000000u ? drop - 0x10000000u : 0x10000000u - drop;
	*slow = (!zero && (!in_range || (dist < 512u && a != 0.0))) ? 1 : 0;
	float f = (float)a;
	uint32_t re_bits, im_bits, f_bits;
#if defined(__CUDA_ARCH__)
	re_bits = __float_as_uint(re); im_bits = __float_as_uint(im); f_bits = __float_as_uint(f);
#else
	memcpy(&re_bits, &re, 4); memcpy(&im_bits, &im, 4); memcpy(&f_bits, &f, 4);
#endif
	if(zero) f_bits = (re_bits & 0x80000000u) ? 0x40490FDBu /* fl32(pi) */ : 0u;
	f_bits = (f_bits & 0x7FFFFFFFu) | (im_bits & 0x80000000u);
#if defined(__CUDA_ARCH__)
	return __uint_as_float(f_bits);
#else
	memcpy(&f, &f_bits, 4);
	return f;
#endif
}

/* hypotf(re, im) as glibc evaluates it for finite arguments, (float)sqrt((double)re*re + (double)im*im) (src/demod.c:238):
 * the sum is formed exactly as there (both squares are exact in double, one rounding), the square root by one coupled Newton
 * step on the hardware seed plus a residual correction (error < 2 ulp of the double) and the same rounding-boundary test as above decides
 * whether the narrowed float can be trusted; otherwise *slow is set and the caller takes the IEEE square root. */
VDL2_FM_HD double vdl2_fm_rsqrt_seed(double d) {
#if defined(__CUDA_ARCH__)
	double r;
	asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));     /* MUFU.RSQ64H */
	return r;
#else
	return (double)(1.0f / sqrtf((float)d));
#endif
}

VDL2_FM_HD float vdl2_mag_fast(float re, float im, int *slow) {
	const float ax = fabsf(re), ay = fabsf(im);
	const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
	if(!(ax <= 1.0e18f && ay <= 1.0e18f && mx >= 1.0e-18f)) { *slow = 1; return 0.0f; }     /* NaN, inf, zero, extremes */
	const double dmx = (double)mx, dmn = (double)mn;
	const double s = vdl2_fm_fma(dmx, dmx, dmn * dmn);         /* == fl64(re^2 + im^2): both squares are exact */
#ifdef VDL2_FM_RSQRT_SEED_OVERRIDE
	const double y = VDL2_FM_RSQRT_SEED_OVERRIDE(s);
#else
	const double y = vdl2_fm_rsqrt_seed(s);
#endif
	double g = s * y, h = 0.5 * y;
	double e = vdl2_fm_fma(-g, h, 0.5);                        /* one coupled Newton step: relative error <= ~2^-35 ... */
	g = vdl2_fm_fma(g, e, g); h = vdl2_fm_fma(h, e, h);
	g = vdl2_fm_fma(vdl2_fm_fma(-g, g, s), h, g);              /* ... squared by the residual correction: g within an ulp of sqrt(s) */
	uint64_t bits;
#if defined(__CUDA_ARCH__)
	bits = (uint64_t)__double_as_longlong(g);
#else
	memcpy(&bits, &g, 8);
#endif
	const uint32_t drop = (uint32_t)bits & 0x1FFFFFFFu;
	const uint32_t dist = drop > 0x10000000u ? drop - 0x10000000u : 0x10000000u - drop;
	*slow = dist < 512u ? 1 : 0;
	return (float)g;
}

/* vdl2_mag_fast as straight-line code: the range test only feeds *slow, so several evaluations can be interleaved by the
 * instruction scheduler (the K2 walk computes the four magnitudes of a block together). */
VDL2_FM_HD float vdl2_mag_fast_nb(float re, float im, int *slow) {
	const float ax = fabsf(re), ay = fabsf(im);
	const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
	const bool in_range = ax <= 1.0e18f && ay <= 1.0e18f && mx >= 1.0e-18f;
	const double dmx = (double)mx, dmn = (double)mn;
	const double s = vdl2_fm_fma(dmx, dmx, dmn * dmn);
#ifdef VDL2_FM_RSQRT_SEED_OVERRIDE
	const double y = VDL2_FM_RSQRT_SEED_OVERRIDE(s);
#else
	const double y = vdl2_fm_rsqrt_seed(s);
#endif
	double g = s * y, h = 0.5 * y;
	double e = vdl2_fm_fma(-g, h, 0.5);
	g = vdl2_fm_fma(g, e, g); h = vdl2_fm_fma(h, e, h);
	g = vdl2_fm_fma(vdl2_fm_fma(-g, g, s), h, g);
	uint64_t bits;
#if defined(__CUDA_ARCH__)
	bits = (uint64_t)__double_as_longlong(g);
#else
	memcpy(&bits, &g, 8);
#endif
	const uint32_t drop = (uint32_t)bits & 0x1FFFFFFFu;
	const uint32_t dist = drop > 0x10000000u ? drop - 0x10000000u : 0x10000000u - drop;
	*slow = (!in_range || dist < 512u) ? 1 : 0;
	return (float)g;
}

/* ---- the fall-back: atan2(im, re) correctly rounded to double, narrowed to float ----
 * This is the reference's float whenever its libm's atan2 is correctly rounded (glibc's is on every sample of
 * tests/golden/phase_hard.json).  It is not always the float nearest to atan2: within half a double ulp of a float midpoint
 * the double is the midpoint itself and the narrowing goes to the even float (double rounding), and so does the reference.
 * The samples that reach the fall-back are the ones next to a float midpoint, where an atan2 in double with an error of an
 * ulp or two (libdevice documents 2) can narrow to the other float.  This routine continues the reduction of
 * vdl2_phase_fast in double-double:
 *   t = num/den      num, den exact; th = RN(num/den), tl = RN((num - den th)/den), the residual exact: |dt/t| <= 2^-104
 *   atan(t)          |t| <= 1/16: the series to t^23 (truncation t^25/25 <= 2^-100 t); the terms up to t^11 with
 *                    double-double coefficients, the rest in double (their share is below 2^-48 t)
 *   A_k + atan(t)    atan(k/8) and the folding constants pi/2, pi as hi + lo pairs (mpmath at 200 bits)
 *   total            below 2^-98 relative; hi of the normalised sum is the double nearest to it, so hi is the correctly
 *                    rounded double unless atan2 lies within 2^-98 (relative) of a midpoint between two doubles
 * About 150 double operations; the pipeline calls it for a few samples per million. */
/* {atan(k/8) hi, lo} for k = 0..8 (mpmath at 200 bits; the hi parts are VDL2_ATAN_TABLE_INIT's) */
#define VDL2_ATAN_DD_INIT { 0.0, 0.0, 0x1.fd5ba9aac2f6ep-4, -0x1.cd37686760c17p-59, 0x1.f5b75f92c80ddp-3, 0x1.8ab6e3cf7afbdp-57, \
	0x1.6f61941e4def1p-2, -0x1.c63aae6f6e918p-56, 0x1.dac670561bb4fp-2, 0x1.a2b7f222f65e2p-56, 0x1.1e00babdefeb4p-1, -0x1.928df287a668fp-58, \
	0x1.4978fa3269ee1p-1, 0x1.2419a87f2a458p-56, 0x1.700a7c5784634p-1, -0x1.8c34d25aadef6p-56, 0x1.921fb54442d18p-1, 0x1.1a62633145c07p-55 }
#if defined(__CUDACC__)
static __constant__ double c_vdl2_atan_dd[18] = VDL2_ATAN_DD_INIT;
#endif
#if defined(__CUDA_ARCH__)
#define VDL2_ATAN_DD(i) c_vdl2_atan_dd[i]
#else
static const double vdl2_atan_dd_host[18] = VDL2_ATAN_DD_INIT;
#define VDL2_ATAN_DD(i) vdl2_atan_dd_host[i]
#endif

VDL2_FM_HD void vdl2_dd_add(double ah, double al, double bh, double bl, double *rh, double *rl) {
	const double s = ah + bh, v = s - ah;
	const double e = ((ah - (s - v)) + (bh - v)) + (al + bl);          /* two-sum of the high parts, then the low parts */
	*rh = s + e;
	*rl = e - (*rh - s);
}

VDL2_FM_HD void vdl2_dd_mul(double ah, double al, double bh, double bl, double *rh, double *rl) {
	const double p = ah * bh;
	const double e = vdl2_fm_fma(ah, bh, -p) + (ah * bl + al * bh);   /* exact product of the high parts + cross terms */
	*rh = p + e;
	*rl = e - (*rh - p);
}

VDL2_FM_HD float vdl2_atan2_cr(float re, float im) {
	if(!(fabsf(re) <= 3.4028235e38f && fabsf(im) <= 3.4028235e38f) || (re == 0.0f && im == 0.0f)) {
		/* NaN, infinite or (+-0, +-0): the C99 results are those of the sample with each infinity made +-1 and the
		 * finite component +-0, and of (+-1, +-0) for (+-0, +-0) */
		if(isnan(re) || isnan(im)) return re + im;
		const bool ri = isinf(re), ii = isinf(im);
		re = copysignf(ri || !ii ? 1.0f : 0.0f, re);
		im = copysignf(ii ? 1.0f : 0.0f, im);
	}
	const double ax = fabs((double)re), ay = fabs((double)im);
	const double mx = fmax(ax, ay), mn = fmin(ax, ay);
	const int k = (int)(mn / mx * 8.0 + 0.5);                           /* |t| <= 1/16 */
	const double c = 0.125 * k;
	const double num = vdl2_fm_fma(-c, mx, mn), den = vdl2_fm_fma(c, mn, mx);    /* exact */
	const double th = num / den;
	const double tl = vdl2_fm_fma(-th, den, num) / den;
	double sh, sl;
	vdl2_dd_mul(th, tl, th, tl, &sh, &sl);
	/* t^13 .. t^23 in double, then t^3 .. t^11 in double-double */
	double tail = -0x1.642c8590b2164p-5;                                 /* -1/23 */
	tail = tail * sh + 0x1.8618618618618p-5;                             /*  1/21 */
	tail = tail * sh - 0x1.af286bca1af28p-5;                             /* -1/19 */
	tail = tail * sh + 0x1.e1e1e1e1e1e1ep-5;                             /*  1/17 */
	tail = tail * sh - 0x1.1111111111111p-4;                             /* -1/15 */
	tail = tail * sh + 0x1.3b13b13b13b14p-4;                             /*  1/13 */
	const double ch[5] = { -0x1.745d1745d1746p-4, 0x1.c71c71c71c71cp-4, -0x1.2492492492492p-3, 0x1.999999999999ap-3, -0x1.5555555555555p-2 };
	const double cl[5] = { 0x1.745d1745d1746p-59, 0x1.c71c71c71c71cp-58, -0x1.2492492492492p-57, -0x1.999999999999ap-57, -0x1.5555555555555p-56 };
	double ph = tail, pl = 0.0;
#pragma unroll
	for(int j = 0; j < 5; j++) {                                         /* p = p s + (-1)^j / (2j + 1), j = 5 .. 1 */
		vdl2_dd_mul(ph, pl, sh, sl, &ph, &pl);
		vdl2_dd_add(ph, pl, ch[j], cl[j], &ph, &pl);
	}
	double rh, rl;
	vdl2_dd_mul(ph, pl, sh, sl, &ph, &pl);                              /* atan t = t + t (s p) */
	vdl2_dd_mul(th, tl, ph, pl, &ph, &pl);
	vdl2_dd_add(th, tl, ph, pl, &rh, &rl);
	vdl2_dd_add(VDL2_ATAN_DD(2 * k), VDL2_ATAN_DD(2 * k + 1), rh, rl, &rh, &rl);
	if(ay > ax) vdl2_dd_add(VDL2_PIO2_HI, VDL2_PIO2_LO, -rh, -rl, &rh, &rl);
	if(re < 0.0f) vdl2_dd_add(VDL2_PI_HI, VDL2_PI_LO, -rh, -rl, &rh, &rl);
	const float f = (float)rh;
	return copysignf(f, im);
}

#endif
