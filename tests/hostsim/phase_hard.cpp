/*
 * tests/hostsim/phase_hard.cpp — TEST-ONLY host build of vdl2_fastmath.cuh for tests/test_phase_hard.py.
 *
 * phase_hard_eval runs every routine of the header on n samples with the reciprocal / rsqrt seeds scaled by (1 + seed_err),
 * as tools/check_fastmath.cpp does to cover the device's MUFU seeds, and returns per sample:
 *   val[i][0..3]  vdl2_phase_fast, vdl2_phase_fast_nb, vdl2_mag_fast, vdl2_mag_fast_nb (the fast float)
 *   val[i][4]     vdl2_atan2_cr, the device's vdl2_phase_of
 *   val[i][5..6]  the phase as a kernel delivers it: vdl2_phase_fast resp. _nb, and on *slow PHASE_HARD_FALLBACK
 *   slow[i][0..3] the *slow flags of the four fast routines
 * PHASE_HARD_FALLBACK defaults to the device's fall-back, vdl2_atan2_cr.  The tests also build this file with deliberate
 * faults (-DPHASE_HARD_FALLBACK_FAST: the fall-back returns the fast float; a header copy with a narrower guard) to show
 * that the fixture catches them.
 */
#include <cmath>
#include <cstdint>
#include <cstring>

static thread_local double g_seed_err = 0.0;
static inline double perturbed_rcp(double d) { return (double)(1.0f / (float)d) * (1.0 + g_seed_err); }
static inline double perturbed_rsqrt(double d) { return (double)(1.0f / sqrtf((float)d)) * (1.0 + g_seed_err); }
#define VDL2_FM_RCP_SEED_OVERRIDE(d) perturbed_rcp(d)
#define VDL2_FM_RSQRT_SEED_OVERRIDE(d) perturbed_rsqrt(d)
#include "vdl2_fastmath.cuh"

static const double TAB[VDL2_ATAN_TABLE_DOUBLES] = VDL2_ATAN_TABLE_INIT;

static float fallback(float re, float im, float fast) {
#ifdef PHASE_HARD_FALLBACK_FAST
	(void)re; (void)im;
	return fast;
#else
	(void)fast;
	return vdl2_atan2_cr(re, im);
#endif
}

extern "C" void phase_hard_eval(const float *re, const float *im, int n, double seed_err, float *val, int32_t *slow) {
	g_seed_err = seed_err;
	for(int i = 0; i < n; i++) {
		float *v = val + 7 * i;
		int32_t *s = slow + 4 * i;
		int sp = 0, sn = 0, sm = 0, smn = 0;
		v[0] = vdl2_phase_fast(re[i], im[i], TAB, &sp);
		v[1] = vdl2_phase_fast_nb(re[i], im[i], TAB, &sn);
		v[2] = vdl2_mag_fast(re[i], im[i], &sm);
		v[3] = vdl2_mag_fast_nb(re[i], im[i], &smn);
		v[4] = vdl2_atan2_cr(re[i], im[i]);
		v[5] = sp ? fallback(re[i], im[i], v[0]) : v[0];
		v[6] = sn ? fallback(re[i], im[i], v[1]) : v[1];
		s[0] = sp; s[1] = sn; s[2] = sm; s[3] = smn;
	}
}
