/*
 * tests/hostsim/channel_levels.cpp — TEST-ONLY host build of the channel-level arithmetic of dumpvdl2_b200/csrc/vdl2_core.cuh
 * (a decimated sample's power, its bin and its quantised power, the 128-bit fold), the library's own input filter taps
 * (vdl2_tables_host.h) and the layout of vdl2gpu_channel_levels as the C compiler lays it out from include/vdl2gpu.h, so the
 * CPU suite can check them.
 */
#include <stddef.h>
#include <stdint.h>
#include "vdl2_tables_host.h"
#ifndef __CUDACC__
struct float2 { float x, y; };
#endif
#include "vdl2_core.cuh"
#include "../../include/vdl2gpu.h"

extern "C" {

float cl_pow(float re, float im) { return vdl2_chlv_pow(re, im); }
uint32_t cl_bin(float p) { return vdl2_chlv_bin(p); }
uint64_t cl_q(float p) { return vdl2_chlv_q(p); }

/* fold n addends, in the order given, into (lo, hi) */
void cl_fold(const uint64_t *v, uint32_t n, uint64_t *lo, uint64_t *hi) {
	for(uint32_t k = 0; k < n; k++) vdl2_pow_fold(*lo, *hi, v[k]);
}

/* the input filter of a context at this sample rate: A[3], B[3] */
void cl_lpf(uint32_t rate, float *A, float *B) { make_lpf(rate, A, B); }

/* out = {sizeof, offsetof hist, pow_lo, pow_hi, peak_pow, mag_lp, mag_nf, nf_pwr_dbfs} of the public struct */
void cl_layout(uint64_t *out) {
	const uint64_t a[8] = { sizeof(vdl2gpu_channel_levels), offsetof(vdl2gpu_channel_levels, hist), offsetof(vdl2gpu_channel_levels, pow_lo),
			offsetof(vdl2gpu_channel_levels, pow_hi), offsetof(vdl2gpu_channel_levels, peak_pow), offsetof(vdl2gpu_channel_levels, mag_lp),
			offsetof(vdl2gpu_channel_levels, mag_nf), offsetof(vdl2gpu_channel_levels, nf_pwr_dbfs) };
	for(int k = 0; k < 8; k++) out[k] = a[k];
}

uint32_t cl_flag(void) { return VDL2GPU_FLAG_CHANNEL_LEVELS; }
uint32_t cl_bins(void) { return VDL2_CHLV_BINS; }

}
