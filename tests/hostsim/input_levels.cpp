/*
 * tests/hostsim/input_levels.cpp — TEST-ONLY host build of the input-level arithmetic of dumpvdl2_b200/csrc/vdl2_core.cuh
 * (a component's code, rail and magnitude, a sample's square, the 128-bit fold of the sum of squares) and the layout of
 * vdl2gpu_input_levels as the C compiler lays it out from include/vdl2gpu.h, so the CPU suite can check them.
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

int32_t lv_code(uint32_t fmt, int32_t v) { return vdl2_level_code(fmt, v); }
uint32_t lv_rail(uint32_t fmt, int32_t v) { return vdl2_level_rail(fmt, v); }
uint32_t lv_mag(int32_t c) { return vdl2_level_mag(c); }
uint32_t lv_full_scale(uint32_t fmt) { return vdl2_level_full_scale(fmt); }
uint32_t lv_pow(int32_t ci, int32_t cq) { return vdl2_level_pow(ci, cq); }
uint32_t lv_carry(uint64_t old_lo, uint64_t v) { return vdl2_pow_carry(old_lo, v); }

/* fold n addends, in the order given, into (lo, hi) */
void lv_fold(const uint64_t *v, uint32_t n, uint64_t *lo, uint64_t *hi) {
	for(uint32_t k = 0; k < n; k++) vdl2_pow_fold(*lo, *hi, v[k]);
}

/* out = {sizeof, offsetof samples, sum_i, sum_q, pow_lo, pow_hi, clipped, peak, full_scale} of the public struct, then the
 * same of the device accumulator (which the getter copies field by field) */
void lv_layout(uint64_t *out) {
	const uint64_t a[9] = { sizeof(vdl2gpu_input_levels), offsetof(vdl2gpu_input_levels, samples), offsetof(vdl2gpu_input_levels, sum_i),
			offsetof(vdl2gpu_input_levels, sum_q), offsetof(vdl2gpu_input_levels, pow_lo), offsetof(vdl2gpu_input_levels, pow_hi),
			offsetof(vdl2gpu_input_levels, clipped), offsetof(vdl2gpu_input_levels, peak), offsetof(vdl2gpu_input_levels, full_scale) };
	const uint64_t b[9] = { sizeof(vdl2_levels), offsetof(vdl2_levels, samples), offsetof(vdl2_levels, sum_i), offsetof(vdl2_levels, sum_q),
			offsetof(vdl2_levels, pow_lo), offsetof(vdl2_levels, pow_hi), offsetof(vdl2_levels, clipped), offsetof(vdl2_levels, peak),
			offsetof(vdl2_levels, full_scale) };
	for(int k = 0; k < 9; k++) { out[k] = a[k]; out[9 + k] = b[k]; }
}

uint32_t lv_flag(void) { return VDL2GPU_FLAG_INPUT_LEVELS; }

}
