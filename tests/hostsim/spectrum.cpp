/*
 * tests/hostsim/spectrum.cpp — TEST-ONLY host build of the spectrum arithmetic of dumpvdl2_b200/csrc/vdl2_core.cuh (the
 * window and twiddle tables, one segment's butterflies and bin powers, the quantiser, the segment grid with its waiting
 * samples) and the layout of vdl2gpu_spectrum as the C compiler lays it out from include/vdl2gpu.h.  sp_stream restates
 * what the device keeps for one input, chunk by chunk, so the GPU suite can compare the device's figures bit for bit.
 */
#include <stddef.h>
#include <stdint.h>
#include <vector>
#include "vdl2_tables_host.h"
#ifndef __CUDACC__
struct float2 { float x, y; };
#endif
#include "vdl2_core.cuh"
#include "../../include/vdl2gpu.h"

extern "C" {

void sp_tab(float *win, float *tw) {
	vdl2_spec_tab t;
	vdl2_spec_make_tab(&t);
	memcpy(win, t.win, sizeof(t.win));
	memcpy(tw, t.tw, sizeof(t.tw));
}

/* x: 1024 interleaved (re, im) -> p: 1024 bin powers in stored order */
void sp_segment(const float *x, float *p) {
	vdl2_spec_tab t;
	vdl2_spec_make_tab(&t);
	float2 buf[VDL2_SPEC_N];
	vdl2_spec_segment(reinterpret_cast<const float2 *>(x), &t, buf, p);
}

uint64_t sp_q(float p) { return vdl2_spec_q(p); }
uint32_t sp_fft_bin(uint32_t k) { return vdl2_spec_fft_bin(k); }

/* One input fed n_cuts chunks of cuts[k] samples of x (interleaved re, im, back to back); restart[k] != 0 starts a new
 * grid at chunk k and zeroes the figures, as vdl2gpu_restart_receiver does.  Every chunk goes through the grid entry,
 * the segment sources and the waiting samples the kernel uses.  Out: lo, hi, peak bits (1024 each), position. */
void sp_stream(const float *x, const uint32_t *cuts, uint32_t n_cuts, const uint8_t *restart, uint64_t *lo, uint64_t *hi, uint32_t *peak,
		uint64_t *pos_out) {
	vdl2_spec_tab t;
	vdl2_spec_make_tab(&t);
	const float2 *s = reinterpret_cast<const float2 *>(x);
	float2 carry[VDL2_SPEC_N], seg[VDL2_SPEC_N], buf[VDL2_SPEC_N];
	float p[VDL2_SPEC_N];
	uint64_t pos = 0;
	memset(lo, 0, 8 * VDL2_SPEC_N); memset(hi, 0, 8 * VDL2_SPEC_N); memset(peak, 0, 4 * VDL2_SPEC_N);
	for(uint32_t c = 0; c < n_cuts; c++) {
		if(restart && restart[c]) {
			pos = 0;
			memset(lo, 0, 8 * VDL2_SPEC_N); memset(hi, 0, 8 * VDL2_SPEC_N); memset(peak, 0, 4 * VDL2_SPEC_N);
		}
		const vdl2_spec_span e = vdl2_spec_step(pos, cuts[c]);
		const uint32_t nseg = vdl2_spec_segments(e);
		for(uint32_t j = 0; j < nseg; j++) {
			for(uint32_t m = 0; m < VDL2_SPEC_N; m++) {
				const int64_t src = vdl2_spec_src(e, j, m);
				seg[m] = src >= 0 ? s[src] : carry[e.pend + src];
			}
			vdl2_spec_segment(seg, &t, buf, p);
			for(uint32_t k = 0; k < VDL2_SPEC_N; k++) {
				vdl2_pow_fold(lo[k], hi[k], vdl2_spec_q(p[k]));
				const uint32_t b = vdl2_f32_bits(p[k]);
				if(b > peak[k]) peak[k] = b;
			}
		}
		for(uint32_t k = 0; k < vdl2_spec_rest(e); k++) {
			const int64_t src = vdl2_spec_src(e, nseg, k);
			if(src >= 0) carry[k] = s[src];
		}
		s += cuts[c];
	}
	*pos_out = pos;
}

/* the grid entries of n_cuts chunks: pend[k], segments[k], rest[k]; restart as for sp_stream */
void sp_grid(const uint32_t *cuts, uint32_t n_cuts, const uint8_t *restart, uint32_t *pend, uint32_t *segs, uint32_t *rest) {
	uint64_t pos = 0;
	for(uint32_t c = 0; c < n_cuts; c++) {
		if(restart && restart[c]) pos = 0;
		const vdl2_spec_span e = vdl2_spec_step(pos, cuts[c]);
		pend[c] = e.pend; segs[c] = vdl2_spec_segments(e); rest[c] = vdl2_spec_rest(e);
	}
}

/* out = {sizeof, offsetof segments, pending, pow_lo, pow_hi, peak, bins} of the public record */
void sp_layout(uint64_t *out) {
	const uint64_t a[7] = { sizeof(vdl2gpu_spectrum), offsetof(vdl2gpu_spectrum, segments), offsetof(vdl2gpu_spectrum, pending),
			offsetof(vdl2gpu_spectrum, pow_lo), offsetof(vdl2gpu_spectrum, pow_hi), offsetof(vdl2gpu_spectrum, peak), VDL2GPU_SPECTRUM_BINS };
	for(int k = 0; k < 7; k++) out[k] = a[k];
}

uint32_t sp_flag(void) { return VDL2GPU_FLAG_SPECTRUM; }

}
