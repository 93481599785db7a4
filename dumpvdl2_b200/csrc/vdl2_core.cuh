/*
 * vdl2_core.cuh — per-channel / per-burst device functions of libvdl2gpu.so.
 *
 * Everything here is __host__ __device__ so that tests/hostsim can compile the very same source with
 * g++ (-ffp-contract=off) and step it on the CPU against the oracle BEFORE GPU time is spent.  The host
 * instantiation is test-only; the product never runs it (no CPU fallback).
 *
 * Floating-point discipline: the reference source read strictly (no fast-math, no contraction).  Every
 * float/double operation goes through an explicit round-to-nearest intrinsic so that nvcc can neither
 * fuse (FMA) nor reassociate it; promotions to double happen exactly where C's usual arithmetic
 * conversions put them in the reference (M_PI, M_PI_4 are double there).
 * Reference citations are file:line under /root/reference.
 */
#ifndef VDL2_CORE_CUH
#define VDL2_CORE_CUH
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include "vdl2_types.h"
#include "vdl2_fastmath.cuh"

/* branch layout hints: a sync decision, a noise-floor update or a lock are rare events of the walk's hot path */
#define VDL2_UNLIKELY(x) __builtin_expect(!!(x), 0)
#define VDL2_LIKELY(x) __builtin_expect(!!(x), 1)
#if defined(__CUDACC__)
#define VDL2_HD __host__ __device__ __forceinline__
#else
#define VDL2_HD static inline
#endif

#if defined(__CUDA_ARCH__)
#define F_MUL(a, b) __fmul_rn((a), (b))
#define F_ADD(a, b) __fadd_rn((a), (b))
#define F_SUB(a, b) __fsub_rn((a), (b))
#define F_DIV(a, b) __fdiv_rn((a), (b))
#define D_MUL(a, b) __dmul_rn((a), (b))
#define D_ADD(a, b) __dadd_rn((a), (b))
#define D_SUB(a, b) __dsub_rn((a), (b))
#define D_DIV(a, b) __ddiv_rn((a), (b))
#define D_SQRT(a) __dsqrt_rn((a))
#define D_TO_F(a) __double2float_rn((a))
#define VDL2_ATOMIC_ADD_U32(p, v) atomicAdd((unsigned int *)(p), (unsigned int)(v))
#define VDL2_ATOMIC_ADD_I32(p, v) atomicAdd((int *)(p), (int)(v))
#define VDL2_THREADFENCE() __threadfence()
#define VDL2_LDG(p) __ldg(p)
#else
#define VDL2_LDG(p) (*(p))
#define F_MUL(a, b) ((float)(a) * (float)(b))
#define F_ADD(a, b) ((float)(a) + (float)(b))
#define F_SUB(a, b) ((float)(a) - (float)(b))
#define F_DIV(a, b) ((float)(a) / (float)(b))
#define D_MUL(a, b) ((double)(a) * (double)(b))
#define D_ADD(a, b) ((double)(a) + (double)(b))
#define D_SUB(a, b) ((double)(a) - (double)(b))
#define D_DIV(a, b) ((double)(a) / (double)(b))
#define D_SQRT(a) sqrt((double)(a))
#define D_TO_F(a) ((float)(a))
static inline uint32_t vdl2_host_fetch_add_u32(uint32_t *p, uint32_t v) { uint32_t o = *p; *p = o + v; return o; }
static inline int32_t vdl2_host_fetch_add_i32(int32_t *p, int32_t v) { int32_t o = *p; *p = o + v; return o; }
#define VDL2_ATOMIC_ADD_U32(p, v) vdl2_host_fetch_add_u32((uint32_t *)(p), (uint32_t)(v))
#define VDL2_ATOMIC_ADD_I32(p, v) vdl2_host_fetch_add_i32((int32_t *)(p), (int32_t)(v))
#define VDL2_THREADFENCE() do {} while (0)
#endif

#define VDL2_PURE_SATURATED 0x40000000u
/* the metric at sample n reads the phases of samples n-150, n-140, ..., n: it is a pure function of the
 * decimated stream (and can be precomputed in parallel) once that many samples were written without a reset */
#define VDL2_PURE_NEEDED 151u

#define VDL2_PI 3.14159265358979323846          /* M_PI */
#define VDL2_TWO_PI 6.28318530717958647692      /* 2.0f * M_PI evaluated in double */
#define VDL2_PI_4 0.78539816339744830962        /* M_PI_4 */
/* smallest floats strictly greater than the double constants: `f > M_PI` (float promoted to double)
 * is the same predicate as `f >= VDL2_PI_F_ABOVE` */
#define VDL2_PI_F_ABOVE 3.14159274101257324f
#define VDL2_TWO_PI_F_ABOVE 6.28318548202514648f

/* ------------------------------------------------------------------------------------------------
 * K2: demodulator + header decode, one decimated sample at a time      src/demod.c:205-286
 * ---------------------------------------------------------------------------------------------- */
struct vdl2_chan {
	float prev_phi, prev_dphi, dphi, pherr0, pherr1, pherr2, ppm_error, mag_lp, mag_nf, frame_pwr;
	int32_t ring_pos, sclk, nfcnt, frame_pwr_cnt;
	uint32_t state;
	uint64_t acc;                /* last 64 burst bits, newest in bit 0 */
	uint32_t nbits, need_bits, datalen, syndrome;
	int32_t slot;
	uint32_t burst_seq;
	uint64_t sync_dec_index;
	uint32_t freq;
	uint32_t cnt_sync, cnt_hdr_good;
	uint32_t pure_run;           /* consecutive DM_INIT samples since the last demod_reset (saturating) */
};

struct vdl2_event_rec {          /* == vdl2gpu_event / vo_event */
	uint32_t channel, kind;
	uint64_t dec_index;
	int32_t i[8];
	float f[8];
};

struct vdl2_k2_env {
	const float *pr_phase;       /* 16 */
	const float *lr_X;           /* 16 */
	float lr_denom;
	float max_ppm;
	const uint32_t *unwrap_lut;  /* vdl2_tables::unwrap_lut (shared memory on the device) */
	uint32_t s27;                /* first 27 scrambler output bits, first bit in bit 26 */
	vdl2_burst_slot *pool;
	int32_t *free_list;
	uint32_t *ready;
	vdl2_queue_ctl *ctl;
	vdl2_event_rec *events;
	uint32_t event_cap;
	uint32_t trace;
};

VDL2_HD uint32_t vdl2_dec_state(const vdl2_chan &v) { return (v.state >> VDL2_DEC_SHIFT) & 3u; }
VDL2_HD void vdl2_set_dec_state(vdl2_chan &v, uint32_t s) { v.state = (v.state & VDL2_ST_LOCKED) | (s << VDL2_DEC_SHIFT); }

/* src/demod.c:205-220 */
VDL2_HD void vdl2_demod_reset(vdl2_chan &v) {
	v.state = (VDL2_DEC_HEADER << VDL2_DEC_SHIFT);      /* DM_INIT + DEC_HEADER */
	v.need_bits = VDL2_HEADER_LEN;
	v.nbits = 0;
	v.acc = 0;
	v.sclk = 0;
	v.pherr1 = v.pherr2 = 1000.f;
	v.frame_pwr = 0.f;
	v.frame_pwr_cnt = 0;
	v.pure_run = 0;
}

/* src/demod.c:379-392 */
VDL2_HD void vdl2_chan_init(vdl2_chan &v, uint32_t freq) {
	memset(&v, 0, sizeof(v));
	v.mag_nf = 2.0f;
	v.freq = freq;
	v.slot = -1;
	vdl2_demod_reset(v);
	v.pure_run = VDL2_PURE_SATURATED;      /* the ring starts as zeros == "phases" of the samples before the stream */
}

VDL2_HD void vdl2_emit_event(const vdl2_k2_env &env, const vdl2_event_rec &e) {
	uint32_t k = VDL2_ATOMIC_ADD_U32(&env.ctl->n_events, 1u);
	if(k < env.event_cap) env.events[k] = e;
}

/* src/decode.c:55-61 */
VDL2_HD uint32_t vdl2_header_syndrome(uint32_t word) {
	const uint32_t rows[VDL2_HDRFECLEN] = { 0x001FFF0u, 0x07E1FE8u, 0x18E61E4u, 0x1B6A662u, 0x0D3CAA1u };
	uint32_t syn = 0;
#pragma unroll
	for(int r = 0; r < VDL2_HDRFECLEN; r++) {
		uint32_t x = word & rows[r];
		x ^= x >> 16; x ^= x >> 8; x ^= x >> 4; x ^= x >> 2; x ^= x >> 1;
		syn |= (x & 1u) << (VDL2_HDRFECLEN - 1 - r);
	}
	return syn;
}

/* error pattern per syndrome (src/decode.c:63-96): syndromes of single-bit errors map back to that bit,
 * the seven remaining syndromes to the reference's chosen double-bit patterns. */
VDL2_HD uint32_t vdl2_header_error_pattern(uint32_t syn) {
	switch(syn) {
		case 0: return 0;
		case 3: return 0x0800004u; case 5: return 0x0800002u; case 13: return 0x1100000u;
		case 18: return 0x0804000u; case 20: return 0x0808000u; case 23: return 0x1010000u;
		default: break;
	}
	/* single-bit: find the column of the check matrix equal to syn */
	const uint32_t rows[VDL2_HDRFECLEN] = { 0x001FFF0u, 0x07E1FE8u, 0x18E61E4u, 0x1B6A662u, 0x0D3CAA1u };
	for(int bit = 0; bit < VDL2_HEADER_LEN; bit++) {
		uint32_t col = 0;
#pragma unroll
		for(int r = 0; r < VDL2_HDRFECLEN; r++) col |= ((rows[r] >> bit) & 1u) << (VDL2_HDRFECLEN - 1 - r);
		if(col == syn) return 1u << bit;
	}
	return 0;
}

VDL2_HD uint32_t vdl2_synd_weight(uint32_t syn) {          /* src/decode.c:98-100 */
	if(syn == 0) return 0;
	return (syn == 3 || syn == 5 || syn == 13 || syn == 18 || syn == 20 || syn == 23) ? 2u : 1u;
}

VDL2_HD int vdl2_fec_octets_for(uint32_t len) {             /* src/decode.c:124-133 */
	return len < 3 ? 0 : len < 31 ? 2 : len < 68 ? 4 : 6;
}

VDL2_HD uint32_t vdl2_reverse17(uint32_t v) {               /* reverse(v, 17): src/bitstream.c:152-164 */
	uint32_t r = 0;
#pragma unroll
	for(int b = 0; b < VDL2_TRLEN; b++) r |= ((v >> b) & 1u) << (VDL2_TRLEN - 1 - b);
	return r;
}

/* src/demod.c:98-103 */
VDL2_HD float vdl2_para_vertex(float x, float y1, float y2, float y3) {
	const float d = 3.f, d2 = 6.f, denom = -54.f;   /* d = SYNC_SKIP, denom = (float)(d * 2*d * (-d)) */
	float xd = F_SUB(x, d), x2d = F_SUB(x, d2);
	float qa = F_DIV(F_ADD(F_ADD(F_MUL(x, F_SUB(y2, y1)), F_MUL(xd, F_SUB(y1, y3))), F_MUL(x2d, F_SUB(y3, y2))), denom);
	float qb = F_DIV(F_ADD(F_ADD(F_MUL(F_MUL(x, x), F_SUB(y1, y2)), F_MUL(F_MUL(xd, xd), F_SUB(y3, y1))),
				F_MUL(F_MUL(x2d, x2d), F_SUB(y2, y3))), denom);
	return F_DIV(-qb, F_MUL(2.f, qa));
}

/* src/demod.c:137-141: `unwrap -= 2.0f * M_PI` / `unwrap += 2.0f * M_PI` — double arithmetic narrowed to float on
 * store: unwrap' = fl32((double)unwrap -/+ 2pi_d).  The same value is obtained here in FP32 only, branch-free:
 * with 2pi_d = H + L (H = fl32(2pi_d), L = fl32(2pi_d - H)) and (s, e) = TwoSum(unwrap, sg*H) exactly,
 * unwrap' = fl32(s + fl32(e + sg*L)).  unwrap can only take the 77 values reachable from 0 in at most 15 steps of
 * +-2pi; the identity holds for every one of their 138 transitions (tests/test_hostsim.py enumerates them), and
 * for sg == 0 it returns unwrap unchanged.  No double-precision conversions, no divergent branch. */
#define VDL2_TWO_PI_HI 6.28318548202514648f      /* fl32(2*M_PI) */
#define VDL2_TWO_PI_LO -1.74845553146951715e-7f  /* fl32(2*M_PI - VDL2_TWO_PI_HI) */
VDL2_HD float vdl2_unwrap_step(float unwrap, float step) {
	const float sg = (step >= VDL2_PI_F_ABOVE) ? -1.f : ((step <= -VDL2_PI_F_ABOVE) ? 1.f : 0.f);
	const float b = F_MUL(sg, VDL2_TWO_PI_HI);
	const float s = F_ADD(unwrap, b);
	const float bb = F_SUB(s, unwrap);
	const float e = F_ADD(F_SUB(unwrap, F_SUB(s, bb)), F_SUB(b, bb));
	return F_ADD(s, F_ADD(e, F_MUL(sg, VDL2_TWO_PI_LO)));
}

/* src/demod.c:129-171: regression metric over the 16 preamble-spaced phases ph[.][0..15] (oldest first) for N
 * independent evaluations at once.  p0[k] = squared-error sum, slope[k] = fitted phase slope (freq_err).
 * The N evaluations share nothing; interleaving them in one instruction stream gives the N-fold instruction
 * level parallelism a single warp per SM sub-partition needs to hide the FP32/FP64 pipeline latency.
 * Every evaluation performs exactly the reference's operations in the reference's order. */
/* the same update through the transition table (vdl2_tables::unwrap_lut): `row` is the byte offset of the current
 * state's row; one 8-byte look-up gives the next row and the next value.  Bit-identical to vdl2_unwrap_step by
 * construction (the table is built with the reference's double arithmetic) and checked state by state in
 * tests/test_hostsim.py. */
VDL2_HD float vdl2_unwrap_lut_step(const uint32_t *lut, uint32_t &row, float step) {
	const uint32_t off = row + ((step >= VDL2_PI_F_ABOVE) ? 8u : 0u) + ((step <= -VDL2_PI_F_ABOVE) ? 16u : 0u);
#ifdef __CUDA_ARCH__
	const uint2 e = *reinterpret_cast<const uint2 *>(reinterpret_cast<const char *>(lut) + off);
	row = e.x;
	return __uint_as_float(e.y);
#else
	const uint32_t *e = lut + (off >> 2);
	float val;
	row = e[0];
	memcpy(&val, &e[1], 4);
	return val;
#endif
}

template<int N, bool LUT>
VDL2_HD void vdl2_metric_core_n(const float (*ph)[VDL2_PREAMBLE_SYMS], const float *pr_phase, const float *lr_X,
		float lr_denom, const uint32_t *unwrap_lut, float *p0_out, float *slope_out) {
	float err[N][VDL2_PREAMBLE_SYMS];
	float unwrap[N], prev[N], mean[N], slope[N], p0[N];
	uint32_t row[N];
#pragma unroll
	for(int k = 0; k < N; k++) {
		unwrap[k] = 0.f;
		row[k] = 0u;
		prev[k] = F_SUB(ph[k][0], pr_phase[0]);
		mean[k] = prev[k];
		err[k][0] = prev[k];
	}
#pragma unroll
	for(int i = 1; i < VDL2_PREAMBLE_SYMS; i++) {
#pragma unroll
		for(int k = 0; k < N; k++) {
			float cur = F_SUB(ph[k][i], pr_phase[i]);
			float step = F_SUB(cur, prev[k]);
			prev[k] = cur;
			if(LUT) unwrap[k] = vdl2_unwrap_lut_step(unwrap_lut, row[k], step);
			else unwrap[k] = vdl2_unwrap_step(unwrap[k], step);
			err[k][i] = F_ADD(cur, unwrap[k]);
			mean[k] = F_ADD(mean[k], err[k][i]);
		}
	}
#pragma unroll
	for(int k = 0; k < N; k++) { mean[k] = F_MUL(mean[k], 0.0625f); slope[k] = 0.f; p0[k] = 0.f; }   /* /= 16: exact */
#pragma unroll
	for(int i = 0; i < VDL2_PREAMBLE_SYMS; i++) {
#pragma unroll
		for(int k = 0; k < N; k++) {
			err[k][i] = F_SUB(err[k][i], mean[k]);
			slope[k] = F_ADD(slope[k], F_MUL(lr_X[i], err[k][i]));
		}
	}
#pragma unroll
	for(int k = 0; k < N; k++) slope[k] = F_DIV(slope[k], lr_denom);
#pragma unroll
	for(int i = 0; i < VDL2_PREAMBLE_SYMS; i++) {
#pragma unroll
		for(int k = 0; k < N; k++) {
			float e = F_SUB(err[k][i], F_MUL(slope[k], lr_X[i]));
			p0[k] = F_ADD(p0[k], F_MUL(e, e));
		}
	}
#pragma unroll
	for(int k = 0; k < N; k++) { p0_out[k] = p0[k]; slope_out[k] = slope[k]; }
}

VDL2_HD float vdl2_metric_core(const float *ph, const float *pr_phase, const float *lr_X, float lr_denom, float *slope_out) {
	float p0;
	vdl2_metric_core_n<1, false>(reinterpret_cast<const float (*)[VDL2_PREAMBLE_SYMS]>(ph), pr_phase, lr_X, lr_denom, nullptr, &p0, slope_out);
	return p0;
}

/* src/demod.c:105-198.  `ring` points at this channel's column, consecutive phases `rs` floats apart.
 * When `have_pre` the metric pair (pre_p0, pre_slope) was computed by the parallel pre-pass from the same 16
 * phases and is used as is; otherwise it is evaluated here from the ring. */
VDL2_HD int vdl2_preamble_metric(vdl2_chan &v, const float *ring, int rs, const vdl2_k2_env &env,
		uint32_t chan_idx, uint64_t dec_index, bool have_pre, float pre_p0, float pre_slope) {
	float p0, slope;
	if(have_pre) {
		p0 = pre_p0; slope = pre_slope;
	} else {
		float ph[VDL2_PREAMBLE_SYMS];
		int idx = v.ring_pos;
#pragma unroll
		for(int i = 0; i < VDL2_PREAMBLE_SYMS; i++) {
			idx += VDL2_SPS;
			if(idx >= VDL2_SYNC_BUFLEN) idx -= VDL2_SYNC_BUFLEN;
			ph[i] = ring[idx * rs];
		}
		p0 = vdl2_metric_core(ph, env.pr_phase, env.lr_X, env.lr_denom, &slope);
	}
	v.pherr0 = p0;
	if(VDL2_UNLIKELY(v.pherr1 < 4.f && p0 > v.pherr1)) {
		float vertex = vdl2_para_vertex((float)v.sclk, v.pherr2, v.pherr1, p0);
		float neg = -roundf(vertex);
		/* reachable metric triples give vertex in [-4.5,-1.5] (DESIGN.md); the guard only keeps the
		 * conversion defined for inputs the reference itself would mis-handle */
		v.sclk = (neg > -1.0e6f && neg < 1.0e6f) ? (int)neg : 0;
		int sp = v.ring_pos - v.sclk;
		if(sp < 0) sp += VDL2_SYNC_BUFLEN;
		sp = ((sp % VDL2_SYNC_BUFLEN) + VDL2_SYNC_BUFLEN) % VDL2_SYNC_BUFLEN;
		v.prev_phi = ring[sp * rs];
		v.dphi = v.prev_dphi;
		v.ppm_error = D_TO_F(D_MUL(D_DIV((double)F_MUL((float)VDL2_SYMBOL_RATE, v.dphi),
						D_MUL(VDL2_TWO_PI, (double)v.freq)), 1e+6));
		int accepted = !(env.max_ppm != 0.f && fabsf(v.ppm_error) > env.max_ppm);
		if(env.trace) {
			vdl2_event_rec e;
			memset(&e, 0, sizeof(e));
			e.channel = chan_idx; e.kind = 1; e.dec_index = dec_index;
			e.i[0] = v.sclk; e.i[1] = v.ring_pos; e.i[2] = sp; e.i[3] = accepted;
			e.f[0] = v.pherr2; e.f[1] = v.pherr1; e.f[2] = p0; e.f[3] = vertex;
			e.f[4] = v.prev_phi; e.f[5] = v.dphi; e.f[6] = v.ppm_error;
			vdl2_emit_event(env, e);
		}
		v.pherr1 = v.pherr2 = 1000.f;
		return accepted;
	}
	v.pherr2 = v.pherr1;
	v.pherr1 = p0;
	v.prev_dphi = slope;
	return 0;
}

/* DEC_HEADER branch of decode_vdl2_burst: src/decode.c:198-258 */
VDL2_HD void vdl2_header_step(vdl2_chan &v, const vdl2_k2_env &env, uint32_t chan_idx, uint64_t dec_index) {
	/* nbits == 27 here: 9 symbols; descramble all of them, the header is the first 25 */
	uint32_t raw27 = (uint32_t)(v.acc & 0x7FFFFFFu) ^ env.s27;
	uint32_t word = raw27 >> 2;
	uint32_t raw25 = word;
	word &= (1u << (VDL2_TRLEN + VDL2_HDRFECLEN)) - 1u;
	uint32_t syn = vdl2_header_syndrome(word);
	word ^= vdl2_header_error_pattern(syn);
	v.syndrome = syn;
	if(syn == 0) v.cnt_hdr_good++;
	int status = VDL2_BURST_OK;
	uint32_t datalen = 0, octets = 0, fec = 0;
	if((word & ((1u << (VDL2_TRLEN + VDL2_HDRFECLEN)) - 1u)) != word) {
		status = VDL2_ERR_CRC_BAD;
	} else {
		datalen = vdl2_reverse17((word >> VDL2_HDRFECLEN) & 0x1FFFFu);
		if((syn != 0 && datalen > VDL2_MAX_FRAME_LENGTH_CORRECTED) || datalen > VDL2_MAX_FRAME_LENGTH)
			status = VDL2_ERR_TOO_LONG;
	}
	if(status == VDL2_BURST_OK) {
		octets = datalen / 8 + ((datalen % 8) != 0);
		fec = (octets / VDL2_RS_K) * (VDL2_RS_N - VDL2_RS_K) + (uint32_t)vdl2_fec_octets_for(octets % VDL2_RS_K);
		if(fec == 0) status = VDL2_ERR_NO_FEC;
	}
	if(status == VDL2_BURST_OK) {
		v.datalen = datalen;
		v.need_bits = VDL2_HEADER_LEN + 8 * (octets + fec);
		vdl2_set_dec_state(v, VDL2_DEC_DATA);
		/* take a burst slot from the pool (K3 returns it) */
		int32_t top = VDL2_ATOMIC_ADD_I32(&env.ctl->free_top, -1) - 1;
		if(top >= 0) {
			v.slot = env.free_list[top];
		} else {
			VDL2_ATOMIC_ADD_I32(&env.ctl->free_top, 1);
			VDL2_ATOMIC_ADD_U32(&env.ctl->pool_overflows, 1u);
			v.slot = -1;
		}
	} else {
		vdl2_set_dec_state(v, VDL2_DEC_IDLE);
	}
	if(env.trace) {
		vdl2_event_rec e;
		memset(&e, 0, sizeof(e));
		e.channel = chan_idx; e.kind = 2; e.dec_index = dec_index;
		e.i[0] = (int32_t)raw25; e.i[1] = (int32_t)syn; e.i[2] = (int32_t)datalen; e.i[3] = status;
		e.i[4] = (int32_t)(status == VDL2_BURST_OK ? v.need_bits - VDL2_HEADER_LEN : VDL2_HEADER_LEN);
		vdl2_emit_event(env, e);
	}
}

/* all requested bits are in: hand the burst to K3 (the data part of decode_vdl2_burst runs there) */
VDL2_HD void vdl2_burst_complete(vdl2_chan &v, const vdl2_k2_env &env, uint32_t chan_idx) {
	if(v.slot >= 0) {
		vdl2_burst_slot *s = &env.pool[v.slot];
		if(v.nbits & 31u) s->words[v.nbits >> 5] = (uint32_t)(v.acc << (32u - (v.nbits & 31u)));
		s->channel = chan_idx;
		s->burst_seq = v.burst_seq;
		s->datalen_bits = v.datalen;
		s->syndrome = v.syndrome;
		s->nbits = v.nbits;
		s->frame_pwr = v.frame_pwr;
		s->mag_nf = v.mag_nf;
		s->ppm_error = v.ppm_error;
		s->sync_lo = (uint32_t)v.sync_dec_index;
		s->sync_hi = (uint32_t)(v.sync_dec_index >> 32);
		s->freq = v.freq;
		uint32_t k = VDL2_ATOMIC_ADD_U32(&env.ctl->n_ready, 1u);
		env.ready[k] = (uint32_t)v.slot;
		v.slot = -1;
	}
	v.burst_seq++;
	vdl2_set_dec_state(v, VDL2_DEC_IDLE);
}

/* phase and magnitude of one decimated sample, exactly as the reference obtains them:
 *   (float)atan2((double)im, (double)re)                 src/demod.c:232,256 (double atan2, narrowed on store)
 *   hypotf(re, im)                                       src/demod.c:238; glibc evaluates sqrt(x*x + y*y) in double and narrows
 * Both are pure functions of the sample, so the K2a pre-pass computes them for every decimated sample of the
 * chunk in parallel and the sequential state machine only consumes them.
 * The phase is atan2 correctly rounded to double, narrowed.  On the device that is vdl2_atan2_cr (vdl2_fastmath.cuh):
 * libdevice's double atan2 (2 ulp) narrows to the wrong float on some samples next to a float rounding boundary
 * (tests/golden/phase_hard.json).  Host builds use glibc's atan2, which the reference uses. */
VDL2_HD float vdl2_phase_of(float re, float im) {
#if defined(__CUDA_ARCH__)
	return vdl2_atan2_cr(re, im);
#else
	return D_TO_F(atan2((double)im, (double)re));
#endif
}
VDL2_HD float vdl2_mag_of(float re, float im) {
	return D_TO_F(D_SQRT(D_ADD(D_MUL((double)re, (double)re), D_MUL((double)im, (double)im))));
}

/* DM_INIT, every sample: src/demod.c:231-232 */
VDL2_HD void vdl2_init_write(vdl2_chan &v, float *ring, int rs, float phi) {
	v.ring_pos = (v.ring_pos + 1 == VDL2_SYNC_BUFLEN) ? 0 : v.ring_pos + 1;
	ring[v.ring_pos * rs] = phi;
	if(v.pure_run < VDL2_PURE_SATURATED) v.pure_run++;
}

/* DM_INIT, every SYNC_SKIP-th sample: noise floor + sync attempt, src/demod.c:236-249 */
VDL2_HD void vdl2_init_eval(vdl2_chan &v, const float *ring, int rs, const vdl2_k2_env &env, uint32_t chan_idx,
		uint64_t dec_index, float mag, bool have_pre, float pre_p0, float pre_slope) {
	const float one_minus_mag_lp = 1.0f - 0.9f, one_minus_nf_lp = 1.0f - 0.85f;
	v.mag_lp = F_ADD(F_MUL(v.mag_lp, 0.9f), F_MUL(mag, one_minus_mag_lp));
	if(VDL2_UNLIKELY(++v.nfcnt == 1000)) {
		v.nfcnt = 0;
		v.mag_nf = F_ADD(F_ADD(F_MUL(0.85f, v.mag_nf), F_MUL(one_minus_nf_lp, fminf(v.mag_lp, v.mag_nf))), 0.0001f);
	}
	if(vdl2_preamble_metric(v, ring, rs, env, chan_idx, dec_index, have_pre, pre_p0, pre_slope)) {
		v.cnt_sync++;
		v.sync_dec_index = dec_index;
		v.state |= VDL2_ST_LOCKED;
	}
}

/* DM_SYNC, every SPS-th sample: one D8PSK symbol, src/demod.c:256-283: slicing, frame power and bit packing (vdl2_symbol
 * without what a full bit count triggers) */
VDL2_HD void vdl2_symbol_bits(vdl2_chan &v, const vdl2_k2_env &env, float re, float im, float phi) {
	float dphi = F_SUB(F_SUB(phi, v.prev_phi), v.dphi);
	if(dphi < 0.f) dphi = D_TO_F(D_ADD((double)dphi, VDL2_TWO_PI));
	else if(dphi >= VDL2_TWO_PI_F_ABOVE) dphi = D_TO_F(D_SUB((double)dphi, VDL2_TWO_PI));
	dphi = D_TO_F(D_DIV((double)dphi, VDL2_PI_4));
	int sym = (int)roundf(dphi) % 8;
	if(sym < 0) sym += 8;
	float p = F_ADD(F_MUL(re, re), F_MUL(im, im));
	v.frame_pwr = F_DIV(F_ADD(F_MUL(v.frame_pwr, (float)v.frame_pwr_cnt), p), (float)(v.frame_pwr_cnt + 1));
	v.frame_pwr_cnt++;
	v.prev_phi = phi;
	/* Gray map {0,1,3,2,6,7,5,4} (src/demod.c:223), three bits MSB first (src/bitstream.c:46-56) */
	uint32_t bits = (uint32_t)(sym ^ (sym >> 1));
	uint32_t before = v.nbits;
	v.acc = (v.acc << 3) | bits;
	v.nbits = before + 3;
	if((before >> 5) != (v.nbits >> 5) && v.slot >= 0)
		env.pool[v.slot].words[before >> 5] = (uint32_t)(v.acc >> (v.nbits & 31u));
}

VDL2_HD void vdl2_symbol(vdl2_chan &v, const vdl2_k2_env &env, uint32_t chan_idx, uint64_t dec_index,
		float re, float im, float phi) {
	vdl2_symbol_bits(v, env, re, im, phi);
	if(v.nbits >= v.need_bits) {
		if(vdl2_dec_state(v) == VDL2_DEC_HEADER) vdl2_header_step(v, env, chan_idx, dec_index);
		else if(vdl2_dec_state(v) == VDL2_DEC_DATA) vdl2_burst_complete(v, env, chan_idx);
	}
}

/* src/demod.c:222-286 — one decimated sample of one channel; `phi`/`mag` = vdl2_phase_of / vdl2_mag_of of it */
VDL2_HD void vdl2_demod_step_pm(vdl2_chan &v, float *ring, int rs, const vdl2_k2_env &env,
		uint32_t chan_idx, uint64_t dec_index, float re, float im, float phi, float mag,
		bool pre_valid, float pre_p0, float pre_slope) {
	if(vdl2_dec_state(v) == VDL2_DEC_IDLE) vdl2_demod_reset(v);
	if(!(v.state & VDL2_ST_LOCKED)) {
		vdl2_init_write(v, ring, rs, phi);
		if(++v.sclk < VDL2_SYNC_SKIP) return;
		v.sclk = 0;
		vdl2_init_eval(v, ring, rs, env, chan_idx, dec_index, mag, pre_valid && v.pure_run >= VDL2_PURE_NEEDED, pre_p0, pre_slope);
		return;
	}
	if(++v.sclk < VDL2_SPS) return;
	v.sclk = 0;
	vdl2_symbol(v, env, chan_idx, dec_index, re, im, phi);
}

/* K2 walks the chunk in blocks of VDL2_WALK_BLOCK decimated samples per channel.  `dec`, `phase`, `mag` point at
 * this channel's entry for the first sample of the block; consecutive samples are `stride` elements apart and
 * phase[-k*stride] is valid for k <= 160 (history prefix).  Three paths, chosen per channel:
 *   fast    searching (DM_INIT) with a pure phase ring: the four sync attempts that fall into the block are
 *           evaluated together (vdl2_metric_core_n<4>) from the phase plane, then the twelve samples are applied;
 *   locked  in a burst (DM_SYNC): only the one or two symbol instants of the block are touched;
 *   generic anything else (the 150 samples after a reset, the sample after a burst): the per-sample step.
 * All three produce exactly what twelve calls of vdl2_demod_step_pm would. */
#define VDL2_WALK_BLOCK 12
template<bool LUT>
VDL2_HD void vdl2_walk_block(vdl2_chan &v, float *ring, int rs, const vdl2_k2_env &env, uint32_t chan_idx, uint64_t idx0,
		const float2 *dec, const float *phase, const float *mag, size_t stride) {
	int resume = 0;
	if(!(v.state & VDL2_ST_LOCKED) && vdl2_dec_state(v) != VDL2_DEC_IDLE && v.pure_run >= VDL2_PURE_NEEDED
			&& v.sclk >= 0 && v.sclk < VDL2_SYNC_SKIP) {      /* sclk can sit above SYNC_SKIP after a max_ppm veto */
		const int first = (VDL2_SYNC_SKIP - 1) - v.sclk;                  /* offset of the first attempt in the block */
		float ph[4][VDL2_PREAMBLE_SYMS], p0[4], sl[4], mg[4], pw[VDL2_WALK_BLOCK];
#pragma unroll
		for(int j = 0; j < 4; j++) {
			const ptrdiff_t e = (ptrdiff_t)(first + VDL2_SYNC_SKIP * j);
#pragma unroll
			for(int i = 0; i < VDL2_PREAMBLE_SYMS; i++)
				ph[j][i] = VDL2_LDG(phase + (e - 150 + 10 * i) * (ptrdiff_t)stride);
			mg[j] = VDL2_LDG(mag + e * (ptrdiff_t)stride);
		}
#pragma unroll
		for(int t = 0; t < VDL2_WALK_BLOCK; t++) pw[t] = VDL2_LDG(phase + (ptrdiff_t)t * (ptrdiff_t)stride);
		vdl2_metric_core_n<4, LUT>(ph, env.pr_phase, env.lr_X, env.lr_denom, env.unwrap_lut, p0, sl);
		/* the block is four groups of SYNC_SKIP samples; in each the attempt falls on local offset `first`,
		 * and the sample clock is back at its entry value at every group boundary */
		const int sclk_entry = v.sclk;
		bool go = true;
#pragma unroll
		for(int g = 0; g < 4; g++) {
			if(go) {
#pragma unroll
				for(int u = 0; u < VDL2_SYNC_SKIP; u++)
					if(u <= first) vdl2_init_write(v, ring, rs, pw[VDL2_SYNC_SKIP * g + u]);
				v.sclk = 0;
				vdl2_init_eval(v, ring, rs, env, chan_idx, idx0 + (uint64_t)(VDL2_SYNC_SKIP * g + first), mg[g], true, p0[g], sl[g]);
				if(VDL2_UNLIKELY((v.state & VDL2_ST_LOCKED) || v.sclk != 0)) {
					/* locked on a preamble, or the preamble was vetoed by max_ppm (src/demod.c:190-192 leaves the
					 * sample clock at the sync point): the per-sample path takes over for the rest of the block */
					go = false;
					resume = VDL2_SYNC_SKIP * g + first + 1;
				} else {
#pragma unroll
					for(int u = 0; u < VDL2_SYNC_SKIP; u++)
						if(u > first) vdl2_init_write(v, ring, rs, pw[VDL2_SYNC_SKIP * g + u]);
					v.sclk = sclk_entry;
				}
			}
		}
		if(go) resume = VDL2_WALK_BLOCK;
	}
	int t = resume;
	while(t < VDL2_WALK_BLOCK) {
		if((v.state & VDL2_ST_LOCKED) && vdl2_dec_state(v) != VDL2_DEC_IDLE) {
			const int tsym = t + (VDL2_SPS - 1) - v.sclk;                  /* sample on which ++sclk reaches SPS */
			if(tsym >= VDL2_WALK_BLOCK) { v.sclk += VDL2_WALK_BLOCK - t; break; }
			const float2 d = VDL2_LDG(dec + (ptrdiff_t)tsym * (ptrdiff_t)stride);
			const float phi = VDL2_LDG(phase + (ptrdiff_t)tsym * (ptrdiff_t)stride);
			v.sclk = 0;
			vdl2_symbol(v, env, chan_idx, idx0 + (uint64_t)tsym, d.x, d.y, phi);
			t = tsym + 1;
		} else {
			const float2 d = VDL2_LDG(dec + (ptrdiff_t)t * (ptrdiff_t)stride);
			const float phi = VDL2_LDG(phase + (ptrdiff_t)t * (ptrdiff_t)stride);
			const float mgt = VDL2_LDG(mag + (ptrdiff_t)t * (ptrdiff_t)stride);
			vdl2_demod_step_pm(v, ring, rs, env, chan_idx, idx0 + (uint64_t)t, d.x, d.y, phi, mgt, false, 0.f, 0.f);
			t++;
		}
	}
}

/* The blocked walk with the sync attempts fed from the phase RING instead of the phase plane.
 *
 * With ring_pos = P at block entry (the slot of the sample before the block), local sample t is written to slot
 * P+1+t, and the attempt on local sample e reads, in the reference, the slots of samples e-150+10i (i = 0..15) after
 * samples 0..e were written.  Those writes only replace samples <= e-160, which the attempt does not read, so every
 * sample < 0 can be read from the ring BEFORE the block is applied, and samples >= 0 (i = 15 always, i = 14 for
 * e >= 10) are the block's own inputs pw[].  This holds for any ring content, so the 150 samples after a reset take
 * the same path; per block the walk then needs 12 phase + 4 magnitude values from global memory instead of 80, and
 * they are requested one block ahead (`pf`), so no load latency is exposed.
 * pf carries the next block's inputs: pw[0..11], and mg[] for the attempt offsets predicted from this block's
 * `first` (the sample clock returns to the same value every 12 samples while searching). */
struct vdl2_walk_pref {
	float pw[VDL2_WALK_BLOCK];
	float mg[4];
	int first;
	int valid;
};

/* offset of the first sync attempt in a block entered with this state (0 when the block will not take the fast path) */
VDL2_HD int vdl2_walk_first(const vdl2_chan &v) {
	const bool fast = !(v.state & VDL2_ST_LOCKED) && vdl2_dec_state(v) != VDL2_DEC_IDLE && v.sclk >= 0 && v.sclk < VDL2_SYNC_SKIP;
	return fast ? (VDL2_SYNC_SKIP - 1) - v.sclk : 0;
}

/* STAGED: dec / phase / mag point into a shared-memory staging buffer (plain loads) instead of global memory (read-only path) */
#define VDL2_LD(STAGED, p) ((STAGED) ? *(p) : VDL2_LDG(p))
template<bool STAGED = false>
VDL2_HD void vdl2_walk_tail(vdl2_chan &v, float *ring, int rs, const vdl2_k2_env &env, uint32_t chan_idx, uint64_t idx0,
		const float2 *dec, const float *phase, const float *mag, size_t stride, int resume) {
	int t = resume;
	while(t < VDL2_WALK_BLOCK) {
		if((v.state & VDL2_ST_LOCKED) && vdl2_dec_state(v) != VDL2_DEC_IDLE) {
			const int tsym = t + (VDL2_SPS - 1) - v.sclk;                  /* sample on which ++sclk reaches SPS */
			if(tsym >= VDL2_WALK_BLOCK) { v.sclk += VDL2_WALK_BLOCK - t; break; }
			const float2 d = VDL2_LD(STAGED, dec + (ptrdiff_t)tsym * (ptrdiff_t)stride);
			const float phi = VDL2_LD(STAGED, phase + (ptrdiff_t)tsym * (ptrdiff_t)stride);
			v.sclk = 0;
			vdl2_symbol(v, env, chan_idx, idx0 + (uint64_t)tsym, d.x, d.y, phi);
			t = tsym + 1;
		} else {
			const float2 d = VDL2_LD(STAGED, dec + (ptrdiff_t)t * (ptrdiff_t)stride);
			const float phi = VDL2_LD(STAGED, phase + (ptrdiff_t)t * (ptrdiff_t)stride);
			if(mag) {
				const float mgt = VDL2_LD(STAGED, mag + (ptrdiff_t)t * (ptrdiff_t)stride);
				vdl2_demod_step_pm(v, ring, rs, env, chan_idx, idx0 + (uint64_t)t, d.x, d.y, phi, mgt, false, 0.f, 0.f);
			} else {
				/* no magnitude plane: vdl2_demod_step_pm with the magnitude taken from the sample, and only on the
				 * samples that consume it (every SYNC_SKIP-th while searching) */
				if(vdl2_dec_state(v) == VDL2_DEC_IDLE) vdl2_demod_reset(v);
				vdl2_init_write(v, ring, rs, phi);
				if(++v.sclk >= VDL2_SYNC_SKIP) {
					v.sclk = 0;
					vdl2_init_eval(v, ring, rs, env, chan_idx, idx0 + (uint64_t)t, vdl2_mag_of(d.x, d.y), false, 0.f, 0.f);
				}
			}
			t++;
		}
	}
}

/* The searching path reads and writes the ring at one of two positions per block (before and after the wrap at 160)
 * plus a compile-time offset.  vdl2_ring_at(ring, i) is the position of ring[i], vdl2_ring_ld / vdl2_ring_st access
 * ring[i + k] from it.  On the device the position is the 32-bit shared-memory address of ring[i], hidden from the
 * compiler's value tracking, so that picking one of two positions is one select and the access folds k into its
 * immediate: written as indices, the select is rewritten into a select of indices followed, per access, by the
 * arithmetic both positions share (the lane's column, the scaling, the ring's base).  ring is the lane's column of the
 * shared-memory ring there; on the host the position is the index itself. */
#ifdef __CUDA_ARCH__
typedef uint32_t vdl2_ring_pos;
VDL2_HD vdl2_ring_pos vdl2_ring_at(const float *ring, int i) {
	uint32_t a = (uint32_t)__cvta_generic_to_shared(ring) + 4u * (uint32_t)i;
	asm("" : "+r"(a));
	return a;
}
VDL2_HD float vdl2_ring_ld(const float *, vdl2_ring_pos a, int k) {
	float x;
	asm("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(a + 4u * (uint32_t)k) : "memory");
	return x;
}
VDL2_HD void vdl2_ring_st(float *, vdl2_ring_pos a, int k, float x) {
	asm volatile("st.shared.f32 [%0], %1;" :: "r"(a + 4u * (uint32_t)k), "f"(x) : "memory");
}
#else
typedef int vdl2_ring_pos;
VDL2_HD vdl2_ring_pos vdl2_ring_at(const float *, int i) { return i; }
VDL2_HD float vdl2_ring_ld(const float *ring, vdl2_ring_pos a, int k) { return ring[a + k]; }
VDL2_HD void vdl2_ring_st(float *ring, vdl2_ring_pos a, int k, float x) { ring[a + k] = x; }
#endif

template<bool STAGED = false>
VDL2_HD void vdl2_walk_block_ring(vdl2_chan &v, float *ring, int rs, const vdl2_k2_env &env, uint32_t chan_idx, uint64_t idx0,
		const float2 *dec, const float *phase, const float *mag, size_t stride, vdl2_walk_pref &pf, bool has_next) {
	const bool fast = !(v.state & VDL2_ST_LOCKED) && vdl2_dec_state(v) != VDL2_DEC_IDLE && v.sclk >= 0 && v.sclk < VDL2_SYNC_SKIP;
	const int first = fast ? (VDL2_SYNC_SKIP - 1) - v.sclk : 0;          /* offset of the first attempt in the block */
	float pw[VDL2_WALK_BLOCK], mg[4];
	const bool have_pw = pf.valid != 0, have_mg = pf.valid != 0 && pf.first == first;
#pragma unroll
	for(int t = 0; t < VDL2_WALK_BLOCK; t++) pw[t] = pf.pw[t];
#pragma unroll
	for(int j = 0; j < 4; j++) mg[j] = pf.mg[j];
	if(VDL2_UNLIKELY(!have_pw && fast)) {
#pragma unroll
		for(int t = 0; t < VDL2_WALK_BLOCK; t++) pw[t] = VDL2_LD(STAGED, phase + (ptrdiff_t)t * (ptrdiff_t)stride);
	}
	if(VDL2_UNLIKELY(!have_mg && fast)) {
#pragma unroll
		for(int j = 0; j < 4; j++) {
			const ptrdiff_t o = (ptrdiff_t)(first + VDL2_SYNC_SKIP * j) * (ptrdiff_t)stride;
			if(mag) mg[j] = VDL2_LD(STAGED, mag + o);
			else { const float2 d = VDL2_LD(STAGED, dec + o); mg[j] = vdl2_mag_of(d.x, d.y); }
		}
	}
	/* request the next block's inputs now; they arrive while this block is evaluated */
	if(has_next) {
#pragma unroll
		for(int t = 0; t < VDL2_WALK_BLOCK; t++) pf.pw[t] = VDL2_LD(STAGED, phase + (ptrdiff_t)(VDL2_WALK_BLOCK + t) * (ptrdiff_t)stride);
#pragma unroll
		for(int j = 0; j < 4; j++) pf.mg[j] = VDL2_LD(STAGED, mag + (ptrdiff_t)(VDL2_WALK_BLOCK + first + VDL2_SYNC_SKIP * j) * (ptrdiff_t)stride);
		pf.first = first;
		pf.valid = 1;
	} else {
		pf.valid = 0;
	}
	int resume = 0;
	if(fast) {
		float ph[4][VDL2_PREAMBLE_SYMS], p0[4], sl[4];
		/* slot of sample e-150 with e = first + 3j: P + 1 + e - 150 == P + e + 11 (mod 160).  With b = that slot for j = 0,
		 * read i of attempt j is slot b + o, o = 3j + 10i <= 149, and b + o < 320: the ring wraps at most once over all 60
		 * reads, so each is one of two positions (before / after the wrap) plus a compile-time offset, picked by one
		 * compare against an immediate. */
		int b = v.ring_pos + first + 11;
		if(b >= VDL2_SYNC_BUFLEN) b -= VDL2_SYNC_BUFLEN;
		const vdl2_ring_pos rd_lo = vdl2_ring_at(ring, b * rs), rd_hi = vdl2_ring_at(ring, (b - VDL2_SYNC_BUFLEN) * rs);
#pragma unroll
		for(int j = 0; j < 4; j++) {
#pragma unroll
			for(int i = 0; i < VDL2_PREAMBLE_SYMS - 1; i++) {
				const int o = VDL2_SYNC_SKIP * j + VDL2_SPS * i;
				ph[j][i] = vdl2_ring_ld(ring, b < VDL2_SYNC_BUFLEN - o ? rd_lo : rd_hi, o * rs);
			}
			/* i = 15 is the attempt's own sample, one of the block's inputs */
			ph[j][15] = (first == 0) ? pw[VDL2_SYNC_SKIP * j] : ((first == 1) ? pw[VDL2_SYNC_SKIP * j + 1] : pw[VDL2_SYNC_SKIP * j + 2]);
		}
		/* i = 14 of the last attempt is sample first - 1: still the ring for first == 0, else pw[0] / pw[1] */
		if(first == 1) ph[3][14] = pw[0];
		else if(first == 2) ph[3][14] = pw[1];
		vdl2_metric_core_n<4, true>(ph, env.pr_phase, env.lr_X, env.lr_denom, env.unwrap_lut, p0, sl);
		const int sclk_entry = v.sclk;
		/* The twelve ring slots of the block follow from the entry position (vdl2_init_write advances by one with a
		 * wrap at 160): slot of sample t = entry + 1 + t, wrapped at most once over the block (entry + 1 + 11 < 320), so
		 * each store is one of two positions plus a compile-time offset, like the reads above; the saturating run
		 * counter is advanced once, by the number of samples written. */
		const int rp_entry = v.ring_pos + 1;
		const vdl2_ring_pos wr_lo = vdl2_ring_at(ring, rp_entry * rs), wr_hi = vdl2_ring_at(ring, (rp_entry - VDL2_SYNC_BUFLEN) * rs);
#define VDL2_RING_SLOT(t) ((rp_entry + (t)) >= VDL2_SYNC_BUFLEN ? (rp_entry + (t)) - VDL2_SYNC_BUFLEN : (rp_entry + (t)))
#define VDL2_RING_PUT(t) vdl2_ring_st(ring, rp_entry < VDL2_SYNC_BUFLEN - (t) ? wr_lo : wr_hi, (t) * rs, pw[t])
		/* which of a group's three samples precede its attempt (u <= first), decided once for the block */
		static_assert(VDL2_SYNC_SKIP == 3, "a group is three samples");
		const bool pre1 = first >= 1, pre2 = first >= 2;
		bool go = true;
#pragma unroll
		for(int g = 0; g < 4; g++) {
			if(go) {
				VDL2_RING_PUT(VDL2_SYNC_SKIP * g);
				if(pre1) VDL2_RING_PUT(VDL2_SYNC_SKIP * g + 1);
				if(pre2) VDL2_RING_PUT(VDL2_SYNC_SKIP * g + 2);
				v.ring_pos = VDL2_RING_SLOT(VDL2_SYNC_SKIP * g + first);
				v.sclk = 0;
				vdl2_init_eval(v, ring, rs, env, chan_idx, idx0 + (uint64_t)(VDL2_SYNC_SKIP * g + first), mg[g], true, p0[g], sl[g]);
				if(VDL2_UNLIKELY((v.state & VDL2_ST_LOCKED) || v.sclk != 0)) {
					go = false;                      /* locked, or vetoed by max_ppm: the per-sample path takes over */
					resume = VDL2_SYNC_SKIP * g + first + 1;
				} else {
					if(!pre1) VDL2_RING_PUT(VDL2_SYNC_SKIP * g + 1);
					if(!pre2) VDL2_RING_PUT(VDL2_SYNC_SKIP * g + 2);
					v.ring_pos = VDL2_RING_SLOT(VDL2_SYNC_SKIP * g + VDL2_SYNC_SKIP - 1);
					v.sclk = sclk_entry;
				}
			}
		}
#undef VDL2_RING_PUT
#undef VDL2_RING_SLOT
		if(go) resume = VDL2_WALK_BLOCK;
		{
			const uint32_t run = v.pure_run + (uint32_t)resume;       /* `resume` samples were written above */
			v.pure_run = run < VDL2_PURE_SATURATED ? run : VDL2_PURE_SATURATED;
		}
	}
	vdl2_walk_tail<STAGED>(v, ring, rs, env, chan_idx, idx0, dec, phase, mag, stride, resume);
}

/* Data symbols sliced after the walk (the default walk, k2_sync_slice<128, true, 4> and k2_sync_slice_ragged).
 *
 * Once the header has fixed a burst's length, its data symbols depend on nothing else the walk does: symbol k reads its
 * own sample and phase and symbol k-1's phase from the planes, `dphi` and the sample clock; only frame_pwr, the bit
 * accumulator and the pool words chain from one symbol to the next, and while locked no ring slot, mag_lp or nfcnt changes.
 * With the 32 lanes of a warp on 32 different signals almost every block has a lane inside a burst, and slicing its
 * symbols there kept the other 31 idle behind a serial FP64 chain per symbol.  So a lane in DEC_DATA skips its blocks
 * (only the sample clock is implied: the burst's last symbol falls at a known sample), and the symbols are sliced after
 * the block loop, for all lanes of the warp together, by the same vdl2_symbol operations in the same order:
 *   - a burst that ends inside the launch, followed by at least one more sample, is queued: its state before the first
 *     pending symbol is kept (`q`, one burst per lane); the lane takes what the last symbol leaves behind that the next
 *     sample's demod_reset does not clear (prev_phi, burst_seq, slot, IDLE, sclk) and walks on.  With the queue taken, the
 *     burst is sliced at once instead.  A burst without a pool slot (slot < 0) writes nothing: it needs no queue.
 *   - a burst still open at the launch's end (its last symbol on the launch's last sample or later) is sliced up to its
 *     last symbol in the launch, on the lane's own state.
 * Every field of the channel, its ring and the pool words are at the end of a launch what the inline walk leaves; only
 * the order of ready-list entries within a launch differs, and K3 decodes the list in any order. */
struct vdl2_defer {
	int32_t at;          /* launch-local sample of the next unsliced symbol of the burst the lane is in; < 0: none */
	int32_t last;        /* launch-local sample of that burst's last symbol */
	int32_t q_at;        /* queued burst: sample of its first unsliced symbol; < 0: the queue is empty */
	vdl2_chan q;         /* the queued burst's state before that symbol */
};

VDL2_HD void vdl2_defer_init(vdl2_defer &d) { d.at = -1; d.last = -1; d.q_at = -1; }

/* sample of the last symbol of the burst whose next symbol falls at sample `at` */
VDL2_HD int vdl2_burst_last(const vdl2_chan &v, int at) {
	return at + VDL2_SPS * ((int)((v.need_bits - v.nbits + 2u) / 3u) - 1);
}

/* at launch-local sample m, before it is walked: a lane that is in a burst's data part starts skipping */
VDL2_HD void vdl2_defer_enter(vdl2_defer &d, const vdl2_chan &v, int m) {
	if(d.at < 0 && (v.state & VDL2_ST_LOCKED) && vdl2_dec_state(v) == VDL2_DEC_DATA) {
		d.at = m + (VDL2_SPS - 1) - v.sclk;                    /* the sample on which ++sclk reaches SPS */
		d.last = vdl2_burst_last(v, d.at);
	}
}

/* slice the symbols at samples at, at + SPS, ... < end of a channel in DEC_DATA (vdl2_symbol; a data symbol emits no event);
 * returns the sample of the next one.  dec / phase: the lane's launch-local sample 0, consecutive samples `stride` apart */
VDL2_HD int vdl2_slice_run(vdl2_chan &w, const vdl2_k2_env &env, uint32_t chan_idx, const float2 *dec, const float *phase,
		size_t stride, int at, int end) {
	for(; at < end; at += VDL2_SPS) {
		const float2 d = VDL2_LDG(dec + (ptrdiff_t)at * (ptrdiff_t)stride);
		const float phi = VDL2_LDG(phase + (ptrdiff_t)at * (ptrdiff_t)stride);
		w.sclk = 0;
		vdl2_symbol_bits(w, env, d.x, d.y, phi);
		if(w.nbits >= w.need_bits) vdl2_burst_complete(w, env, chan_idx);
	}
	return at;
}

/* the lane's burst ends on sample d.last and the walk goes on at d.last + 1; last_phi = that sample's phase */
VDL2_HD void vdl2_defer_burst_end(vdl2_defer &d, vdl2_chan &v, const vdl2_k2_env &env, uint32_t chan_idx,
		const float2 *dec, const float *phase, size_t stride, float last_phi) {
	if(v.slot >= 0 && d.q_at >= 0) {
		vdl2_slice_run(v, env, chan_idx, dec, phase, stride, d.at, d.last + 1);      /* queue taken: slice it now */
	} else {
		if(v.slot >= 0) { d.q = v; d.q_at = d.at; v.slot = -1; }
		/* the rest of what the last symbol leaves (vdl2_burst_complete) is cleared by the next sample's demod_reset */
		v.prev_phi = last_phi;
		v.sclk = 0;
		v.burst_seq++;
		vdl2_set_dec_state(v, VDL2_DEC_IDLE);
	}
	d.at = -1;
}

/* after the walk of a launch of n_dec samples: the queued burst, then the one still open */
VDL2_HD void vdl2_defer_finish(vdl2_defer &d, vdl2_chan &v, const vdl2_k2_env &env, uint32_t chan_idx,
		const float2 *dec, const float *phase, size_t stride, int n_dec) {
	if(d.q_at >= 0) vdl2_slice_run(d.q, env, chan_idx, dec, phase, stride, d.q_at, vdl2_burst_last(d.q, d.q_at) + 1);
	if(d.at >= 0) {
		const int next = vdl2_slice_run(v, env, chan_idx, dec, phase, stride, d.at, d.last < n_dec ? d.last + 1 : n_dec);
		v.sclk = (VDL2_SPS - 1) + n_dec - next;               /* samples since the last symbol, as ++sclk would count them */
	}
	vdl2_defer_init(d);
}

/* the default walk's block at launch-local sample m with the lane deferring: false when the block is not taken here.  The
 * lane skips the block while its burst goes on past it or to the launch's end; when the burst ends in the block, the rest
 * of the block is walked per sample.  bdec / bphase: the block's samples, `bs` apart (STAGED: shared memory) */
template<bool STAGED>
VDL2_HD bool vdl2_defer_block(vdl2_defer &d, vdl2_chan &v, float *ring, int rs, const vdl2_k2_env &env, uint32_t chan_idx,
		uint64_t idx0, int m, int n_dec, const float2 *bdec, const float *bphase, size_t bs,
		const float2 *dec, const float *phase, size_t stride) {
	vdl2_defer_enter(d, v, m);
	if(d.at < 0) return false;
	const int t = d.last - m;
	if(t >= VDL2_WALK_BLOCK || d.last + 1 >= n_dec) return true;
	vdl2_defer_burst_end(d, v, env, chan_idx, dec, phase, stride, VDL2_LD(STAGED, bphase + (ptrdiff_t)t * (ptrdiff_t)bs));
	vdl2_walk_tail<STAGED>(v, ring, rs, env, chan_idx, idx0, bdec, bphase, nullptr, bs, t + 1);
	return true;
}

/* the same for one sample of the per-sample tail: returns the next sample to walk (n_dec: the walk is done) or -1 when
 * sample m is not taken here */
VDL2_HD int vdl2_defer_sample(vdl2_defer &d, vdl2_chan &v, const vdl2_k2_env &env, uint32_t chan_idx, int m, int n_dec,
		const float2 *dec, const float *phase, size_t stride) {
	vdl2_defer_enter(d, v, m);
	if(d.at < 0) return -1;
	if(d.last + 1 >= n_dec) return n_dec;
	vdl2_defer_burst_end(d, v, env, chan_idx, dec, phase, stride, VDL2_LDG(phase + (ptrdiff_t)d.last * (ptrdiff_t)stride));
	return d.last + 1;
}

/* same, computing phase and magnitude in place (host simulation, unit tests) */
VDL2_HD void vdl2_demod_step(vdl2_chan &v, float *ring, int rs, const vdl2_k2_env &env,
		uint32_t chan_idx, uint64_t dec_index, float re, float im) {
	vdl2_demod_step_pm(v, ring, rs, env, chan_idx, dec_index, re, im, vdl2_phase_of(re, im), vdl2_mag_of(re, im), false, 0.f, 0.f);
}

/* ------------------------------------------------------------------------------------------------
 * K3: data part of decode_vdl2_burst        src/decode.c:259-380
 * ---------------------------------------------------------------------------------------------- */
struct vdl2_burst_work {
	uint32_t datalen_bits, datalen_octets, num_blocks, last_len, last_fec, fec_octets;
	int32_t status;
	int32_t fec_corr;
	uint32_t n_frames, frame_bytes;
	int32_t rs_ret[VDL2_MAX_BLOCKS + 3];
	uint8_t tab[VDL2_MAX_BLOCKS][256];       /* RS blocks, row = block, 255 used */
	uint8_t frames[2064];
	uint16_t flen[VDL2_MAX_FRAMES];
	uint16_t fcrc[VDL2_MAX_FRAMES];
};

VDL2_HD uint8_t vdl2_gf_mul(const uint8_t *gexp, const uint8_t *glog, uint8_t a, uint8_t b) {
	return (a && b) ? gexp[(int)glog[a] + (int)glog[b]] : (uint8_t)0;
}
VDL2_HD uint8_t vdl2_gf_alpha(const uint8_t *gexp, int e) { return gexp[e % 255]; }    /* e >= 0 */

/* 8 burst bits starting at bit `pos`, first bit in bit 7, descrambled */
VDL2_HD uint32_t vdl2_take8(const uint32_t *words, const uint32_t *lfsr, uint32_t pos) {
	uint32_t w = pos >> 5, sh = pos & 31u;
	uint64_t two = ((uint64_t)(words[w] ^ lfsr[w]) << 32) | (uint64_t)(words[w + 1] ^ lfsr[w + 1]);
	return (uint32_t)(two >> (56u - sh)) & 0xFFu;
}
VDL2_HD uint8_t vdl2_brev8(uint32_t b) {
	b = ((b & 0xF0u) >> 4) | ((b & 0x0Fu) << 4);
	b = ((b & 0xCCu) >> 2) | ((b & 0x33u) << 2);
	b = ((b & 0xAAu) >> 1) | ((b & 0x55u) << 1);
	return (uint8_t)b;
}

/* geometry: src/decode.c:233-256.  Returns status. */
VDL2_HD int vdl2_burst_geometry(vdl2_burst_work &w, uint32_t datalen_bits, uint32_t nbits) {
	w.datalen_bits = datalen_bits;
	w.datalen_octets = datalen_bits / 8 + ((datalen_bits % 8) != 0);
	w.num_blocks = w.datalen_octets / VDL2_RS_K;
	w.fec_octets = w.num_blocks * (VDL2_RS_N - VDL2_RS_K);
	w.last_len = w.datalen_octets % VDL2_RS_K;
	if(w.last_len != 0) w.num_blocks++;
	w.last_fec = (uint32_t)vdl2_fec_octets_for(w.last_len);
	w.fec_octets += w.last_fec;
	if(w.last_len == 0) { w.last_len = VDL2_RS_K; w.last_fec = VDL2_RS_N - VDL2_RS_K; }
	w.status = VDL2_BURST_OK;
	w.fec_corr = 0;
	w.n_frames = 0;
	w.frame_bytes = 0;
	for(int r = 0; r < VDL2_MAX_BLOCKS + 3; r++) w.rs_ret[r] = -128;
	if(w.fec_octets == 0) return w.status = VDL2_ERR_NO_FEC;
	if(w.num_blocks > VDL2_MAX_BLOCKS) return w.status = VDL2_ERR_TOO_LONG;
	if(nbits < VDL2_HEADER_LEN + 8 * w.datalen_octets) return w.status = VDL2_ERR_DATA_TRUNCATED;
	if(nbits < VDL2_HEADER_LEN + 8 * (w.datalen_octets + w.fec_octets)) return w.status = VDL2_ERR_FEC_TRUNCATED;
	return VDL2_BURST_OK;
}

/* descramble (src/bitstream.c:94-107), octets LSB first (src/bitstream.c:70-81) and column-wise
 * de-interleave (src/decode.c:135-163,282-297); work item t of the data part / FEC part is independent,
 * so threads tid, tid+nthr, ... each place their own octets.  Rows must have been zeroed. */
VDL2_HD void vdl2_burst_unpack(vdl2_burst_work &w, const uint32_t *words, const uint32_t *lfsr, uint32_t tid, uint32_t nthr) {
	const uint32_t nb = w.num_blocks;
	const uint32_t full = w.last_len * nb;            /* transmit positions that cover every row */
	for(uint32_t t = tid; t < w.datalen_octets; t += nthr) {
		uint32_t row, col;
		if(t < full) { col = t / nb; row = t % nb; }
		else { uint32_t u = t - full; col = w.last_len + u / (nb - 1); row = u % (nb - 1); }
		w.tab[row][col] = vdl2_brev8(vdl2_take8(words, lfsr, VDL2_HEADER_LEN + 8 * t));
	}
	const uint32_t last_fec = (w.last_len == VDL2_RS_K) ? (uint32_t)(VDL2_RS_N - VDL2_RS_K) : w.last_fec;
	const uint32_t fec_rows = nb - (last_fec == 0 ? 1u : 0u);
	const uint32_t ffull = last_fec * fec_rows;       /* positions covering every FEC row (0 if last row has none left) */
	for(uint32_t t = tid; t < w.fec_octets; t += nthr) {
		uint32_t row, col;
		if(fec_rows == nb && t >= ffull) { uint32_t u = t - ffull; col = last_fec + u / (nb - 1); row = u % (nb - 1); }
		else { col = t / fec_rows; row = t % fec_rows; }
		w.tab[row][VDL2_RS_K + col] = vdl2_brev8(vdl2_take8(words, lfsr, VDL2_HEADER_LEN + 8 * (w.datalen_octets + t)));
	}
}

/* RS(255,249) errors-and-erasures decoder, one block per caller.  src/rs.c:32-49 ->
 * src/libfec/decode_rs.h:71-298 (Karn): syndromes by Horner, erasure-seeded Berlekamp-Massey, Chien search
 * with early exit, failure iff deg(lambda) != number of roots, Forney.  Polynomial (not log) form. */
/* rootmul[i][x] = x * alpha^(120+i): the six syndrome recurrences of decode_rs.h:82-93 become one table look-up per
 * symbol and root, and run interleaved (six independent Horner chains) */
VDL2_HD void vdl2_rs_build_rootmul(uint8_t *rootmul, const uint8_t *gexp, const uint8_t *glog, uint32_t tid, uint32_t nthr) {
	for(uint32_t k = tid; k < 6u * 256u; k += nthr) {
		const uint32_t i = k >> 8, x = k & 255u;
		rootmul[k] = x ? gexp[(uint32_t)glog[x] + 120u + i] : (uint8_t)0;
	}
}

/* The decoder in three steps so that a warp can share the two long loops (syndromes over 255 symbols, Chien search
 * over 255 positions) while the short algebra in between stays with one lane:
 *   vdl2_rs_syndromes          S[0..5], serial Horner                          decode_rs.h:82-93
 *   vdl2_rs_syndrome_partial   the same sums, lane l of 32 covering symbols 8l..8l+7 (XOR of the 32 results = S)
 *   vdl2_rs_locator            erasure-seeded Berlekamp-Massey -> lambda, deg  decode_rs.h:112-213
 *   vdl2_rs_chien_serial       roots in increasing position order              decode_rs.h:216-239
 *   vdl2_rs_chien_lane         lane l of 32 tests positions l+1, l+33, ...     (same set, same order once merged)
 *   vdl2_rs_forney             omega, error values, correction                 decode_rs.h:240-291
 * vdl2_rs_verify chains the serial forms; K3 uses the lane forms (vdl2_kernels.cu) and must return the same. */
enum { VDL2_RS_NR = VDL2_RS_N - VDL2_RS_K, VDL2_RS_FCR = 120 };

VDL2_HD int vdl2_rs_syndromes(const uint8_t *data, const uint8_t *rootmul, uint8_t *S) {
	uint32_t s0 = data[0], s1 = s0, s2 = s0, s3 = s0, s4 = s0, s5 = s0;
	for(int j = 1; j < VDL2_RS_N; j++) {
		const uint32_t d = data[j];
		s0 = rootmul[s0] ^ d;
		s1 = rootmul[256 + s1] ^ d;
		s2 = rootmul[512 + s2] ^ d;
		s3 = rootmul[768 + s3] ^ d;
		s4 = rootmul[1024 + s4] ^ d;
		s5 = rootmul[1280 + s5] ^ d;
	}
	S[0] = (uint8_t)s0; S[1] = (uint8_t)s1; S[2] = (uint8_t)s2; S[3] = (uint8_t)s3; S[4] = (uint8_t)s4; S[5] = (uint8_t)s5;
	return (int)(s0 | s1 | s2 | s3 | s4 | s5);
}

/* lane's share of the six syndromes, packed one per byte (S[i] in bits 8i..8i+7): Horner over its own symbols
 * (8 lane .. 8 lane + 7, the last lane has 7), then moved to the weight of its segment:
 * S_i = sum_j d_j a_i^(254-j), a_i = alpha^(120+i), so the segment ending at symbol e is multiplied by a_i^(254-e). */
VDL2_HD uint64_t vdl2_rs_syndrome_partial(const uint8_t *data, uint32_t lane, const uint8_t *gexp, const uint8_t *glog, const uint8_t *rootmul) {
	const uint32_t first = 8u * lane, last = (first + 7u < (uint32_t)VDL2_RS_N - 1u) ? first + 7u : (uint32_t)VDL2_RS_N - 1u;
	uint32_t t[6] = { 0, 0, 0, 0, 0, 0 };
	for(uint32_t j = first; j <= last; j++) {
		const uint32_t d = data[j];
#pragma unroll
		for(int i = 0; i < 6; i++) t[i] = rootmul[256 * i + t[i]] ^ d;
	}
	const uint32_t e = (uint32_t)VDL2_RS_N - 1u - last;
	uint64_t out = 0;
#pragma unroll
	for(int i = 0; i < 6; i++) {
		const uint32_t sh = ((uint32_t)(VDL2_RS_FCR + i) * e) % 255u;
		const uint32_t v = t[i] ? gexp[(uint32_t)glog[t[i]] + sh] : 0u;
		out |= (uint64_t)v << (8 * i);
	}
	return out;
}

/* erasure locator + Berlekamp-Massey; returns deg(lambda) */
VDL2_HD int vdl2_rs_locator(const uint8_t *S, int fec_octets, const uint8_t *gexp, const uint8_t *glog, uint8_t *lambda) {
	enum { NR = VDL2_RS_NR };
	const int no_eras = NR - fec_octets;
	for(int i = 0; i <= NR; i++) lambda[i] = 0;
	lambda[0] = 1;
	if(no_eras > 0) {
		/* erasures are the untransmitted parity octets RS_K+fec .. 254 (src/rs.c:40-43) */
		lambda[1] = vdl2_gf_alpha(gexp, 254 - (VDL2_RS_K + fec_octets));
		for(int i = 1; i < no_eras; i++) {
			uint8_t x = vdl2_gf_alpha(gexp, 254 - (VDL2_RS_K + fec_octets + i));
			for(int j = i + 1; j > 0; j--)
				lambda[j] ^= vdl2_gf_mul(gexp, glog, x, lambda[j - 1]);
		}
	}
	uint8_t B[NR + 1];
	for(int i = 0; i <= NR; i++) B[i] = lambda[i];
	int el = no_eras;
	for(int r = no_eras + 1; r <= NR; r++) {
		uint8_t discr = 0;
		for(int i = 0; i < r; i++) discr ^= vdl2_gf_mul(gexp, glog, lambda[i], S[r - i - 1]);
		if(discr == 0) {
			for(int i = NR; i > 0; i--) B[i] = B[i - 1];
			B[0] = 0;
		} else {
			uint8_t T[NR + 1];
			T[0] = lambda[0];
			for(int i = 0; i < NR; i++) T[i + 1] = lambda[i + 1] ^ vdl2_gf_mul(gexp, glog, discr, B[i]);
			if(2 * el <= r + no_eras - 1) {
				el = r + no_eras - el;
				uint8_t inv = gexp[255 - glog[discr]];
				for(int i = 0; i <= NR; i++) B[i] = vdl2_gf_mul(gexp, glog, lambda[i], inv);
			} else {
				for(int i = NR; i > 0; i--) B[i] = B[i - 1];
				B[0] = 0;
			}
			for(int i = 0; i <= NR; i++) lambda[i] = T[i];
		}
	}
	int deg = 0;
	for(int i = 0; i <= NR; i++) if(lambda[i]) deg = i;
	return deg;
}

/* Chien search, decode_rs.h:216-239: reg[j] = log(lambda_j) + i*j mod 255, advanced by j per step; stops at deg roots */
VDL2_HD int vdl2_rs_chien_serial(const uint8_t *lambda, int deg, const uint8_t *gexp, const uint8_t *glog, int *root) {
	enum { NR = VDL2_RS_NR };
	int reg[NR + 1], count = 0;
	for(int j = 1; j <= NR; j++) reg[j] = lambda[j] ? (int)glog[lambda[j]] : -1;
	for(int i = 1; i <= 255; i++) {
		uint8_t q = 1;
		for(int j = deg; j > 0; j--) {
			if(reg[j] >= 0) {
				reg[j] += j;
				if(reg[j] >= 255) reg[j] -= 255;
				q ^= gexp[reg[j]];
			}
		}
		if(q != 0) continue;
		root[count] = i;
		if(++count == deg) break;
	}
	return count;
}

/* the same test for the positions i = lane + 1 + 32 k (k = 0..7, i <= 255): bit k of the result = "i is a root".  A
 * polynomial of degree deg has at most deg roots, so the serial search's early exit never hides one. */
VDL2_HD uint32_t vdl2_rs_chien_lane(const uint8_t *lambda, int deg, uint32_t lane, const uint8_t *gexp, const uint8_t *glog) {
	enum { NR = VDL2_RS_NR };
	uint32_t mask = 0;
	for(uint32_t k = 0; k < 8; k++) {
		const uint32_t i = lane + 1u + 32u * k;
		if(i > 255u) break;
		uint32_t q = 1;
		for(int j = 1; j <= deg && j <= NR; j++)
			if(lambda[j]) q ^= gexp[((uint32_t)glog[lambda[j]] + i * (uint32_t)j) % 255u];
		if(q == 0) mask |= 1u << k;
	}
	return mask;
}

/* omega, error values (Forney) and correction for the `count` roots found (decode_rs.h:240-291); returns count */
VDL2_HD int vdl2_rs_forney(uint8_t *data, const uint8_t *S, const uint8_t *lambda, int deg, const int *root, int count,
		const uint8_t *gexp, const uint8_t *glog) {
	enum { NR = VDL2_RS_NR, FCR = VDL2_RS_FCR };
	const int deg_omega = deg - 1;
	uint8_t omega[NR + 1] = { 0, 0, 0, 0, 0, 0, 0 };
	for(int i = 0; i <= deg_omega; i++) {
		uint8_t acc = 0;
		for(int j = i; j >= 0; j--) acc ^= vdl2_gf_mul(gexp, glog, S[i - j], lambda[j]);
		omega[i] = acc;
	}
	for(int j = count - 1; j >= 0; j--) {
		uint8_t num1 = 0;
		for(int i = deg_omega; i >= 0; i--)
			if(omega[i]) num1 ^= gexp[(glog[omega[i]] + i * root[j]) % 255];
		uint8_t num2 = gexp[(root[j] * (FCR - 1) + 255) % 255];
		uint8_t den = 0;
		int top = (deg < NR - 1 ? deg : NR - 1) & ~1;
		for(int i = top; i >= 0; i -= 2)
			if(lambda[i + 1]) den ^= gexp[(glog[lambda[i + 1]] + i * root[j]) % 255];
		if(num1 != 0) {
			/* decode_rs.h:289 uses log(0) = 255, so a zero denominator divides by alpha^0 */
			int e = (int)glog[num1] + (int)glog[num2] + 255 - (den ? (int)glog[den] : 255);
			data[root[j] - 1] ^= gexp[e % 255];          /* loc = root - 1 (prim = 1) */
		}
	}
	return count;
}

VDL2_HD int vdl2_rs_verify(uint8_t *data, int fec_octets, const uint8_t *gexp, const uint8_t *glog, const uint8_t *rootmul) {
	enum { NR = VDL2_RS_NR };
	if(fec_octets == 0) return 0;
	uint8_t S[NR], lambda[NR + 1];
	if(!vdl2_rs_syndromes(data, rootmul, S)) return 0;
	const int deg = vdl2_rs_locator(S, fec_octets, gexp, glog, lambda);
	int root[NR + 1];
	const int count = vdl2_rs_chien_serial(lambda, deg, gexp, glog, root);
	if(deg != count) return -1;
	return vdl2_rs_forney(data, S, lambda, deg, root, count, gexp, glog);
}

/* Octet-at-a-time table for the unstuffer: entry [ones][octet] (ones = 0..6, the run of one-bits before the octet)
 * says whether the eight bits of the octet can be taken as they are - no stuffed zero to delete, no flag, no abort -
 * and what the run of ones is afterwards: bit 7 = plain, bits 0..2 = run length after the octet.  Built by stepping
 * the bit rules of vdl2_burst_unstuff itself. */
#define VDL2_UNSTUFF_TABLE_BYTES (7 * 256)
VDL2_HD void vdl2_unstuff_build_table(uint8_t *table, uint32_t tid, uint32_t nthr) {
	for(uint32_t k = tid; k < VDL2_UNSTUFF_TABLE_BYTES; k += nthr) {
		int ones = (int)(k >> 8), plain = 1;
		const uint32_t b = k & 255u;
		for(int i = 0; i < 8 && plain; i++) {
			const uint32_t bit = (b >> i) & 1u;
			if(bit == 0) { if(ones >= 5) plain = 0; else ones = 0; }      /* stuffed zero (5) or closing flag (6) */
			else if(++ones > 6) plain = 0;                                /* seven ones */
		}
		table[k] = (uint8_t)(plain ? (0x80 | ones) : 0);
	}
}

/* serialise corrected octets, cut to datalen bits, split on HDLC flags with zero-bit deletion:
 * src/decode.c:325-370 + src/bitstream.c:109-150.  Single caller.  Returns status; frames found before a
 * late error stay (the reference has already pushed them).
 * `utab` (vdl2_unstuff_build_table, or NULL) lets whole input octets that contain no stuffing, flag or abort event
 * for the current run of ones be appended in one step; an octet the table does not clear goes through the bit rules. */
VDL2_HD int vdl2_burst_unstuff(vdl2_burst_work &w, const uint8_t *utab = nullptr) {
	const uint32_t total_bits = (8u * w.datalen_octets < w.datalen_bits) ? 8u * w.datalen_octets : w.datalen_bits;
	uint32_t pos = 0, row = 0, col = 0, cur = 0;     /* input: corrected octets row by row, LSB first */
	uint32_t out_base = 0;
	for(;;) {
		uint32_t j = 0;          /* bits of the candidate frame, flag prefix included */
		uint32_t acc = 0;        /* output octet being assembled */
		int ones = 0;
		for(;;) {                /* one pass of bitstream_copy_next_frame, restarts folded in */
			if(pos >= total_bits) break;
			if((pos & 7u) == 0) {
				cur = w.tab[row][col];
				if(++col == VDL2_RS_K) { col = 0; row++; }
				if(utab != nullptr && pos + 8u <= total_bits) {
					const uint32_t e = utab[((uint32_t)ones << 8) | cur];
					if(e & 0x80u) {
						/* eight plain bits: exactly one output octet completes (the one holding bit j | 7) */
						const uint32_t both = acc | (cur << (j & 7u));
						const uint32_t ob = out_base + (j >> 3);
						if(ob >= sizeof(w.frames)) return w.status = VDL2_ERR_BITSTREAM;
						w.frames[ob] = (uint8_t)both;
						acc = both >> 8;
						ones = (int)(e & 7u);
						j += 8; pos += 8;
						continue;
					}
				}
			}
			const uint32_t bit = (cur >> (pos & 7u)) & 1u;
			if(bit == 0 && ones == 5) { ones = 0; pos++; continue; }         /* stuffed zero */
			if(bit == 1 && ++ones > 6) return w.status = VDL2_ERR_UNSTUFF;   /* seven ones */
			acc |= bit << (j & 7u);
			if(bit == 0) {
				if(ones == 6) {                                              /* 01111110 */
					if(j == 7) { pos++; j = 0; acc = 0; ones = 0; continue; }    /* opening flag: restart */
					if(j < 7) return w.status = VDL2_ERR_UNSTUFF;
					j -= 7; pos++;
					goto frame_done;
				}
				ones = 0;
			}
			if((j & 7u) == 7u) {
				const uint32_t ob = out_base + (j >> 3);
				if(ob >= sizeof(w.frames)) return w.status = VDL2_ERR_BITSTREAM;
				w.frames[ob] = (uint8_t)acc;
				acc = 0;
			}
			j++; pos++;
		}
	frame_done:
		{
			int more = pos < total_bits;
			if(j % 8 != 0) return w.status = VDL2_ERR_TRUNCATED_OCTETS;
			if(w.n_frames >= VDL2_MAX_FRAMES) return w.status = VDL2_ERR_BITSTREAM;
			w.flen[w.n_frames++] = (uint16_t)(j / 8);
			out_base += j / 8;
			w.frame_bytes = out_base;
			if(!more) break;
		}
	}
	return VDL2_BURST_OK;
}

/* K4: AVLC FCS residue, src/crc.c:21-64 (reflected 0x1021): byte-wise with a 256-entry table built by
 * vdl2_crc16_build_table (the same table the reference carries as a literal), or bitwise without one */
VDL2_HD void vdl2_crc16_build_table(uint16_t *table, uint32_t tid, uint32_t nthr) {
	for(uint32_t b = tid; b < 256u; b += nthr) {
		uint32_t c = b;
		for(int k = 0; k < 8; k++) c = (c >> 1) ^ ((c & 1u) ? 0x8408u : 0u);
		table[b] = (uint16_t)c;
	}
}
VDL2_HD uint16_t vdl2_crc16_tab(const uint8_t *p, uint32_t len, const uint16_t *table) {
	uint32_t crc = 0xFFFFu;
	for(uint32_t n = 0; n < len; n++) crc = (crc >> 8) ^ table[(crc ^ p[n]) & 0xFFu];
	return (uint16_t)crc;
}

VDL2_HD uint16_t vdl2_crc16(const uint8_t *p, uint32_t len) {
	uint32_t crc = 0xFFFFu;
	for(uint32_t n = 0; n < len; n++) {
		crc ^= p[n];
#pragma unroll
		for(int b = 0; b < 8; b++) crc = (crc >> 1) ^ ((crc & 1u) ? 0x8408u : 0u);
	}
	return (uint16_t)crc;
}

/* ------------------------------------------------------------------------------------------------
 * Channel layout: slot -> channel -> receiver, and the tile geometry of the receiver-group K1
 * ---------------------------------------------------------------------------------------------- */
/* slot (index into every per-channel array) -> public channel number and activity: a warp holds `lanes` channels in its
 * first `lanes` lanes (the first full_warps warps) or lanes - 1 (the others); see the slot mapping in vdl2_host.cu */
VDL2_HD bool vdl2_slot_channel(uint32_t slot, uint32_t lanes, uint32_t full_warps, uint32_t n_ch, uint32_t &chan) {
	const uint32_t lane = slot & 31u, w = slot >> 5;
	const uint32_t mine = w < full_warps ? lanes : lanes - 1u;                 /* channels of this warp */
	chan = (w < full_warps ? w * lanes : full_warps * lanes + (w - full_warps) * (lanes - 1u)) + lane;
	return lane < mine && chan < n_ch;
}

/* Multi-receiver context (vdl2gpu_create_receivers): receiver r owns channels [rx_first[r], rx_first[r + 1]), every
 * receiver at least one.  Returns the receiver of a channel (binary search over the n_rx + 1 boundaries). */
VDL2_HD uint32_t vdl2_rx_of_channel(uint32_t chan, const uint32_t *rx_first, uint32_t n_rx) {
	uint32_t lo = 0, hi = n_rx;                   /* rx_first[lo] <= chan < rx_first[hi] */
	while(hi - lo > 1u) {
		const uint32_t mid = (lo + hi) >> 1;
		if(rx_first[mid] <= chan) lo = mid; else hi = mid;
	}
	return lo;
}

#define VDL2_RX_K1_BLOCK 128u                         /* slots per block of the receiver-group K1 */
/* Shared memory of one receiver-group K1 block: with one K2 block (~116 KB) it must fit the 228 KB of an SM, or the
 * K2(c) || K1(c+1) schedule of the pipeline (one block of each per SM) breaks */
#define VDL2_RX_K1_SMEM_BUDGET (110u * 1024u)
#define VDL2_RX_K1_LUT_BYTES (257u * 8u * 16u)         /* the eight NCO table copies */

/* Every 128-slot block covers a contiguous channel range, hence a contiguous receiver range.  Fills slot_rx[n_blocks * 128]
 * (receiver of the slot's channel; an inactive slot gets its block's first receiver) and block_rx[n_blocks][2] = {first
 * receiver, number of receivers G} (G = 0 for a block without channels); returns the largest G. */
VDL2_HD uint32_t vdl2_rx_layout(uint32_t n_blocks, uint32_t lanes, uint32_t full_warps, uint32_t n_ch, const uint32_t *rx_first,
		uint32_t n_rx, uint32_t *slot_rx, uint32_t *block_rx) {
	uint32_t g_max = 0;
	for(uint32_t b = 0; b < n_blocks; b++) {
		uint32_t first = 0xFFFFFFFFu, last = 0;
		for(uint32_t t = 0; t < VDL2_RX_K1_BLOCK; t++) {
			uint32_t chan;
			if(!vdl2_slot_channel(b * VDL2_RX_K1_BLOCK + t, lanes, full_warps, n_ch, chan)) continue;
			const uint32_t r = vdl2_rx_of_channel(chan, rx_first, n_rx);
			slot_rx[b * VDL2_RX_K1_BLOCK + t] = r;
			if(first == 0xFFFFFFFFu) first = r;
			last = r;
		}
		const uint32_t g = first == 0xFFFFFFFFu ? 0u : last - first + 1u;
		if(first == 0xFFFFFFFFu) first = 0;
		for(uint32_t t = 0; t < VDL2_RX_K1_BLOCK; t++) {
			uint32_t chan;
			if(!vdl2_slot_channel(b * VDL2_RX_K1_BLOCK + t, lanes, full_warps, n_ch, chan)) slot_rx[b * VDL2_RX_K1_BLOCK + t] = first;
		}
		block_rx[2 * b] = first;
		block_rx[2 * b + 1] = g;
		if(g > g_max) g_max = g;
	}
	return g_max;
}

/* float2 elements per staged receiver row for a tile of T samples: room for T + 2 (the odd-phase shift and the odd
 * trailing sample), rounded up to 2 mod 16.  Even keeps every row 16-byte aligned for the bulk copy; 2 mod 16 starts row
 * r 4 r banks further on, so up to eight receivers of one warp read different banks. */
VDL2_HD uint32_t vdl2_rx_tile_stride(uint32_t T) { return T + 2u + (16u - T % 16u) % 16u; }

VDL2_HD uint32_t vdl2_rx_k1_smem_bytes(uint32_t G, uint32_t T) {
	return 2u * G * vdl2_rx_tile_stride(T) * 8u + VDL2_RX_K1_LUT_BYTES + 16u;     /* two tile buffers, table, two mbarriers */
}

/* T for blocks of up to G receivers: the most whole decimation groups, an even number of samples (16-byte bulk copies),
 * that keep vdl2_rx_k1_smem_bytes(G, T) within VDL2_RX_K1_SMEM_BUDGET; 0 if not even one fits */
VDL2_HD uint32_t vdl2_rx_tile_samples(uint32_t G, uint32_t oversample) {
	if(G == 0) G = 1;
	const uint32_t avail = VDL2_RX_K1_SMEM_BUDGET - VDL2_RX_K1_LUT_BYTES - 16u;
	const uint32_t r_max = avail / (16u * G);
	if(r_max < 2u + 2u) return 0;
	const uint32_t r = r_max - (r_max - 2u) % 16u;                  /* largest row stride <= r_max that is 2 mod 16 */
	const uint32_t step = (oversample & 1u) ? 2u * oversample : oversample;
	return (r - 2u) / step * step;
}

/* ------------------------------------------------------------------------------------------------
 * Mixed-rate receivers (vdl2gpu_create_mixed_receivers): every receiver has its own oversample factor (10, 13 or 20) and
 * sample format, and a span carries the same number n_dec of decimated samples for each of them
 * ---------------------------------------------------------------------------------------------- */
/* one receiver's input: oversample factor, sample format and the bytes that lie before its buffer in a span, per decimated
 * sample of the span (receiver r's buffer starts n_dec * off_per_dec bytes in) */
typedef struct {
	uint64_t off_per_dec;
	uint32_t oversample, fmt;
} vdl2_rx_input;

/* rate class of an oversample factor (index into the per-class filter taps); 10, 13 and 20 only */
VDL2_HD uint32_t vdl2_rx_class(uint32_t oversample) { return oversample == 10u ? 0u : oversample == 13u ? 1u : 2u; }

/* fills rx[r].off_per_dec = sum over q < r of os_q x bytes per complex sample of q; returns the bytes of one decimated
 * sample of every receiver, i.e. a span of n_dec is n_dec times that long */
VDL2_HD uint64_t vdl2_rx_span_layout(const uint32_t *oversample, const uint32_t *fmt, uint32_t n_rx, vdl2_rx_input *rx) {
	uint64_t off = 0;
	for(uint32_t r = 0; r < n_rx; r++) {
		rx[r].off_per_dec = off;
		rx[r].oversample = oversample[r];
		rx[r].fmt = fmt[r];
		off += (uint64_t)oversample[r] * (fmt[r] == 1u ? 4u : 2u);
	}
	return off;
}

/* byte offset of receiver r's buffer in a span of n_dec decimated samples (64 bits: 65535 cs16 receivers at oversample 20
 * pass 4 GiB within a span of 55 decimated samples) */
VDL2_HD uint64_t vdl2_rx_span_offset(const vdl2_rx_input *rx, uint32_t r, uint32_t n_dec) { return (uint64_t)n_dec * rx[r].off_per_dec; }

/* Decimation groups per tile of the mixed K1 for blocks of up to G receivers whose largest oversample factor is os_max:
 * row r of a tile stages TG x os_r samples into a row of vdl2_rx_tile_stride(TG x os_max) elements.  TG is even, so every
 * row start and every copy size is a multiple of 16 bytes whatever the factors.  The largest even TG that keeps
 * vdl2_rx_k1_smem_bytes within VDL2_RX_K1_SMEM_BUDGET; never below 2: with os_max 20 and 100 or more receivers in one
 * block not even two groups fit, and the block then takes vdl2_rx_k1_smem_bytes(G, 40) > budget (at most
 * VDL2_RX_MIXED_SMEM_MAX) - correct, but its K1 block no longer shares an SM with a K2 block. */
VDL2_HD uint32_t vdl2_rx_mixed_tile_groups(uint32_t G, uint32_t os_max) {
	if(G == 0) G = 1;
	uint32_t tg = 2;
	while(vdl2_rx_k1_smem_bytes(G, (tg + 2u) * os_max) <= VDL2_RX_K1_SMEM_BUDGET) tg += 2u;
	return tg;
}
#define VDL2_RX_MIXED_SMEM_MAX (2u * VDL2_RX_K1_BLOCK * (40u + 10u) * 8u + VDL2_RX_K1_LUT_BYTES + 16u)   /* G = 128, TG = 2, os 20 */

/* ------------------------------------------------------------------------------------------------
 * Ragged spans (VDL2GPU_FLAG_RAGGED on a mixed-receivers context): receiver r brings its own number n_r >= 0 of decimated
 * samples to every span, and the chain walks each receiver's lanes to that count
 * ---------------------------------------------------------------------------------------------- */
/* one receiver's entry of a span's receiver table: where its buffer starts in the span, the decimated samples it brings to
 * this span (n) and brought to the previous one (prev_n), and its position before this span (dec_base: decimated samples
 * accepted so far, the index of its first sample in this span) */
typedef struct {
	uint64_t off;
	uint32_t n, prev_n;
	uint64_t dec_base;
} vdl2_rx_span;

/* The table of one span from the counts n[r]: the buffers lie back to back, receiver 0 first, n[r] x os_r x bytes per
 * complex sample each (64-bit offsets).  pos[r] (decimated samples accepted so far) and prev[r] (the count of the previous
 * span) carry over from span to span: read into the table, then advanced.  Returns the bytes of the span. */
VDL2_HD uint64_t vdl2_rx_span_table(const vdl2_rx_input *rx, uint32_t n_rx, const uint32_t *n, uint64_t *pos, uint32_t *prev,
		vdl2_rx_span *out) {
	uint64_t off = 0;
	for(uint32_t r = 0; r < n_rx; r++) {
		out[r].off = off;
		out[r].n = n[r];
		out[r].prev_n = prev[r];
		out[r].dec_base = pos[r];
		off += (uint64_t)n[r] * rx[r].oversample * (rx[r].fmt == 1u ? 4u : 2u);
		pos[r] += n[r];
		prev[r] = n[r];
	}
	return off;
}

/* What row r of the ragged K1's tile at decimation group g0 stages: the groups receiver r still has in the tile,
 * clamp(n_r - g0, 0, TG), i.e. `samples` = groups x os_r samples; a bulk copy of the even part (`bytes`, 0 = no copy is
 * issued) and, for an odd count (oversample 13), the last sample copied by hand.  g0 is a multiple of the even TG, so
 * every copy starts 16-byte aligned, as in the lock-step kernel. */
typedef struct {
	uint32_t groups, samples, bytes, odd;
} vdl2_rx_tile_row;

VDL2_HD vdl2_rx_tile_row vdl2_rx_ragged_row(uint32_t n_r, uint32_t g0, uint32_t TG, uint32_t os_r) {
	vdl2_rx_tile_row t;
	t.groups = n_r > g0 ? (n_r - g0 < TG ? n_r - g0 : TG) : 0u;
	t.samples = t.groups * os_r;
	t.bytes = (t.samples & ~1u) * 8u;                  /* float2 */
	t.odd = t.samples & 1u;
	return t;
}

/* ------------------------------------------------------------------------------------------------
 * Restarting one receiver of a ragged context (vdl2gpu_restart_receiver): from the start of a span on, its channels
 * decode what a freshly started reference process, tuned to the receiver's (possibly new) centre and frequencies, decodes
 * from the samples the receiver brings from then on.  One rule for create and restart, so the two cannot drift apart.
 * ---------------------------------------------------------------------------------------------- */
/* the NCO step of a channel (src/demod.c:385); a channel on the centre frequency skips the mixer in the reference
 * (src/demod.c:312): with a zero step the table gives cos = 1, sin = 0 and the products are exact, so no branch is needed */
VDL2_HD uint32_t vdl2_nco_dphi(uint32_t centerfreq, uint32_t freq, uint32_t rate) {
	if(centerfreq == freq) return 0u;
	return (uint32_t)(int)F_MUL(F_MUL(F_DIV(F_SUB((float)centerfreq, (float)freq), (float)rate), 256.0f), 65536.0f);
}

/* the K1 state of a freshly started channel in slot ch of the K1 planes: zero delay lines, NCO phase 0, the channel's step
 * (the decimation counter is not per channel: it is 0 at the start of every span of a mixed-receivers context) */
VDL2_HD void vdl2_k1_fresh(uint32_t *st, size_t stride, uint32_t ch, uint32_t dphi) {
	for(int f = 0; f < K1_NFIELDS; f++) st[(size_t)f * stride + ch] = 0u;
	st[(size_t)K1_DPHI * stride + ch] = dphi;
}

/* one channel's K2 state as the K2 planes hold it (field f of slot ch at st[f * stride + ch]) */
VDL2_HD void vdl2_chan_store(const vdl2_chan &v, uint32_t *st, size_t stride, uint32_t ch) {
	union { float f; uint32_t u; } b;
#define VDL2_ST_F(F, X) do { b.f = (X); st[(size_t)(F) * stride + ch] = b.u; } while(0)
	VDL2_ST_F(K2_PREV_PHI, v.prev_phi); VDL2_ST_F(K2_PREV_DPHI, v.prev_dphi); VDL2_ST_F(K2_DPHI, v.dphi);
	VDL2_ST_F(K2_PHERR0, v.pherr0); VDL2_ST_F(K2_PHERR1, v.pherr1); VDL2_ST_F(K2_PHERR2, v.pherr2);
	VDL2_ST_F(K2_PPM, v.ppm_error); VDL2_ST_F(K2_MAG_LP, v.mag_lp); VDL2_ST_F(K2_MAG_NF, v.mag_nf);
	VDL2_ST_F(K2_FRAME_PWR, v.frame_pwr);
#undef VDL2_ST_F
	st[(size_t)K2_RING_POS * stride + ch] = (uint32_t)v.ring_pos; st[(size_t)K2_SCLK * stride + ch] = (uint32_t)v.sclk;
	st[(size_t)K2_NFCNT * stride + ch] = (uint32_t)v.nfcnt; st[(size_t)K2_FRAME_PWR_CNT * stride + ch] = (uint32_t)v.frame_pwr_cnt;
	st[(size_t)K2_STATE * stride + ch] = v.state;
	st[(size_t)K2_ACC_LO * stride + ch] = (uint32_t)v.acc; st[(size_t)K2_ACC_HI * stride + ch] = (uint32_t)(v.acc >> 32);
	st[(size_t)K2_NBITS * stride + ch] = v.nbits; st[(size_t)K2_NEED_BITS * stride + ch] = v.need_bits;
	st[(size_t)K2_DATALEN * stride + ch] = v.datalen; st[(size_t)K2_SYNDROME * stride + ch] = v.syndrome;
	st[(size_t)K2_SLOT * stride + ch] = (uint32_t)v.slot; st[(size_t)K2_BURST_SEQ * stride + ch] = v.burst_seq;
	st[(size_t)K2_SYNC_LO * stride + ch] = (uint32_t)v.sync_dec_index; st[(size_t)K2_SYNC_HI * stride + ch] = (uint32_t)(v.sync_dec_index >> 32);
	st[(size_t)K2_FREQ * stride + ch] = v.freq;
	st[(size_t)K2_CNT_SYNC * stride + ch] = v.cnt_sync; st[(size_t)K2_CNT_HDR_GOOD * stride + ch] = v.cnt_hdr_good;
	st[(size_t)K2_PURE_RUN * stride + ch] = v.pure_run;
}

/* a ready-list entry with this bit set is a burst-pool slot given up by a restart, not a burst: K3 puts it back on the
 * free list and writes no record, counts nothing, emits nothing */
#define VDL2_READY_ABANDONED 0x80000000u

/* Restart of one channel's demodulator: the old process is treated as killed here.  A burst still in progress (header
 * decoded, data being collected) is dropped; the burst-pool slot it holds goes back to the pool through K3 (ready list,
 * VDL2_READY_ABANDONED): other lanes pop the free list concurrently, so pushing onto it from here would race them.
 * Every field is then as vdl2_chan_init leaves it, tuned to `freq`, except the burst sequence number and the two
 * per-channel counters kept in the state: they continue, so that (channel, burst_seq, idx) never repeats and the
 * counters are the sum over the old and the new process.  The caller zeroes the channel's syncbuf ring. */
VDL2_HD void vdl2_chan_restart(vdl2_chan &v, const vdl2_k2_env &env, uint32_t freq) {
	if(v.slot >= 0) {
		const uint32_t k = VDL2_ATOMIC_ADD_U32(&env.ctl->n_ready, 1u);
		env.ready[k] = (uint32_t)v.slot | VDL2_READY_ABANDONED;
	}
	const uint32_t seq = v.burst_seq, cnt_sync = v.cnt_sync, cnt_hdr_good = v.cnt_hdr_good;
	vdl2_chan_init(v, freq);
	v.burst_seq = seq; v.cnt_sync = cnt_sync; v.cnt_hdr_good = cnt_hdr_good;
}

/* one channel slot's entry of a span's restart table: restart != 0 = the channel restarts at the start of the span with K1
 * step dphi (vdl2_nco_dphi) and frequency freq */
typedef struct {
	uint32_t restart, dphi, freq;
} vdl2_rx_restart;

/* ------------------------------------------------------------------------------------------------
 * Receivers joining and leaving a ragged context (vdl2gpu_update_receivers): the new receiver list rx[0..n_rx) names, per
 * entry, the old receiver it continues (from[r] >= 0) or none (from[r] == -1, a new receiver).  A kept receiver repeats its
 * description, so its channel k is old channel old_first[from[r]] + k; each kept channel carries its whole state from
 * its old slot to its new one, and a new receiver's channels start as create starts them.
 * ---------------------------------------------------------------------------------------------- */
/* channel -> slot, the inverse of vdl2_slot_channel */
VDL2_HD uint32_t vdl2_channel_slot(uint32_t ch, uint32_t lanes, uint32_t full_warps) {
	const uint32_t head = full_warps * lanes;
	if(ch < head) return (ch / lanes) * 32u + ch % lanes;
	const uint32_t c = ch - head;
	return (full_warps + c / (lanes - 1u)) * 32u + c % (lanes - 1u);
}

/* the old channel new channel `chan` continues, or -1 (a channel of a new receiver); rx_first[n_rx + 1] are the new
 * receivers' first channels, old_first those of the old list */
VDL2_HD int32_t vdl2_rx_chan_from(uint32_t chan, const uint32_t *rx_first, uint32_t n_rx, const int32_t *from, const uint32_t *old_first) {
	const uint32_t r = vdl2_rx_of_channel(chan, rx_first, n_rx);
	if(from[r] < 0) return -1;
	return (int32_t)(old_first[from[r]] + (chan - rx_first[r]));
}

#define VDL2_MIGRATE_FRESH (-1)                /* the slot's channel belongs to a new receiver */
#define VDL2_MIGRATE_NONE (-2)                 /* the slot holds no channel */

/* The old slot new slot `slot` continues (new layout: lanes, full_warps, n_ch, rx_first; old layout: old_lanes,
 * old_full_warps, old_first), VDL2_MIGRATE_FRESH or VDL2_MIGRATE_NONE.  Each kept channel maps to its own old slot and
 * nothing else maps to an old slot, since from[] names each old receiver at most once. */
VDL2_HD int32_t vdl2_rx_slot_from(uint32_t slot, uint32_t lanes, uint32_t full_warps, uint32_t n_ch, const uint32_t *rx_first,
		uint32_t n_rx, const int32_t *from, uint32_t old_lanes, uint32_t old_full_warps, const uint32_t *old_first) {
	uint32_t chan;
	if(!vdl2_slot_channel(slot, lanes, full_warps, n_ch, chan)) return VDL2_MIGRATE_NONE;
	const int32_t old = vdl2_rx_chan_from(chan, rx_first, n_rx, from, old_first);
	return old < 0 ? VDL2_MIGRATE_FRESH : (int32_t)vdl2_channel_slot((uint32_t)old, old_lanes, old_full_warps);
}

/* entry i of the migration table: slot i of the new planes and channel i of the new counters (the counters are kept by
 * channel, the state by slot) */
typedef struct {
	int32_t slot_from;           /* slot i: vdl2_rx_slot_from */
	uint32_t hist_row;           /* ... kept: its receiver's count in the last span (prev_n), where its last 160 phases start */
	uint32_t dphi, freq;         /* ... fresh: NCO step (vdl2_nco_dphi) and frequency */
	int32_t chan_from;           /* channel i: the old channel whose counters it continues, or -1 (zero counters) */
} vdl2_rx_migrate;

/* ------------------------------------------------------------------------------------------------
 * Pushed input (vdl2gpu_push / vdl2gpu_submit_pushed on a ragged context): every receiver has a byte ring in device memory
 * (mirrored byte for byte in pinned host memory) that its pushes fill at any length and spans drain in whole decimation
 * groups.  Positions are 64-bit stream positions, bytes pushed since the ring was made; a position's place in the ring is
 * position mod cap.  Per receiver: head (bytes pushed), tail (first byte not yet taken into a span or dropped) and freed
 * (every byte before it has been read by the copies and the K0 that needed it, so it may be overwritten).
 * ---------------------------------------------------------------------------------------------- */
/* receiver r's ring: bytes [base, base + cap) of the ring buffer */
typedef struct {
	uint64_t base, cap;
} vdl2_rx_ring;

/* Ring capacity of a receiver of group_bytes (oversample x bytes per complex sample) bytes per decimated sample: one push
 * of max_chunk_bytes, a full span of max_span groups and one group (a remainder that waits for the next push), rounded up
 * to 16 bytes.  A multiple of the sample size (2 or 4) and every span fits, so no sample straddles the end of the ring. */
VDL2_HD uint64_t vdl2_push_ring_cap(uint32_t max_chunk_bytes, uint32_t max_span, uint32_t group_bytes) {
	const uint64_t need = (uint64_t)max_chunk_bytes + ((uint64_t)max_span + 1u) * group_bytes;
	return (need + 15u) & ~(uint64_t)15u;
}

/* the rings of all receivers back to back, each 16-byte aligned; returns the bytes of the ring buffer */
VDL2_HD uint64_t vdl2_push_ring_layout(const vdl2_rx_input *rx, uint32_t n_rx, uint32_t max_chunk_bytes, uint32_t max_span, vdl2_rx_ring *out) {
	uint64_t base = 0;
	for(uint32_t r = 0; r < n_rx; r++) {
		out[r].base = base;
		out[r].cap = vdl2_push_ring_cap(max_chunk_bytes, max_span, rx[r].oversample * (rx[r].fmt == 1u ? 4u : 2u));
		base += out[r].cap;
	}
	return base;
}

/* bytes a push may write without touching a byte still queued or in flight */
VDL2_HD uint64_t vdl2_push_room(uint64_t cap, uint64_t head, uint64_t freed) { return cap - (head - freed); }

/* the one or two pieces of `len` bytes at stream position pos in a ring of cap bytes: ring offsets off[k], lengths len[k]
 * (len[1] = 0 unless the bytes wrap) */
typedef struct {
	uint64_t off[2];
	uint64_t len[2];
} vdl2_ring_segs;

VDL2_HD vdl2_ring_segs vdl2_ring_segments(uint64_t cap, uint64_t pos, uint64_t len) {
	vdl2_ring_segs s;
	s.off[0] = pos % cap;
	s.len[0] = len < cap - s.off[0] ? len : cap - s.off[0];
	s.off[1] = 0;
	s.len[1] = len - s.len[0];
	return s;
}

/* a span's take from one receiver: its whole queued groups, at most max_span */
VDL2_HD uint32_t vdl2_push_take(uint64_t head, uint64_t tail, uint32_t group_bytes, uint32_t max_span) {
	const uint64_t g = (head - tail) / group_bytes;
	return g < max_span ? (uint32_t)g : max_span;
}

/* the write position after a restart drops the queue: the next sample boundary at or after head (the queue's bytes,
 * a split sample included, belong to the old process) */
VDL2_HD uint64_t vdl2_push_realign(uint64_t head, uint32_t bpp) { return (head + bpp - 1u) / bpp * bpp; }

/* The table of one pushed span: as vdl2_rx_span_table, but receiver r's off is the ring offset of its tail (the span's
 * first byte) and its tail advances by n[r] groups */
VDL2_HD void vdl2_push_span_table(const vdl2_rx_input *rx, const vdl2_rx_ring *ring, uint32_t n_rx, const uint32_t *n, uint64_t *tail,
		uint64_t *pos, uint32_t *prev, vdl2_rx_span *out) {
	for(uint32_t r = 0; r < n_rx; r++) {
		out[r].off = tail[r] % ring[r].cap;
		out[r].n = n[r];
		out[r].prev_n = prev[r];
		out[r].dec_base = pos[r];
		tail[r] += (uint64_t)n[r] * rx[r].oversample * (rx[r].fmt == 1u ? 4u : 2u);
		pos[r] += n[r];
		prev[r] = n[r];
	}
}

/* Timestamp anchor of a burst whose sync lies in decimation group `sync` of a receiver: the stream position just past
 * the last input sample of that group, given a span that took groups from dec_base on starting at stream position
 * byte_base */
VDL2_HD uint64_t vdl2_push_sync_end(uint64_t sync, uint64_t dec_base, uint64_t byte_base, uint32_t group_bytes) {
	return byte_base + (sync - dec_base + 1u) * group_bytes;
}

/* ... and how far before its push's arrival that sample arrived: the input samples the push (which ends at stream
 * position push_end) carried after it, at the receiver's rate (samples per second) */
VDL2_HD double vdl2_push_back_seconds(uint64_t sample_end, uint64_t push_end, uint32_t bpp, uint32_t rate) {
	return (double)((push_end - sample_end) / bpp) / (double)rate;
}

/* ------------------------------------------------------------------------------------------------
 * Input levels (VDL2GPU_FLAG_INPUT_LEVELS): exact integer figures of every raw sample K0 converts.  A component's code c
 * is an integer whose ratio to the format's full scale is exactly the float the reference makes of it: cu8 c = 2v - 255
 * (c / 255 = (v - 127.5) / 127.5, src/demod.c:349-354), cs16 c = v (c / 32768, src/demod.c:361-363).  Formats as K0
 * takes them: 0 cu8, 1 interleaved cs16, 2 planar cs16.
 * ---------------------------------------------------------------------------------------------- */
/* per input, in device memory: the layout of vdl2gpu_input_levels (full_scale is filled in by the getter) */
typedef struct {
	uint64_t samples;
	uint64_t sum_i, sum_q;       /* int64 sums kept as two's complement, so that unsigned 64-bit atomics can add to them */
	uint64_t pow_lo, pow_hi;
	uint64_t clipped;
	uint32_t peak, full_scale;
} vdl2_levels;

VDL2_HD int32_t vdl2_level_code(uint32_t fmt, int32_t v) { return fmt == 0u ? 2 * v - 255 : v; }
VDL2_HD uint32_t vdl2_level_rail(uint32_t fmt, int32_t v) { return fmt == 0u ? (v == 0 || v == 255) : (v == -32768 || v == 32767); }
VDL2_HD uint32_t vdl2_level_mag(int32_t c) { return c < 0 ? (uint32_t)(-c) : (uint32_t)c; }
VDL2_HD uint32_t vdl2_level_full_scale(uint32_t fmt) { return fmt == 0u ? 255u : 32768u; }
/* c_I^2 + c_Q^2 of one complex sample: at most 2 x 32768^2 = 2^31 */
VDL2_HD uint32_t vdl2_level_pow(int32_t ci, int32_t cq) { return (uint32_t)(ci * ci) + (uint32_t)(cq * cq); }

/* The 128-bit sum of squares: a 64-bit addend v goes into (lo, hi).  lo + v wraps exactly when the sum comes out below v,
 * and then hi takes the carry.  The device does the same with an atomic add on lo, whose return value is the old lo: every
 * addend carries exactly once when it wraps lo, whatever order the blocks of a chunk add in, so the total is exact and
 * deterministic with any number of writers. */
VDL2_HD uint32_t vdl2_pow_carry(uint64_t old_lo, uint64_t v) { return old_lo + v < v ? 1u : 0u; }
VDL2_HD void vdl2_pow_fold(uint64_t &lo, uint64_t &hi, uint64_t v) {
	const uint64_t old = lo;
	lo = old + v;
	hi += vdl2_pow_carry(old, v);
}

/* ------------------------------------------------------------------------------------------------
 * Channel levels (VDL2GPU_FLAG_CHANNEL_LEVELS): every decimated sample's power p = fl32(fl32(re re) + fl32(im im)), no FMA,
 * the reference's symbol power (src/demod.c:266), on the dBFS scale of frame_pwr.  The levels form of K2a adds, per slot,
 * a histogram of p by octave, the 128-bit sum of q = (uint64)(p 2^48) and the largest p (as float bits: p >= 0, so the
 * bits order like the values) to planes of uint64 [VDL2_CHLV_ROWS][n_chp] followed by uint32 [n_chp] (the peak).
 * ---------------------------------------------------------------------------------------------- */
#define VDL2_CHLV_BINS 40
#define VDL2_CHLV_POW_LO VDL2_CHLV_BINS         /* rows of the uint64 plane: bins, then the power's low and high words */
#define VDL2_CHLV_POW_HI (VDL2_CHLV_BINS + 1)
#define VDL2_CHLV_ROWS (VDL2_CHLV_BINS + 2)

VDL2_HD uint32_t vdl2_f32_bits(float f) {
#if defined(__CUDA_ARCH__)
	return __float_as_uint(f);
#else
	uint32_t u;
	memcpy(&u, &f, 4);
	return u;
#endif
}
VDL2_HD float vdl2_chlv_pow(float re, float im) { return F_ADD(F_MUL(re, re), F_MUL(im, im)); }
/* from the biased exponent E alone: [0] p < 2^-36 (zeros and subnormals included), [b] 2^(b-37) <= p < 2^(b-36) for
 * b = 1..38, [39] p >= 2^2 */
VDL2_HD uint32_t vdl2_chlv_bin(float p) {
	const int32_t e = (int32_t)((vdl2_f32_bits(p) >> 23) & 0xFFu) - 90;
	return (uint32_t)(e < 0 ? 0 : e > VDL2_CHLV_BINS - 1 ? VDL2_CHLV_BINS - 1 : e);
}
/* p 2^48 truncated: the scaling is exact, and p < 2^15 for every decimated sample (inputs within full scale), so q < 2^63 */
VDL2_HD uint64_t vdl2_chlv_q(float p) {
#if defined(__CUDA_ARCH__)
	return __float2ull_rz(p * 281474976710656.0f);
#else
	return (uint64_t)(p * 281474976710656.0f);
#endif
}

/* ------------------------------------------------------------------------------------------------
 * Spectrum (VDL2GPU_FLAG_SPECTRUM): the power spectrum of every input in VDL2_SPEC_N bins.  Segment j of an input is its
 * complex samples [N j, N (j + 1)) counted from the grid's origin (create, the receiver's joining, its restart), x_n the
 * float K0 made of sample n.  Per segment: y_n = fl32(x_n w_n) with the periodic Hann window w; a radix-2 decimation-in-time
 * FFT over the bit-reversed y, every product and sum rounded on its own; the power of each bin p = fl32(fl32(re re) +
 * fl32(im im)) (vdl2_chlv_pow), stored shifted: stored bin k holds FFT bin (k + N/2) mod N, frequency (k - N/2) fs / N.
 * Per input and stored bin, cumulative: the 128-bit sum of q = (uint64)(p 2^40) and the largest p.
 * |X_k| <= sum of w |x| <= 512 sqrt(2), so p <= 2^19 and q < 2^60.
 * ---------------------------------------------------------------------------------------------- */
#define VDL2_SPEC_N 1024u
#define VDL2_SPEC_LOG2N 10u

/* per input, in device memory: the accumulators (lo, hi: q sums; peak: p's float bits, p >= 0 so the bits order like the
 * values), then the samples of the segment not yet complete (carry[0, pending)) */
typedef struct {
	uint64_t lo[VDL2_SPEC_N];
	uint64_t hi[VDL2_SPEC_N];
	uint32_t peak[VDL2_SPEC_N];
	float2 carry[VDL2_SPEC_N];
} vdl2_spec_acc;

/* the window and the twiddles, made once on the host: w_n = 0.5 - 0.5 cos(2 pi n / N) and W^k = (cos(2 pi k / N),
 * -sin(2 pi k / N)) for k < N/2, each evaluated in double and rounded to float once */
typedef struct {
	float win[VDL2_SPEC_N];
	float2 tw[VDL2_SPEC_N / 2];
} vdl2_spec_tab;

static inline void vdl2_spec_make_tab(vdl2_spec_tab *t) {
	for(uint32_t n = 0; n < VDL2_SPEC_N; n++) t->win[n] = (float)(0.5 - 0.5 * cos(2.0 * VDL2_PI * (double)n / (double)VDL2_SPEC_N));
	for(uint32_t k = 0; k < VDL2_SPEC_N / 2; k++) {
		t->tw[k].x = (float)cos(2.0 * VDL2_PI * (double)k / (double)VDL2_SPEC_N);
		t->tw[k].y = (float)-sin(2.0 * VDL2_PI * (double)k / (double)VDL2_SPEC_N);
	}
}

VDL2_HD uint32_t vdl2_spec_bitrev(uint32_t n) {
	uint32_t r = 0;
	for(uint32_t b = 0; b < VDL2_SPEC_LOG2N; b++) r |= ((n >> b) & 1u) << (VDL2_SPEC_LOG2N - 1u - b);
	return r;
}
VDL2_HD float2 vdl2_spec_windowed(float2 x, float w) { float2 y; y.x = F_MUL(x.x, w); y.y = F_MUL(x.y, w); return y; }
/* butterfly b (< N/2) of stage s (0 .. LOG2N - 1): the pair it combines and the twiddle it takes */
VDL2_HD void vdl2_spec_pair(uint32_t s, uint32_t b, uint32_t &i0, uint32_t &i1, uint32_t &k) {
	const uint32_t half = 1u << s, j = b & (half - 1u);
	i0 = ((b >> s) << (s + 1u)) + j;
	i1 = i0 + half;
	k = j << (VDL2_SPEC_LOG2N - 1u - s);
}
/* a, b <- a + w b, a - w b */
VDL2_HD void vdl2_spec_bfly(float2 &a, float2 &b, float2 w) {
	const float tr = F_SUB(F_MUL(b.x, w.x), F_MUL(b.y, w.y));
	const float ti = F_ADD(F_MUL(b.x, w.y), F_MUL(b.y, w.x));
	b.x = F_SUB(a.x, tr); b.y = F_SUB(a.y, ti);
	a.x = F_ADD(a.x, tr); a.y = F_ADD(a.y, ti);
}
/* the FFT bin stored bin k holds */
VDL2_HD uint32_t vdl2_spec_fft_bin(uint32_t k) { return (k + VDL2_SPEC_N / 2u) & (VDL2_SPEC_N - 1u); }
/* p 2^40 truncated: the scaling is exact and p < 2^20, so q < 2^60 */
VDL2_HD uint64_t vdl2_spec_q(float p) {
#if defined(__CUDA_ARCH__)
	return __float2ull_rz(p * 1099511627776.0f);
#else
	return (uint64_t)(p * 1099511627776.0f);
#endif
}

/* One segment, serially (the device runs the same butterflies in parallel): x[N] in, p[N] (stored order) out; buf[N] is
 * scratch */
VDL2_HD void vdl2_spec_segment(const float2 *x, const vdl2_spec_tab *t, float2 *buf, float *p) {
	for(uint32_t n = 0; n < VDL2_SPEC_N; n++) buf[vdl2_spec_bitrev(n)] = vdl2_spec_windowed(x[n], t->win[n]);
	for(uint32_t s = 0; s < VDL2_SPEC_LOG2N; s++)
		for(uint32_t b = 0; b < VDL2_SPEC_N / 2u; b++) {
			uint32_t i0, i1, k;
			vdl2_spec_pair(s, b, i0, i1, k);
			vdl2_spec_bfly(buf[i0], buf[i1], t->tw[k]);
		}
	for(uint32_t k = 0; k < VDL2_SPEC_N; k++) {
		const float2 v = buf[vdl2_spec_fft_bin(k)];
		p[k] = vdl2_chlv_pow(v.x, v.y);
	}
}

/* The segment grid of one input in one chunk or span: it holds `pend` samples of its incomplete segment (its position
 * since the grid's origin, mod N) and brings n.  Sample m of the chunk's segment j is the input's sample N j + m - pend of
 * the chunk when that is >= 0, else carry[pend + (N j + m - pend)]. */
typedef struct {
	uint32_t pend, n;
} vdl2_spec_span;

/* the grid entry of a chunk that brings n samples to an input at position pos (samples since the grid's origin), which
 * then advances */
VDL2_HD vdl2_spec_span vdl2_spec_step(uint64_t &pos, uint32_t n) {
	vdl2_spec_span e;
	e.pend = (uint32_t)(pos & (VDL2_SPEC_N - 1u));
	e.n = n;
	pos += n;
	return e;
}
VDL2_HD uint32_t vdl2_spec_segments(vdl2_spec_span e) { return (uint32_t)(((uint64_t)e.pend + e.n) >> VDL2_SPEC_LOG2N); }
VDL2_HD uint32_t vdl2_spec_rest(vdl2_spec_span e) { return (e.pend + e.n) & (VDL2_SPEC_N - 1u); }
/* where sample m of segment j comes from: >= 0 the chunk's sample, < 0 carry[pend + that] */
VDL2_HD int64_t vdl2_spec_src(vdl2_spec_span e, uint32_t j, uint32_t m) { return (int64_t)j * VDL2_SPEC_N + m - e.pend; }

#endif
