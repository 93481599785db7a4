/*
 * oracle/vdl2_oracle.c — CPU restatement of dumpvdl2's per-channel DSP hot path.
 * TEST INFRASTRUCTURE ONLY — see vdl2_oracle.h for who may call this and how parity is pinned.
 *
 * This is a restatement, not a copy: the data structures are this repo's own (packed event
 * records, frame arena, polynomial-form Reed-Solomon), but every arithmetic step keeps the
 * operand order and the float/double promotion of the reference source so that, compiled
 * without fast-math, it reproduces the "strict" build of the reference bit for bit.
 * Citations are file:line under /root/reference.
 */
#define _GNU_SOURCE
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "vdl2_oracle.h"

/* ------------------------------------------------------------------------------------------
 * Tables that the reference computes at start-up
 * ---------------------------------------------------------------------------------------- */

/* src/demod.c:349-354 — cu8 level table */
void vo_levels_u8(float levels[256]) {
	for(int code = 0; code < 256; code++)
		levels[code] = ((float)code - 127.5f) / 127.5f;
}

/* src/demod.c:372-377 — 256-step sine/cosine table with a wrap entry */
void vo_sincos_lut(float sin_lut[257], float cos_lut[257]) {
	for(uint32_t step = 0; step < 256; step++) {
		/* 2.0f * M_PI is a double product; the argument narrows to float at the call */
		float angle = (float)(2.0f * M_PI * (float)step / 256.0f);
		sincosf(angle, &sin_lut[step], &cos_lut[step]);
	}
	sin_lut[256] = sin_lut[0];
	cos_lut[256] = cos_lut[0];
}

/* src/demod.c:367-370 -> src/chebyshev.c:67-119 with npoles == 2 (INP_LPF_NPOLES), cutoff
 * 8000 Hz, ripple 0.5 %.  Smith, "The Scientist and Engineer's Guide to DSP", ch. 20.
 * With two poles the cascade loop of chebyshev.c:94-105 runs once and, the seed polynomials
 * being {1}, leaves A = AA and B = {-0, BB1, BB2}; the gain normalisation (chebyshev.c:111-118)
 * then divides A by sum(A)/(1-sum(B)).  Adding the reference's zero-valued tail terms is exact,
 * so they are omitted. */
void vo_lpf_design(uint32_t sample_rate, float A[3], float B[3]) {
	const float cutoff = (float)8000 / (float)sample_rate;
	const float ripple = 0.5f;
	const int npoles = 2;
	float pole_im, pole_re;
	/* chebyshev.c:35 — pole on the unit circle (p == 1) */
	sincosf((float)(M_PI / (2 * npoles) + (1 - 1) * M_PI / npoles), &pole_im, &pole_re);
	pole_re = -pole_re;
	/* chebyshev.c:37-45 — warp the circle into an ellipse */
	float es = sqrtf(powf(100.f / (100.f - ripple), 2.f) - 1.f);
	float vx = (1.f / npoles) * logf((1.f / es) + sqrtf(1.f / (es * es) + 1.f));
	float kx = (1.f / npoles) * logf((1.f / es) + sqrtf(1.f / (es * es) - 1.f));
	kx = (expf(kx) + expf(-kx)) / 2.f;
	pole_re *= ((expf(vx) - expf(-vx)) / 2.f) / kx;
	pole_im *= ((expf(vx) + expf(-vx)) / 2.f) / kx;
	/* chebyshev.c:47-56 — s-domain to z-domain */
	float t = 2.f * tanf(0.5f);
	float w = (float)(2.f * M_PI * cutoff);
	float m = pole_re * pole_re + pole_im * pole_im;
	float d = 4.f - 4.f * pole_re * t + m * t * t;
	float x0 = t * t / d;
	float x1 = 2.f * x0;
	float x2 = x0;
	float y1 = (8.f - 2.f * m * t * t) / d;
	float y2 = (-4.f - 4.f * pole_re * t - m * t * t) / d;
	/* chebyshev.c:58-64 — low-pass to low-pass frequency transform */
	float k = sinf(0.5f - w / 2.f) / sinf(0.5f + w / 2.f);
	d = 1 + y1 * k - y2 * k * k;
	float aa0 = (x0 - x1 * k + x2 * k * k) / d;
	float aa1 = (-2.f * x0 * k + x1 + x1 * k * k - 2.f * x2 * k) / d;
	float aa2 = (x0 * k * k - x1 * k + x2) / d;
	float bb1 = (2.f * k + y1 + y1 * k * k - 2.f * y2 * k) / d;
	float bb2 = (-(k * k) - y1 * k + y2) / d;
	/* chebyshev.c:107-118 — unity DC gain */
	float sa = 0.f, sb = 0.f;
	sa += aa0; sa += aa1; sa += aa2;
	sb += -0.f; sb += bb1; sb += bb2;
	float gain = sa / (1.f - sb);
	A[0] = aa0 / gain;
	A[1] = aa1 / gain;
	A[2] = aa2 / gain;
	B[0] = -0.f;
	B[1] = bb1;
	B[2] = bb2;
}

/* src/demod.c:84-96 (regression constants) and :107-124 (preamble phases) */
void vo_sync_consts(float lr_X[16], float *lr_denom, float pr_phase[16]) {
	static const int quarter_pi_steps[VO_PREAMBLE_SYMS] = { 0, 3, -3, 1, 1, 2, 0, 4, -3, 4, -2, 3, 1, -2, -3, 0 };
	float mean_x = 0.f;
	for(int i = 0; i < VO_PREAMBLE_SYMS; i++)
		mean_x += i;
	mean_x /= VO_PREAMBLE_SYMS;
	float denom = 0.f;
	for(int i = 0; i < VO_PREAMBLE_SYMS; i++) {
		lr_X[i] = i - mean_x;
		denom += (i - mean_x) * (i - mean_x);
	}
	*lr_denom = denom;
	for(int i = 0; i < VO_PREAMBLE_SYMS; i++)
		pr_phase[i] = (float)(quarter_pi_steps[i] * M_PI / 4);
}

/* src/demod.c:385 */
uint32_t vo_downmix_dphi(uint32_t centerfreq, uint32_t freq, uint32_t rate) {
	return (uint32_t)(int)(((float)centerfreq - (float)freq) / (float)rate * 256.0f * 65536.0f);
}

/* ------------------------------------------------------------------------------------------
 * Header block code (25,20)   src/decode.c:55-122
 * ---------------------------------------------------------------------------------------- */
static const uint32_t hdr_check_rows[VO_HDRFECLEN] = {
	0x001FFF0u, 0x07E1FE8u, 0x18E61E4u, 0x1B6A662u, 0x0D3CAA1u
};
/* error pattern per syndrome: src/decode.c:63-96 (single-bit errors, plus the double-bit patterns
 * the reference assigns to the remaining syndromes).  The values are wire-contract data; they are
 * checked against the reference's binary literals by tests/test_oracle_tables.py. */
static const uint32_t hdr_error_pattern[32] = {
	0x0000000u, 0x0000001u, 0x0000002u, 0x0800004u, 0x0000004u, 0x0800002u, 0x1000000u, 0x0800000u,
	0x0000008u, 0x0400000u, 0x0200000u, 0x0100000u, 0x0080000u, 0x1100000u, 0x0040000u, 0x0020000u,
	0x0000010u, 0x0010000u, 0x0804000u, 0x0008000u, 0x0808000u, 0x0004000u, 0x0002000u, 0x1010000u,
	0x0001000u, 0x0000800u, 0x0000400u, 0x0000200u, 0x0000100u, 0x0000080u, 0x0000040u, 0x0000020u
};
static const uint8_t hdr_synd_weight[32] = {
	0, 1, 1, 2, 1, 2, 1, 1, 1, 1, 1, 1, 1, 2, 1, 1, 1, 1, 2, 1, 2, 1, 1, 2, 1, 1, 1, 1, 1, 1, 1, 1
};

static uint32_t parity32(uint32_t v) {
	v ^= v >> 16; v ^= v >> 8; v ^= v >> 4; v ^= v >> 2; v ^= v >> 1;
	return v & 1u;
}

uint32_t vo_header_decode(uint32_t *word25) {
	uint32_t syndrome = 0;
	for(int row = 0; row < VO_HDRFECLEN; row++)
		syndrome |= parity32(*word25 & hdr_check_rows[row]) << (VO_HDRFECLEN - 1 - row);
	*word25 ^= hdr_error_pattern[syndrome];
	return syndrome;
}

uint32_t vo_synd_weight(uint32_t syndrome) { return hdr_synd_weight[syndrome & 31u]; }

/* src/bitstream.c:152-164 — bit reversal within a numbits-wide field */
uint32_t vo_reverse_bits(uint32_t v, int numbits) {
	uint32_t r = 0;
	for(int b = 0; b < numbits; b++)
		if(v & (1u << b)) r |= 1u << (numbits - 1 - b);
	return r;
}

/* inverse of the header decode: [24:22]=0, [21:5]=length sent LSB first, [4:0] parity (SURVEY App. A.4) */
uint32_t vo_header_encode(uint32_t datalen_bits) {
	uint32_t word = vo_reverse_bits(datalen_bits & 0x1FFFFu, VO_TRLEN) << VO_HDRFECLEN;
	for(int row = 0; row < VO_HDRFECLEN; row++)
		word |= parity32(word & hdr_check_rows[row] & ~0x1Fu) << (VO_HDRFECLEN - 1 - row);
	return word;
}

/* src/decode.c:124-133 */
int vo_fec_octets_for(uint32_t len) {
	if(len < 3) return 0;
	if(len < 31) return 2;
	if(len < 68) return 4;
	return 6;
}

/* ------------------------------------------------------------------------------------------
 * CRC-16 (AVLC FCS)   src/crc.c:21-64: reflected 0x1021 (0x8408), table driven there,
 * bitwise here (same function).
 * ---------------------------------------------------------------------------------------- */
uint16_t vo_crc16(const uint8_t *data, uint32_t len, uint16_t init) {
	uint16_t crc = init;
	for(uint32_t n = 0; n < len; n++) {
		crc ^= data[n];
		for(int b = 0; b < 8; b++)
			crc = (crc & 1u) ? (uint16_t)((crc >> 1) ^ 0x8408u) : (uint16_t)(crc >> 1);
	}
	return crc;
}

/* ------------------------------------------------------------------------------------------
 * Scrambler   src/bitstream.c:94-107 (x^15 + x + 1, 15-bit state, output = b0 ^ b14)
 * ---------------------------------------------------------------------------------------- */
void vo_scramble_bits(uint8_t *bits, uint32_t nbits, uint16_t *lfsr) {
	uint16_t s = *lfsr;
	for(uint32_t n = 0; n < nbits; n++) {
		uint8_t out = (uint8_t)((s ^ (s >> 14)) & 1u);
		s = (uint16_t)((s >> 1) | (out << 14));
		bits[n] ^= out;
	}
	*lfsr = s;
}

/* ------------------------------------------------------------------------------------------
 * Reed-Solomon RS(255,249) over GF(2^8)/0x187, first root alpha^120, 6 roots.
 * src/rs.c:27-49 -> src/libfec/init_rs.h:48-103, src/libfec/decode_rs.h:71-298 (Karn).
 * Restated in polynomial form; the control flow (erasure-seeded Berlekamp-Massey, Chien search
 * with early exit, "deg(lambda) != roots" failure rule, Forney) follows decode_rs.h so that
 * behaviour beyond the correction capacity (mis-corrections, failures) is identical.
 * ---------------------------------------------------------------------------------------- */
enum { GF_NN = 255, RS_ROOTS = 6, RS_FCR = 120 };
static uint8_t gf_exp[512];
static int gf_log[256];
static int gf_ready;

static void gf_init(void) {
	if(gf_ready) return;
	int v = 1;
	for(int e = 0; e < GF_NN; e++) {              /* init_rs.h:48-58 */
		gf_exp[e] = (uint8_t)v;
		gf_log[v] = e;
		v <<= 1;
		if(v & 0x100) v ^= 0x187;
	}
	for(int e = GF_NN; e < 512; e++) gf_exp[e] = gf_exp[e - GF_NN];
	gf_log[0] = -1;
	gf_ready = 1;
}
static inline uint8_t gf_mul(uint8_t a, uint8_t b) { return (a && b) ? gf_exp[gf_log[a] + gf_log[b]] : 0; }
static inline uint8_t gf_alpha(int e) { e %= GF_NN; if(e < 0) e += GF_NN; return gf_exp[e]; }

/* decode_rs.h; returns number of located symbols (erasures included) or -1 */
static int rs_decode_255_249(uint8_t *data, const int *eras_pos, int no_eras) {
	gf_init();
	uint8_t S[RS_ROOTS];
	/* syndromes by Horner, data[0] is the highest-order coefficient: decode_rs.h:82-93 */
	for(int i = 0; i < RS_ROOTS; i++) {
		uint8_t acc = data[0], root = gf_alpha(RS_FCR + i);
		for(int j = 1; j < GF_NN; j++)
			acc = gf_mul(acc, root) ^ data[j];
		S[i] = acc;
	}
	int any = 0;
	for(int i = 0; i < RS_ROOTS; i++) any |= S[i];
	if(!any) return 0;                                                      /* decode_rs.h:102-108 */

	uint8_t lambda[RS_ROOTS + 1] = { 1, 0, 0, 0, 0, 0, 0 };
	if(no_eras > 0) {                                                       /* decode_rs.h:112-122 */
		lambda[1] = gf_alpha(GF_NN - 1 - eras_pos[0]);
		for(int i = 1; i < no_eras; i++) {
			uint8_t x = gf_alpha(GF_NN - 1 - eras_pos[i]);
			for(int j = i + 1; j > 0; j--)
				lambda[j] ^= gf_mul(x, lambda[j - 1]);
		}
	}
	uint8_t B[RS_ROOTS + 1];
	memcpy(B, lambda, sizeof(B));                                           /* decode_rs.h:158-159 */

	/* Berlekamp-Massey, decode_rs.h:165-206 */
	int el = no_eras;
	for(int r = no_eras + 1; r <= RS_ROOTS; r++) {
		uint8_t discr = 0;
		for(int i = 0; i < r; i++)
			discr ^= gf_mul(lambda[i], S[r - i - 1]);
		if(discr == 0) {
			memmove(&B[1], B, RS_ROOTS);
			B[0] = 0;
		} else {
			uint8_t T[RS_ROOTS + 1];
			T[0] = lambda[0];
			for(int i = 0; i < RS_ROOTS; i++)
				T[i + 1] = lambda[i + 1] ^ gf_mul(discr, B[i]);
			if(2 * el <= r + no_eras - 1) {
				el = r + no_eras - el;
				uint8_t inv = gf_alpha(GF_NN - gf_log[discr]);
				for(int i = 0; i <= RS_ROOTS; i++)
					B[i] = gf_mul(lambda[i], inv);
			} else {
				memmove(&B[1], B, RS_ROOTS);
				B[0] = 0;
			}
			memcpy(lambda, T, sizeof(T));
		}
	}
	int deg_lambda = 0;
	for(int i = 0; i <= RS_ROOTS; i++)
		if(lambda[i]) deg_lambda = i;

	/* Chien search, decode_rs.h:214-239: i = 1..255, position k = i-1, stop once deg roots found */
	int root[RS_ROOTS], loc[RS_ROOTS], count = 0;
	for(int i = 1; i <= GF_NN; i++) {
		uint8_t q = 1;
		for(int j = deg_lambda; j > 0; j--)
			if(lambda[j]) q ^= gf_mul(lambda[j], gf_alpha(i * j));
		if(q != 0) continue;
		root[count] = i;
		loc[count] = i - 1;
		if(++count == deg_lambda) break;
	}
	if(deg_lambda != count) return -1;                                       /* decode_rs.h:240-247 */

	/* omega = S * lambda mod x^NROOTS, up to degree deg_lambda-1: decode_rs.h:252-260 */
	int deg_omega = deg_lambda - 1;
	uint8_t omega[RS_ROOTS + 1] = { 0 };
	for(int i = 0; i <= deg_omega; i++) {
		uint8_t acc = 0;
		for(int j = i; j >= 0; j--)
			acc ^= gf_mul(S[i - j], lambda[j]);
		omega[i] = acc;
	}
	/* Forney, decode_rs.h:266-291 */
	for(int j = count - 1; j >= 0; j--) {
		uint8_t num1 = 0;
		for(int i = deg_omega; i >= 0; i--)
			num1 ^= gf_mul(omega[i], gf_alpha(i * root[j]));
		uint8_t num2 = gf_alpha(root[j] * (RS_FCR - 1) + GF_NN);
		uint8_t den = 0;
		int top = (deg_lambda < RS_ROOTS - 1 ? deg_lambda : RS_ROOTS - 1) & ~1;
		for(int i = top; i >= 0; i -= 2)
			den ^= gf_mul(lambda[i + 1], gf_alpha(i * root[j]));
		if(num1 != 0) {
			/* index arithmetic of decode_rs.h:289: log(0) is 255 there, so den == 0 divides by alpha^0 */
			int e = gf_log[num1] + gf_log[num2] + GF_NN - (den ? gf_log[den] : GF_NN);
			data[loc[j]] ^= gf_alpha(e);
		}
	}
	return count;
}

/* src/rs.c:32-49 */
int vo_rs_verify(uint8_t block[255], int fec_octets) {
	if(fec_octets == 0) return 0;
	int n_erased = VO_RS_N - VO_RS_K - fec_octets;
	int erasures[RS_ROOTS];
	for(int i = 0; i < n_erased; i++)
		erasures[i] = VO_RS_K + fec_octets + i;
	return rs_decode_255_249(block, n_erased > 0 ? erasures : NULL, n_erased > 0 ? n_erased : 0);
}

/* Systematic encoder (the reference ships none).  g(x) = prod_{i<6} (x - alpha^(120+i)),
 * as formed in init_rs.h:87-103; parity = x^6 * m(x) mod g(x), data[0] highest order. */
void vo_rs_encode(uint8_t block[255]) {
	gf_init();
	uint8_t g[RS_ROOTS + 1] = { 1, 0, 0, 0, 0, 0, 0 };     /* g[k] = coeff of x^k */
	for(int i = 0; i < RS_ROOTS; i++) {
		uint8_t r = gf_alpha(RS_FCR + i);
		for(int k = i + 1; k > 0; k--)
			g[k] = g[k - 1] ^ gf_mul(g[k], r);
		g[0] = gf_mul(g[0], r);
	}
	uint8_t rem[RS_ROOTS] = { 0 };                          /* rem[0] = highest order */
	for(int j = 0; j < VO_RS_K; j++) {
		uint8_t fb = block[j] ^ rem[0];
		for(int k = 0; k < RS_ROOTS - 1; k++)
			rem[k] = rem[k + 1] ^ gf_mul(fb, g[RS_ROOTS - 1 - k]);
		rem[RS_ROOTS - 1] = gf_mul(fb, g[0]);
	}
	memcpy(block + VO_RS_K, rem, RS_ROOTS);
}

/* ------------------------------------------------------------------------------------------
 * DEC_DATA stage on descrambled bits   src/decode.c:259-380
 * `bits` holds one bit per byte, starting at the first payload bit (i.e. after the 25 header bits).
 * ---------------------------------------------------------------------------------------- */
static uint8_t take_octet_lsb_first(const uint8_t *bits) {            /* src/bitstream.c:70-81 */
	uint8_t v = 0;
	for(int b = 0; b < 8; b++) v |= (uint8_t)((bits[b] & 1u) << b);
	return v;
}

int vo_decode_burst_bits(const uint8_t *bits, uint32_t nbits, uint32_t datalen_bits,
		uint8_t *frames_out, uint32_t frames_cap, uint32_t *frame_lens, uint32_t max_frames,
		uint32_t *n_frames, int32_t *num_fec_corrections, int8_t rs_ret[9]) {
	*n_frames = 0;
	*num_fec_corrections = 0;
	for(int i = 0; i < 9; i++) rs_ret[i] = -128;
	/* geometry: src/decode.c:233-245 */
	uint32_t datalen_octets = datalen_bits / 8 + (datalen_bits % 8 != 0);
	uint32_t num_blocks = datalen_octets / VO_RS_K;
	uint32_t fec_octets = num_blocks * (VO_RS_N - VO_RS_K);
	uint32_t last_len = datalen_octets % VO_RS_K;
	if(last_len != 0) num_blocks++;
	fec_octets += (uint32_t)vo_fec_octets_for(last_len);
	if(last_len == 0) last_len = VO_RS_K;
	if(fec_octets == 0) return VO_ERR_NO_FEC;
	if(num_blocks > 9) return VO_ERR_TOO_LONG;
	if(nbits < 8 * datalen_octets) return VO_ERR_DATA_TRUNCATED;      /* src/decode.c:266-270 */
	if(nbits < 8 * (datalen_octets + fec_octets)) return VO_ERR_FEC_TRUNCATED;

	/* octets LSB first, then column-wise de-interleave: src/decode.c:266-297, 135-163.
	 * Transmit order is "octet c of block 0, of block 1, ... " skipping cells past the end of the
	 * short last row; FEC octets likewise over the rows that carry FEC. */
	uint8_t table[9][VO_RS_N];
	memset(table, 0, sizeof(table));
	const uint8_t *p = bits;
	for(uint32_t col = 0, taken = 0; taken < datalen_octets; col++)
		for(uint32_t row = 0; row < num_blocks && taken < datalen_octets; row++) {
			if(row == num_blocks - 1 && col >= last_len) continue;
			table[row][col] = take_octet_lsb_first(p);
			p += 8; taken++;
		}
	int last_fec = vo_fec_octets_for(last_len);
	uint32_t fec_rows = num_blocks - (last_fec == 0 ? 1u : 0u);
	for(uint32_t col = 0, taken = 0; taken < fec_octets; col++)
		for(uint32_t row = 0; row < fec_rows && taken < fec_octets; row++) {
			if(row == num_blocks - 1 && col >= (uint32_t)last_fec) continue;
			table[row][VO_RS_K + col] = take_octet_lsb_first(p);
			p += 8; taken++;
		}

	/* per-block FEC and re-serialisation: src/decode.c:304-334 */
	static _Thread_local uint8_t stream[VO_MAX_BURST_BITS];
	uint32_t stream_len = 0;
	for(uint32_t row = 0; row < num_blocks; row++) {
		int nfec = (row == num_blocks - 1) ? last_fec : (VO_RS_N - VO_RS_K);
		int ret = vo_rs_verify(table[row], nfec);
		rs_ret[row] = (int8_t)ret;
		if(ret < 0) return VO_ERR_FEC_BAD;
		if(ret > 0) *num_fec_corrections += ret - (VO_RS_N - VO_RS_K - nfec);
		uint32_t take = (row == num_blocks - 1) ? last_len : VO_RS_K;
		for(uint32_t o = 0; o < take; o++)
			for(int b = 0; b < 8; b++)
				stream[stream_len++] = (table[row][o] >> b) & 1u;
	}
	if(datalen_bits < stream_len) stream_len = datalen_bits;              /* src/decode.c:338-342 */

	/* HDLC flag search + zero-bit deletion: src/bitstream.c:109-150, loop src/decode.c:345-370 */
	static _Thread_local uint8_t fbits[VO_MAX_BURST_BITS];
	uint32_t pos = 0, out_used = 0;
	for(;;) {
		uint32_t flen;
		int ones, more;
	rescan:
		ones = 0; flen = 0;
		{
			int closed = 0;
			while(pos < stream_len) {
				uint8_t bit = stream[pos];
				if(bit == 0 && ones == 5) { ones = 0; pos++; continue; }   /* stuffed zero */
				if(bit == 1 && ++ones > 6) return VO_ERR_UNSTUFF;           /* seven ones */
				fbits[flen] = bit;
				if(bit == 0) {
					if(ones == 6) {                                          /* 01111110 */
						if(flen == 7) { pos++; goto rescan; }                /* opening flag */
						if(flen < 7) return VO_ERR_UNSTUFF;
						flen -= 7; pos++; closed = 1;
						break;
					}
					ones = 0;
				}
				flen++; pos++;
			}
			(void)closed;
		}
		more = pos < stream_len;
		if(flen % 8 != 0) return VO_ERR_TRUNCATED_OCTETS;                  /* src/decode.c:346-350 */
		uint32_t octets = flen / 8;
		if(*n_frames >= max_frames || out_used + octets > frames_cap) return VO_ERR_BITSTREAM;
		for(uint32_t o = 0; o < octets; o++)
			frames_out[out_used + o] = take_octet_lsb_first(fbits + 8 * o);
		frame_lens[(*n_frames)++] = octets;
		out_used += octets;
		if(!more) break;                                                     /* src/decode.c:363-365 */
	}
	return VO_BURST_OK;
}

/* ------------------------------------------------------------------------------------------
 * Channel state and the per-sample chain
 * ---------------------------------------------------------------------------------------- */
enum { ST_SEARCH = 0, ST_LOCKED = 1 };               /* DM_INIT / DM_SYNC, src/dumpvdl2.h:294 */
enum { DS_HEADER = 0, DS_DATA = 1, DS_IDLE = 2 };    /* src/dumpvdl2.h:295 */

typedef struct {
	/* front end: src/demod.c:289-298 locals, persistent across buffers */
	float xr[3], xi[3], yr[3], yi[3];
	uint32_t nco_phase, nco_step;
	int mixes;
	int decim_count;
	/* demodulator: src/dumpvdl2.h:321-352 */
	float ring[VO_SYNC_BUFLEN];
	int ring_pos;
	float prev_phi, prev_dphi, dphi;
	float pherr[3];
	float ppm_error, mag_lp, mag_nf, frame_pwr;
	int nfcnt, frame_pwr_cnt, sclk;
	int demod_state, decoder_state;
	uint32_t freq;
	/* burst bits, one per byte, header included */
	uint8_t *bits;
	uint32_t nbits, read_pos, descrambled;
	uint32_t requested_bits, datalen, syndrome;
	uint16_t lfsr;
	uint32_t burst_seq;
	uint64_t dec_index;              /* index of the decimated sample being processed */
	uint64_t sync_dec_index;
} chan_t;

struct vo_ctx {
	uint32_t rate, oversample, centerfreq, n_channels;
	int fmt;
	float max_ppm;
	float levels[256], sin_lut[257], cos_lut[257];
	float A[3], B[3];
	float lr_X[16], lr_denom, pr_phase[16];
	chan_t *ch;
	float *sbuf; uint32_t sbuf_cap;
	vo_frame *frames; uint32_t n_frames, cap_frames;
	uint8_t *arena; uint32_t arena_used, arena_cap;
	int trace; vo_event *events; uint32_t n_events, cap_events;
	int tap; float *dec; uint64_t dec_count, dec_cap;
	int state_tap; uint32_t *state; float *pherr1; uint64_t state_count, state_cap;
	uint64_t *counters;
};

static void push_event(vo_ctx *c, const vo_event *e) {
	if(!c->trace) return;
	if(c->n_events == c->cap_events) {
		c->cap_events = c->cap_events ? 2 * c->cap_events : 256;
		c->events = realloc(c->events, c->cap_events * sizeof(vo_event));
	}
	c->events[c->n_events++] = *e;
}

/* src/demod.c:205-220 */
static void reset_decoder(chan_t *v) {
	v->decoder_state = DS_HEADER;
	v->requested_bits = VO_HEADER_LEN;
	v->nbits = v->read_pos = v->descrambled = 0;
}
static void reset_demod(chan_t *v) {
	reset_decoder(v);
	v->sclk = 0;
	v->demod_state = ST_SEARCH;
	v->pherr[1] = v->pherr[2] = 1000.f;
	v->frame_pwr = 0.f;
	v->frame_pwr_cnt = 0;
}

/* src/demod.c:98-103 */
static float parabola_vertex(float x, int d, float y1, float y2, float y3) {
	float denom = (float)(d * 2 * d * (-d));
	float qa = (x * (y2 - y1) + (x - d) * (y1 - y3) + (x - 2 * d) * (y3 - y2)) / denom;
	float qb = (x * x * (y1 - y2) + (x - d) * (x - d) * (y3 - y1) + (x - 2 * d) * (x - 2 * d) * (y2 - y3)) / denom;
	return -qb / (2 * qa);
}

/* src/demod.c:105-198 */
static int preamble_metric(vo_ctx *c, chan_t *v, uint32_t chan_idx) {
	float err[VO_PREAMBLE_SYMS];
	float unwrap = 0.f, mean;
	float prev = mean = err[0] = v->ring[(v->ring_pos + VO_SPS) % VO_SYNC_BUFLEN] - c->pr_phase[0];
	for(int i = 1; i < VO_PREAMBLE_SYMS; i++) {
		float cur = v->ring[(v->ring_pos + (i + 1) * VO_SPS) % VO_SYNC_BUFLEN] - c->pr_phase[i];
		float step = cur - prev;
		prev = cur;
		if(step > M_PI) unwrap -= 2.0f * M_PI;            /* double arithmetic, narrowed on store */
		else if(step < -M_PI) unwrap += 2.0f * M_PI;
		err[i] = cur + unwrap;
		mean += err[i];
	}
	mean /= VO_PREAMBLE_SYMS;
	for(int i = 0; i < VO_PREAMBLE_SYMS; i++) err[i] -= mean;
	float slope = 0.f;
	for(int i = 0; i < VO_PREAMBLE_SYMS; i++) slope += c->lr_X[i] * err[i];
	slope /= c->lr_denom;
	v->pherr[0] = 0.f;
	for(int i = 0; i < VO_PREAMBLE_SYMS; i++) {
		float e = err[i] - slope * c->lr_X[i];
		v->pherr[0] += e * e;
	}
	if(v->pherr[1] < 4.f && v->pherr[0] > v->pherr[1]) {
		float vertex = parabola_vertex((float)v->sclk, 3, v->pherr[2], v->pherr[1], v->pherr[0]);
		v->sclk = (int)-roundf(vertex);
		int sp = v->ring_pos - v->sclk;
		if(sp < 0) sp += VO_SYNC_BUFLEN;
		/* the reference indexes its ring unchecked here; sclk is in [2,5] for every reachable
		 * metric triple (DESIGN.md), the wrap below only guards the oracle's own memory */
		sp = ((sp % VO_SYNC_BUFLEN) + VO_SYNC_BUFLEN) % VO_SYNC_BUFLEN;
		v->prev_phi = v->ring[sp];
		v->dphi = v->prev_dphi;
		v->ppm_error = (float)(VO_SYMBOL_RATE * v->dphi / (2.0f * M_PI * v->freq) * 1e+6);
		int accepted = !(c->max_ppm && fabsf(v->ppm_error) > c->max_ppm);
		if(c->trace) {
			vo_event e; memset(&e, 0, sizeof(e));
			e.channel = chan_idx; e.kind = VO_EV_SYNC; e.dec_index = v->dec_index;
			e.i[0] = v->sclk; e.i[1] = v->ring_pos; e.i[2] = sp; e.i[3] = accepted;
			e.f[0] = v->pherr[2]; e.f[1] = v->pherr[1]; e.f[2] = v->pherr[0]; e.f[3] = vertex;
			e.f[4] = v->prev_phi; e.f[5] = v->dphi; e.f[6] = v->ppm_error;
			push_event(c, &e);
		}
		v->pherr[1] = v->pherr[2] = 1000.f;
		return accepted;
	}
	v->pherr[2] = v->pherr[1];
	v->pherr[1] = v->pherr[0];
	v->prev_dphi = slope;
	return 0;
}

static void emit_frame(vo_ctx *c, chan_t *v, uint32_t chan_idx, int idx, const uint8_t *buf, uint32_t len,
		uint32_t datalen_octets, int32_t fec_corr) {
	if(c->n_frames == c->cap_frames) {
		c->cap_frames = c->cap_frames ? 2 * c->cap_frames : 64;
		c->frames = realloc(c->frames, c->cap_frames * sizeof(vo_frame));
	}
	if(c->arena_used + len > c->arena_cap) {
		c->arena_cap = 2 * (c->arena_cap + len) + 4096;
		c->arena = realloc(c->arena, c->arena_cap);
	}
	vo_frame *f = &c->frames[c->n_frames++];
	memset(f, 0, sizeof(*f));
	f->channel = chan_idx; f->freq = v->freq; f->burst_seq = v->burst_seq; f->idx = idx;
	f->len = len; f->offset = c->arena_used;
	f->synd_weight = vo_synd_weight(v->syndrome);
	f->datalen_octets = datalen_octets;
	f->num_fec_corrections = fec_corr;
	f->frame_pwr = v->frame_pwr; f->mag_nf = v->mag_nf;
	f->frame_pwr_dbfs = 10.0f * log10f(v->frame_pwr);                  /* src/decode.c:180-182 */
	f->nf_pwr_dbfs = 20.0f * log10f(v->mag_nf + 0.001f);
	f->ppm_error = v->ppm_error;
	f->sync_dec_index = v->sync_dec_index;
	f->fcs_residue = vo_crc16(buf, len, 0xFFFFu);
	memcpy(c->arena + c->arena_used, buf, len);
	c->arena_used += len;
	c->counters[chan_idx * VO_NUM_COUNTERS + VO_CNT_MSG_GOOD]++;
	if(len >= 11)                                                        /* src/avlc.c:39,168-187 */
		c->counters[chan_idx * VO_NUM_COUNTERS + (f->fcs_residue == 0xF0B8u ? VO_CNT_FCS_GOOD : VO_CNT_FCS_BAD)]++;
}

/* src/decode.c:196-384 */
static void burst_step(vo_ctx *c, chan_t *v, uint32_t chan_idx) {
	uint64_t *cnt = &c->counters[chan_idx * VO_NUM_COUNTERS];
	if(v->decoder_state == DS_HEADER) {
		v->lfsr = 0x6959u;
		vo_scramble_bits(v->bits + v->descrambled, v->nbits - v->descrambled, &v->lfsr);
		v->descrambled = v->nbits;
		uint32_t word = 0;
		for(int b = 0; b < VO_HEADER_LEN; b++)                            /* src/bitstream.c:83-92 */
			word |= (uint32_t)(v->bits[v->read_pos++] & 1u) << (VO_HEADER_LEN - 1 - b);
		uint32_t raw = word;
		word &= (1u << (VO_TRLEN + VO_HDRFECLEN)) - 1u;
		v->syndrome = vo_header_decode(&word);
		int status = VO_BURST_OK;
		uint32_t datalen = 0;
		if(v->syndrome == 0) cnt[VO_CNT_HDR_CRC_GOOD]++;
		if((word & ((1u << (VO_TRLEN + VO_HDRFECLEN)) - 1u)) != word) {
			status = VO_ERR_CRC_BAD;
		} else {
			datalen = vo_reverse_bits((word >> VO_HDRFECLEN) & 0x1FFFFu, VO_TRLEN);
			if((v->syndrome != 0 && datalen > 0x1FFFu) || datalen > 0x3FFFu) status = VO_ERR_TOO_LONG;
		}
		uint32_t octets = 0, fec = 0;
		if(status == VO_BURST_OK) {
			octets = datalen / 8 + (datalen % 8 != 0);
			uint32_t blocks = octets / VO_RS_K;
			fec = blocks * (VO_RS_N - VO_RS_K) + (uint32_t)vo_fec_octets_for(octets % VO_RS_K);
			if(fec == 0) status = VO_ERR_NO_FEC;
		}
		if(status == VO_BURST_OK) {
			v->datalen = datalen;
			v->requested_bits = 8 * (octets + fec);
			v->decoder_state = DS_DATA;
		} else {
			v->decoder_state = DS_IDLE;
		}
		if(c->trace) {
			vo_event e; memset(&e, 0, sizeof(e));
			e.channel = chan_idx; e.kind = VO_EV_HEADER; e.dec_index = v->dec_index;
			e.i[0] = (int32_t)raw; e.i[1] = (int32_t)v->syndrome; e.i[2] = (int32_t)datalen; e.i[3] = status;
			e.i[4] = (int32_t)v->requested_bits;
			push_event(c, &e);
		}
		return;
	}
	if(v->decoder_state != DS_DATA) return;
	vo_scramble_bits(v->bits + v->descrambled, v->nbits - v->descrambled, &v->lfsr);
	v->descrambled = v->nbits;
	static _Thread_local uint8_t fbuf[4096];
	uint32_t flens[1100], nfr = 0;
	int32_t corr = 0;
	int8_t rs_ret[9];
	cnt[VO_CNT_BURSTS]++;
	int status = vo_decode_burst_bits(v->bits + v->read_pos, v->nbits - v->read_pos, v->datalen,
			fbuf, sizeof(fbuf), flens, 1100, &nfr, &corr, rs_ret);
	for(int r = 0; r < 9; r++) {
		if(rs_ret[r] == -128) break;
		cnt[VO_CNT_BLOCKS_PROCESSED]++;
		if(rs_ret[r] >= 0) cnt[VO_CNT_BLOCKS_FEC_OK]++;
	}
	if(status != VO_BURST_OK) cnt[VO_CNT_BURST_ERR]++;
	/* frames extracted before a late error stay pushed: src/decode.c:345-369 (goto cleanup) */
	uint32_t datalen_octets = v->datalen / 8 + (v->datalen % 8 != 0);
	uint32_t off = 0;
	for(uint32_t k = 0; k < nfr; k++) {
		emit_frame(c, v, chan_idx, (int)k, fbuf + off, flens[k], datalen_octets, corr);
		off += flens[k];
	}
	if(c->trace) {
		vo_event e; memset(&e, 0, sizeof(e));
		e.channel = chan_idx; e.kind = VO_EV_BURST; e.dec_index = v->dec_index;
		e.i[0] = status; e.i[1] = (int32_t)((datalen_octets + VO_RS_K - 1) / VO_RS_K); e.i[2] = (int32_t)nfr; e.i[3] = corr;
		for(int r = 0; r < 9; r++) e.i[4 + r / 4] |= (int32_t)((uint32_t)(uint8_t)rs_ret[r] << (8 * (r % 4)));
		e.f[0] = v->frame_pwr; e.f[1] = v->mag_nf;
		push_event(c, &e);
	}
	v->burst_seq++;
	v->decoder_state = DS_IDLE;
}

/* src/demod.c:222-286 — one decimated sample */
static void demod_step(vo_ctx *c, chan_t *v, uint32_t chan_idx, float re, float im) {
	static const uint8_t gray[8] = { 0, 1, 3, 2, 6, 7, 5, 4 };
	if(v->decoder_state == DS_IDLE) reset_demod(v);
	if(v->demod_state == ST_SEARCH) {
		v->ring_pos = (v->ring_pos + 1) % VO_SYNC_BUFLEN;
		v->ring[v->ring_pos] = (float)atan2(im, re);
		if(++v->sclk < 3) return;
		v->sclk = 0;
		float mag = hypotf(re, im);
		v->mag_lp = v->mag_lp * 0.9f + mag * (1.0f - 0.9f);
		if(++v->nfcnt == 1000) {
			v->nfcnt = 0;
			v->mag_nf = 0.85f * v->mag_nf + (1.0f - 0.85f) * fminf(v->mag_lp, v->mag_nf) + 0.0001f;
		}
		if(preamble_metric(c, v, chan_idx)) {
			c->counters[chan_idx * VO_NUM_COUNTERS + VO_CNT_SYNC_GOOD]++;
			v->sync_dec_index = v->dec_index;
			v->demod_state = ST_LOCKED;
		}
		return;
	}
	if(++v->sclk < VO_SPS) return;
	v->sclk = 0;
	float phi = (float)atan2(im, re);
	float dphi = phi - v->prev_phi - v->dphi;
	if(dphi < 0) dphi += 2.0f * M_PI;
	else if(dphi > 2.0f * M_PI) dphi -= 2.0f * M_PI;
	dphi /= M_PI_4;
	int sym = (int)roundf(dphi) % 8;
	if(sym < 0) sym += 8;                            /* reference would index out of bounds; unreachable for |dphi err| < 2*pi */
	float p = re * re + im * im;
	v->frame_pwr = (v->frame_pwr * v->frame_pwr_cnt + p) / (v->frame_pwr_cnt + 1);
	v->frame_pwr_cnt++;
	v->prev_phi = phi;
	if(v->nbits + VO_BPS > VO_MAX_BURST_BITS) { reset_demod(v); return; }   /* src/demod.c:274-278 */
	for(int b = VO_BPS - 1; b >= 0; b--)                                       /* src/bitstream.c:46-56 */
		v->bits[v->nbits++] = (gray[sym] >> b) & 1u;
	if(v->nbits - v->read_pos >= v->requested_bits) burst_step(c, v, chan_idx);
}

vo_ctx *vo_create(uint32_t sample_rate, uint32_t oversample, int fmt, uint32_t centerfreq,
		const uint32_t *freqs, uint32_t n_channels, float max_ppm) {
	vo_ctx *c = calloc(1, sizeof(*c));
	c->rate = sample_rate; c->oversample = oversample; c->fmt = fmt; c->centerfreq = centerfreq;
	c->n_channels = n_channels; c->max_ppm = max_ppm;
	vo_levels_u8(c->levels);
	vo_sincos_lut(c->sin_lut, c->cos_lut);
	vo_lpf_design(sample_rate, c->A, c->B);
	vo_sync_consts(c->lr_X, &c->lr_denom, c->pr_phase);
	gf_init();
	c->ch = calloc(n_channels, sizeof(chan_t));
	c->counters = calloc((size_t)n_channels * VO_NUM_COUNTERS, sizeof(uint64_t));
	for(uint32_t k = 0; k < n_channels; k++) {                         /* src/demod.c:379-392 */
		chan_t *v = &c->ch[k];
		v->bits = calloc(VO_MAX_BURST_BITS, 1);
		v->mag_nf = 2.0f;
		v->nco_step = vo_downmix_dphi(centerfreq, freqs[k], sample_rate);
		v->mixes = centerfreq != freqs[k];
		v->freq = freqs[k];
		reset_demod(v);
	}
	return c;
}

void vo_destroy(vo_ctx *c) {
	if(!c) return;
	for(uint32_t k = 0; k < c->n_channels; k++) free(c->ch[k].bits);
	free(c->ch); free(c->sbuf); free(c->frames); free(c->arena); free(c->events); free(c->dec); free(c->state); free(c->pherr1); free(c->counters);
	free(c);
}

void vo_process(vo_ctx *c, const uint8_t *buf, uint32_t len) {
	if(len == 0) return;
	uint32_t nfloat = c->fmt == VO_FMT_S16 ? len / 2 : len;
	if(nfloat > c->sbuf_cap) { c->sbuf = realloc(c->sbuf, nfloat * sizeof(float)); c->sbuf_cap = nfloat; }
	if(c->fmt == VO_FMT_S16) {                                           /* src/demod.c:356-365 */
		const int16_t *s = (const int16_t *)buf;
		for(uint32_t i = 0; i < nfloat; i++) c->sbuf[i] = (float)s[i] / 32768.0f;
	} else {                                                             /* src/demod.c:339-347 */
		for(uint32_t i = 0; i < nfloat; i++) c->sbuf[i] = c->levels[buf[i]];
	}
	const float a0 = c->A[0], a1 = c->A[1], a2 = c->A[2], b1 = c->B[1], b2 = c->B[2];
	uint64_t dec_base = c->ch[0].dec_index;
	uint64_t dec_new = (uint64_t)((uint32_t)c->ch[0].decim_count + nfloat / 2) / c->oversample;
	if(c->tap) {
		uint64_t need = (c->dec_count + dec_new) * c->n_channels * 2;
		if(need > c->dec_cap) { c->dec_cap = 2 * need + 1024; c->dec = realloc(c->dec, c->dec_cap * sizeof(float)); }
	}
	for(uint32_t k = 0; k < c->n_channels; k++) {                       /* src/demod.c:302-329 */
		chan_t *v = &c->ch[k];
		for(uint32_t i = 0; i + 1 < nfloat; ) {      /* a trailing unpaired component is ignored */
			v->xr[2] = v->xr[1]; v->xr[1] = v->xr[0];
			v->xi[2] = v->xi[1]; v->xi[1] = v->xi[0];
			v->yr[2] = v->yr[1]; v->yr[1] = v->yr[0];
			v->yi[2] = v->yi[1]; v->yi[1] = v->yi[0];
			float re = c->sbuf[i++];
			float im = c->sbuf[i++];
			if(v->mixes) {
				uint32_t slot = v->nco_phase >> 16;                     /* src/demod.c:58-72 */
				float frac = (float)(v->nco_phase & 0xffffu) / 65536.0f;
				float s0 = c->sin_lut[slot], s1 = c->sin_lut[slot + 1];
				float sn = s0 + (s1 - s0) * frac;
				float c0 = c->cos_lut[slot], c1 = c->cos_lut[slot + 1];
				float cs = c0 + (c1 - c0) * frac;
				float mr = re * cs - im * sn;                           /* src/demod.c:200-203 */
				float mi = im * cs + re * sn;
				re = mr; im = mi;
				v->nco_phase = (v->nco_phase + v->nco_step) & 0xffffffu;
			}
			v->xr[0] = re; v->xi[0] = im;
			float r = a0 * v->xr[0];                                    /* src/demod.c:74-79 */
			r += a1 * v->xr[1] + a2 * v->xr[2];
			r += b1 * v->yr[1] + b2 * v->yr[2];
			v->yr[0] = r;
			r = a0 * v->xi[0];
			r += a1 * v->xi[1] + a2 * v->xi[2];
			r += b1 * v->yi[1] + b2 * v->yi[2];
			v->yi[0] = r;
			if(++v->decim_count == (int)c->oversample) {
				v->decim_count = 0;
				if(c->tap) {
					uint64_t n = c->dec_count + (v->dec_index - dec_base);
					c->dec[(n * c->n_channels + k) * 2 + 0] = v->yr[0];
					c->dec[(n * c->n_channels + k) * 2 + 1] = v->yi[0];
				}
				demod_step(c, v, k, v->yr[0], v->yi[0]);
				v->dec_index++;
			}
		}
	}
	if(c->tap) c->dec_count += dec_new;
}

/* the demodulator state a decimated sample meets, packed for vo_state_tap (layout in vdl2_oracle.h) */
static uint32_t pack_state(const chan_t *v) {
	return (uint32_t)v->ring_pos | ((uint32_t)(uint8_t)(int8_t)v->sclk << 8) | ((uint32_t)(v->demod_state == ST_LOCKED) << 16)
		| ((uint32_t)(v->decoder_state == DS_IDLE) << 17) | ((uint32_t)v->nfcnt << 18);
}

/* demod() of every channel on decimated samples: the sample loop of process_samples (src/demod.c:302-329) after
 * the decimation, without the front end */
void vo_process_dec(vo_ctx *c, const float *dec, uint32_t n_dec) {
	if(n_dec == 0) return;
	if(c->state_tap) {
		uint64_t need = (c->state_count + n_dec) * c->n_channels;
		if(need > c->state_cap) {
			c->state_cap = 2 * need + 1024;
			c->state = realloc(c->state, c->state_cap * sizeof(uint32_t));
			c->pherr1 = realloc(c->pherr1, c->state_cap * sizeof(float));
		}
	}
	for(uint32_t k = 0; k < c->n_channels; k++) {
		chan_t *v = &c->ch[k];
		for(uint32_t n = 0; n < n_dec; n++) {
			const float *d = &dec[((size_t)n * c->n_channels + k) * 2];
			if(c->state_tap) {
				c->state[(c->state_count + n) * c->n_channels + k] = pack_state(v);
				c->pherr1[(c->state_count + n) * c->n_channels + k] = v->pherr[1];
			}
			demod_step(c, v, k, d[0], d[1]);
			v->dec_index++;
		}
	}
	if(c->state_tap) c->state_count += n_dec;
}

uint32_t vo_num_frames(const vo_ctx *c) { return c->n_frames; }
const vo_frame *vo_frames(const vo_ctx *c) { return c->frames; }
const uint8_t *vo_frame_bytes(const vo_ctx *c) { return c->arena; }
void vo_enable_trace(vo_ctx *c, int on) { c->trace = on; }
uint32_t vo_num_events(const vo_ctx *c) { return c->n_events; }
const vo_event *vo_events(const vo_ctx *c) { return c->events; }
void vo_enable_dec_tap(vo_ctx *c, int on) { c->tap = on; }
uint64_t vo_dec_count(const vo_ctx *c) { return c->dec_count; }
const float *vo_dec_tap(const vo_ctx *c) { return c->dec; }
const uint64_t *vo_counters(const vo_ctx *c) { return c->counters; }
void vo_enable_state_tap(vo_ctx *c, int on) { c->state_tap = on; }
uint64_t vo_state_count(const vo_ctx *c) { return c->state_count; }
const uint32_t *vo_state_tap(const vo_ctx *c) { return c->state; }
const float *vo_pherr1_tap(const vo_ctx *c) { return c->pherr1; }
