/*
 * tests/hostsim/hostsim.cpp — TEST-ONLY host instantiation of the device functions in
 * dumpvdl2_b200/csrc/vdl2_core.cuh (the K2 state machine and the K3 burst decoder), compiled with g++
 * (-ffp-contract=off).  It lets the CPU test-suite step the exact source the kernels compile against the
 * oracle before any GPU time is spent.  It is NOT a fallback: nothing in the product links or loads it.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "vdl2_tables_host.h"
#ifndef __CUDACC__
struct float2 { float x, y; };
#endif
typedef float2 float2x;
#include "vdl2_core.cuh"

static const uint8_t *rootmul_table(const host_tables *h) {
	static uint8_t tab[6 * 256];
	static bool ready = false;
	if(!ready) { vdl2_rs_build_rootmul(tab, h->t.gf_exp, h->t.gf_log, 0, 1); ready = true; }
	return tab;
}
static const uint8_t *unstuff_table() {
	static uint8_t tab[VDL2_UNSTUFF_TABLE_BYTES];
	static bool ready = false;
	if(!ready) { vdl2_unstuff_build_table(tab, 0, 1); ready = true; }
	return tab;
}
/* the unstuffer twice: bit rules only, and with the octet table the kernel uses; any difference in status, frame
 * lengths or frame octets is reported as -100 by the callers */
static int g_unstuff_disagree = 0;
static void unstuff_both(vdl2_burst_work &w) {
	static vdl2_burst_work ref;
	ref = w;
	vdl2_burst_unstuff(ref);
	vdl2_burst_unstuff(w, unstuff_table());
	bool same = ref.status == w.status && ref.n_frames == w.n_frames && ref.frame_bytes == w.frame_bytes;
	for(uint32_t k = 0; same && k < w.n_frames; k++) same = ref.flen[k] == w.flen[k];
	if(same && memcmp(ref.frames, w.frames, w.frame_bytes) != 0) same = false;
	if(!same) g_unstuff_disagree++;
}
static const uint16_t *crc_table() {
	static uint16_t tab[256];
	static bool ready = false;
	if(!ready) { vdl2_crc16_build_table(tab, 0, 1); ready = true; }
	return tab;
}

/* One launch of n samples of one channel in one of the kernels' walk forms (use_pre: 0 the per-sample walk; 1 blocked on the
 * phase plane, TwoSum unwrap; 2 the same, table unwrap; 3 the ring walk, inputs requested one block ahead; 4 the staged ring
 * walk (MODE 3); 5 the default walk (MODE 4), data symbols sliced inline).  dec / phs / mgs: the channel's sample 0 of the
 * launch in the decimated, phase and magnitude planes, consecutive samples n_ch apart; phs[-k * n_ch] is valid for k <= 160. */
static void hostsim_walk_launch(int use_pre, vdl2_chan &v, float *ring, const vdl2_k2_env &env, uint32_t ch, uint64_t base, uint32_t n,
		size_t n_ch, const float2x *dec, const float *phs, const float *mgs) {
	uint32_t m = 0;
	if(use_pre == 4) {                /* the kernel's staged ring walk (MODE 3): same control flow, the cp.async copies done at once */
		float stage[2][16];
		int first_cur = 0;
		uint32_t b = 0;
		if(m + VDL2_WALK_BLOCK <= n) {
			const int f0 = vdl2_walk_first(v);
			for(int t = 0; t < VDL2_WALK_BLOCK; t++) stage[0][t] = phs[(size_t)t * n_ch];
			for(int j = 0; j < 4; j++) stage[0][12 + j] = mgs[(size_t)(f0 + VDL2_SYNC_SKIP * j) * n_ch];
			first_cur = f0;
		}
		for(; m + VDL2_WALK_BLOCK <= n; m += VDL2_WALK_BLOCK, b ^= 1u) {
			const size_t o = (size_t)m * n_ch;
			vdl2_walk_pref pf;
			for(int t = 0; t < VDL2_WALK_BLOCK; t++) pf.pw[t] = stage[b][t];
			for(int j = 0; j < 4; j++) pf.mg[j] = stage[b][12 + j];
			pf.first = first_cur; pf.valid = 1;
			if(m + 2 * VDL2_WALK_BLOCK <= n) {
				const int fn = vdl2_walk_first(v);
				const float *ph_n = phs + o + (size_t)VDL2_WALK_BLOCK * n_ch, *mg_n = mgs + o + (size_t)VDL2_WALK_BLOCK * n_ch;
				for(int t = 0; t < VDL2_WALK_BLOCK; t++) stage[b ^ 1u][t] = ph_n[(size_t)t * n_ch];
				for(int j = 0; j < 4; j++) stage[b ^ 1u][12 + j] = mg_n[(size_t)(fn + VDL2_SYNC_SKIP * j) * n_ch];
				first_cur = fn;
			}
			vdl2_walk_block_ring(v, ring, 1, env, ch, base + m, dec + o, phs + o, mgs + o, n_ch, pf, false);
		}
	} else if(use_pre == 5) {         /* the kernel's default walk (MODE 4): no magnitude plane, the four attempt magnitudes from the samples */
		for(; m + VDL2_WALK_BLOCK <= n; m += VDL2_WALK_BLOCK) {
			const size_t o = (size_t)m * n_ch;
			vdl2_walk_pref pf;
			const int first = vdl2_walk_first(v);
			for(int t = 0; t < VDL2_WALK_BLOCK; t++) pf.pw[t] = phs[o + (size_t)t * n_ch];
			for(int j = 0; j < 4; j++) {
				const float2x d = dec[o + (size_t)(first + VDL2_SYNC_SKIP * j) * n_ch];
				pf.mg[j] = vdl2_mag_of(d.x, d.y);
			}
			pf.first = first; pf.valid = 1;
			vdl2_walk_block_ring(v, ring, 1, env, ch, base + m, dec + o, phs + o, nullptr, n_ch, pf, false);
		}
	} else if(use_pre == 3) {         /* the kernel's ring walk, inputs requested one block ahead */
		vdl2_walk_pref pf;
		memset(&pf, 0, sizeof(pf));
		for(; m + VDL2_WALK_BLOCK <= n; m += VDL2_WALK_BLOCK) {
			const size_t o = (size_t)m * n_ch;
			vdl2_walk_block_ring(v, ring, 1, env, ch, base + m, dec + o, phs + o, mgs + o, n_ch, pf, m + 2 * VDL2_WALK_BLOCK <= n);
		}
	} else if(use_pre) {              /* the kernel's blocked walk on the phase plane */
		for(; m + VDL2_WALK_BLOCK <= n; m += VDL2_WALK_BLOCK) {
			const size_t o = (size_t)m * n_ch;
			if(use_pre == 2)              /* unwrap through the transition table */
				vdl2_walk_block<true>(v, ring, 1, env, ch, base + m, dec + o, phs + o, mgs + o, n_ch);
			else
				vdl2_walk_block<false>(v, ring, 1, env, ch, base + m, dec + o, phs + o, mgs + o, n_ch);
		}
	}
	for(; m < n; m++) {
		const size_t o = (size_t)m * n_ch;
		vdl2_demod_step_pm(v, ring, 1, env, ch, base + m, dec[o].x, dec[o].y, phs[o], mgs[o], false, 0.f, 0.f);
	}
}

extern "C" {

/* K1 restated on the host exactly as the scalar kernel does it (table form of the NCO) */
int hostsim_k1(const float *samples /*[n][2]*/, uint32_t n_pairs, uint32_t rate, uint32_t oversample, uint32_t centerfreq,
		const uint32_t *freqs, uint32_t n_ch, float *dec /*[n_dec][n_ch][2]*/, uint32_t *n_dec_out) {
	host_tables *h = new host_tables();
	make_tables(*h, rate);
	uint32_t n_dec = n_pairs / oversample;
	for(uint32_t ch = 0; ch < n_ch; ch++) {
		float xr1 = 0, xr2 = 0, xi1 = 0, xi2 = 0, yr1 = 0, yr2 = 0, yi1 = 0, yi2 = 0;
		uint32_t phi = 0, cnt = 0, m = 0;
		uint32_t dphi = centerfreq != freqs[ch] ? (uint32_t)(int)(((float)centerfreq - (float)freqs[ch]) / (float)rate * 256.0f * 65536.0f) : 0u;
		const float a0 = h->t.A[0], a1 = h->t.A[1], a2 = h->t.A[2], b1 = h->t.B[1], b2 = h->t.B[2];
		for(uint32_t k = 0; k < n_pairs; k++) {
			const float *e = h->t.lut[(phi >> 16) & 0xFFu];
			const float fr = (float)(phi & 0xFFFFu);
			const float cs = F_ADD(e[0], F_MUL(e[2], fr));
			const float sn = F_ADD(e[1], F_MUL(e[3], fr));
			phi += dphi;
			const float sx = samples[2 * k], sy = samples[2 * k + 1];
			const float re = F_SUB(F_MUL(sx, cs), F_MUL(sy, sn));
			const float im = F_ADD(F_MUL(sy, cs), F_MUL(sx, sn));
			float r = F_MUL(a0, re);
			r = F_ADD(r, F_ADD(F_MUL(a1, xr1), F_MUL(a2, xr2)));
			r = F_ADD(r, F_ADD(F_MUL(b1, yr1), F_MUL(b2, yr2)));
			float q = F_MUL(a0, im);
			q = F_ADD(q, F_ADD(F_MUL(a1, xi1), F_MUL(a2, xi2)));
			q = F_ADD(q, F_ADD(F_MUL(b1, yi1), F_MUL(b2, yi2)));
			xr2 = xr1; xr1 = re; yr2 = yr1; yr1 = r;
			xi2 = xi1; xi1 = im; yi2 = yi1; yi1 = q;
			if(++cnt == oversample) {
				cnt = 0;
				if(m < n_dec) { dec[((size_t)m * n_ch + ch) * 2] = r; dec[((size_t)m * n_ch + ch) * 2 + 1] = q; }
				m++;
			}
		}
	}
	*n_dec_out = n_dec;
	delete h;
	return 0;
}

/* K2 + K3 over a whole decimated stream.  Output: burst records in the device format (vdl2_burst_record +
 * frame table + frame bytes), events in vdl2_event_rec format. */
int hostsim_k2k3(const float *dec /*[n_dec][n_ch][2]*/, uint32_t n_dec, uint32_t n_ch, const uint32_t *freqs,
		uint32_t rate, float max_ppm, uint8_t *out, uint32_t out_cap, uint32_t *out_used, uint32_t *n_records,
		vdl2_event_rec *events, uint32_t event_cap, uint32_t *n_events, uint32_t *chan_counters /*[n_ch][2]: sync, hdr_good*/,
		int use_pre /* 1: consume the parallel pre-pass like K2 does; 0: always evaluate from the ring */,
		const uint32_t *launches /* launch lengths in decimated samples, repeated; nullptr: 1024 */, uint32_t n_launches) {
	host_tables *h = new host_tables();
	make_tables(*h, rate);
	const uint32_t n_slots = 3 * n_ch + 16;
	std::vector<vdl2_burst_slot> pool(n_slots);
	std::vector<int32_t> free_list(n_slots);
	std::vector<uint32_t> ready(n_slots);
	for(uint32_t i = 0; i < n_slots; i++) free_list[i] = (int32_t)i;
	vdl2_queue_ctl ctl;
	memset(&ctl, 0, sizeof(ctl));
	ctl.free_top = (int32_t)n_slots;
	vdl2_k2_env env;
	env.pr_phase = h->t.pr_phase; env.lr_X = h->t.lr_X; env.lr_denom = h->t.lr_denom; env.max_ppm = max_ppm; env.s27 = h->s27; env.unwrap_lut = h->t.unwrap_lut;
	env.pool = pool.data(); env.free_list = free_list.data(); env.ready = ready.data(); env.ctl = &ctl;
	env.events = events; env.event_cap = event_cap; env.trace = events != nullptr;
	std::vector<vdl2_chan> chans(n_ch);
	std::vector<float> rings((size_t)n_ch * VDL2_SYNC_BUFLEN, 0.f);
	for(uint32_t ch = 0; ch < n_ch; ch++) vdl2_chan_init(chans[ch], freqs[ch]);
	*out_used = 0; *n_records = 0;
	vdl2_burst_work *w = new vdl2_burst_work();
	/* the kernels process launch by launch: K2 over all channels, then K3 over the ready list.  Every launch restarts
	 * the walk with the channel state carried over, as K2 does, so each one ends in its own walk tail. */
	/* K2a emulation: phase plane with a 160-row zero history, magnitude plane */
	std::vector<float> phase((size_t)(n_dec + VDL2_SYNC_BUFLEN) * n_ch, 0.f), mag((size_t)n_dec * n_ch);
	for(uint32_t m = 0; m < n_dec; m++)
		for(uint32_t ch = 0; ch < n_ch; ch++) {
			const float *d = &dec[((size_t)m * n_ch + ch) * 2];
			phase[(size_t)(m + VDL2_SYNC_BUFLEN) * n_ch + ch] = vdl2_phase_of(d[0], d[1]);
			mag[(size_t)m * n_ch + ch] = vdl2_mag_of(d[0], d[1]);
		}
	const float2x *dec2 = reinterpret_cast<const float2x *>(dec);
	for(uint32_t base = 0, li = 0; base < n_dec; li++) {
		const uint32_t len = launches && n_launches ? launches[li % n_launches] : 1024u;
		uint32_t n = n_dec - base < len ? n_dec - base : len;
		for(uint32_t ch = 0; ch < n_ch; ch++) {
			const size_t o = (size_t)base * n_ch + ch;
			hostsim_walk_launch(use_pre, chans[ch], &rings[(size_t)ch * VDL2_SYNC_BUFLEN], env, ch, base, n, n_ch, dec2 + o,
					&phase[o + (size_t)VDL2_SYNC_BUFLEN * n_ch], &mag[o]);
		}
		for(uint32_t b = 0; b < ctl.n_ready; b++) {
			const vdl2_burst_slot *slot = &pool[ready[b]];
			vdl2_burst_geometry(*w, slot->datalen_bits, slot->nbits);
			memset(w->tab, 0, sizeof(w->tab));
			if(w->status == VDL2_BURST_OK) {
				vdl2_burst_unpack(*w, slot->words, h->t.lfsr_words, 0, 1);
				for(uint32_t r = 0; r < w->num_blocks; r++) {
					int nfec = (r == w->num_blocks - 1) ? (int)w->last_fec : 6;
					w->rs_ret[r] = vdl2_rs_verify(w->tab[r], nfec, h->t.gf_exp, h->t.gf_log, rootmul_table(h));
				}
				for(uint32_t r = 0; r < w->num_blocks; r++) {
					int nfec = (r == w->num_blocks - 1) ? (int)w->last_fec : 6;
					int ret = w->rs_ret[r];
					if(ret < 0) { w->status = VDL2_ERR_FEC_BAD; for(uint32_t q = r + 1; q < w->num_blocks; q++) w->rs_ret[q] = -128; break; }
					if(ret > 0) w->fec_corr += ret - (6 - nfec);
				}
				if(w->status == VDL2_BURST_OK) unstuff_both(*w);
				uint32_t off = 0;
				for(uint32_t k = 0; k < w->n_frames; k++) { w->fcrc[k] = vdl2_crc16_tab(&w->frames[off], w->flen[k], crc_table()); off += w->flen[k]; }
			}
			uint32_t rec_bytes = (uint32_t)((sizeof(vdl2_burst_record) + 4u * w->n_frames + w->frame_bytes + 15u) & ~15u);
			if(*out_used + rec_bytes > out_cap) { delete w; delete h; return -1; }
			vdl2_burst_record r;
			memset(&r, 0, sizeof(r));
			r.rec_bytes = rec_bytes; r.channel = slot->channel; r.burst_seq = slot->burst_seq; r.status = w->status;
			r.n_frames = w->n_frames; r.datalen_bits = slot->datalen_bits; r.syndrome = slot->syndrome;
			r.num_fec_corrections = w->fec_corr; r.frame_pwr = slot->frame_pwr; r.mag_nf = slot->mag_nf; r.ppm_error = slot->ppm_error;
			r.num_blocks = w->num_blocks; r.sync_lo = slot->sync_lo; r.sync_hi = slot->sync_hi; r.freq = slot->freq; r.frame_bytes = w->frame_bytes;
			for(int q = 0; q < 12; q++) r.rs_ret[q] = (int8_t)w->rs_ret[q];
			uint8_t *dst = out + *out_used;
			memset(dst, 0, rec_bytes);
			memcpy(dst, &r, sizeof(r));
			uint32_t *tab = (uint32_t *)(dst + sizeof(r));
			for(uint32_t k = 0; k < w->n_frames; k++) tab[k] = (uint32_t)w->flen[k] | ((uint32_t)w->fcrc[k] << 16);
			memcpy(tab + w->n_frames, w->frames, w->frame_bytes);
			*out_used += rec_bytes; (*n_records)++;
			free_list[ctl.free_top++] = (int32_t)ready[b];
		}
		ctl.n_ready = 0;
		base += n;
	}
	for(uint32_t ch = 0; ch < n_ch; ch++) { chan_counters[2 * ch] = chans[ch].cnt_sync; chan_counters[2 * ch + 1] = chans[ch].cnt_hdr_good; }
	*n_events = ctl.n_events < event_cap ? ctl.n_events : event_cap;
	int ovf = (int)ctl.pool_overflows;
	delete w; delete h;
	if(g_unstuff_disagree) return -100;
	return ovf;
}

/* K3 alone: `bits` = the burst after the preamble (header + payload + FEC, scrambled, one bit per byte) */
int hostsim_k3(const uint8_t *bits, uint32_t nbits, uint32_t datalen_bits, uint8_t *frames_out, uint32_t cap, uint32_t *lens,
		uint16_t *crcs, uint32_t max_frames, uint32_t *n_frames, int32_t *fec_corr, int8_t *rs_ret9) {
	static host_tables *h = nullptr;
	if(!h) { h = new host_tables(); make_tables(*h, 2100000); }
	static vdl2_burst_slot slot;
	static vdl2_burst_work w;
	memset(&slot, 0, sizeof(slot));
	for(uint32_t i = 0; i < nbits && i < VDL2_MAX_BURST_BITS; i++) slot.words[i >> 5] |= (uint32_t)(bits[i] & 1u) << (31u - (i & 31u));
	vdl2_burst_geometry(w, datalen_bits, nbits);
	memset(w.tab, 0, sizeof(w.tab));
	if(w.status == VDL2_BURST_OK) {
		vdl2_burst_unpack(w, slot.words, h->t.lfsr_words, 0, 1);
		for(uint32_t r = 0; r < w.num_blocks; r++)
			w.rs_ret[r] = vdl2_rs_verify(w.tab[r], (r == w.num_blocks - 1) ? (int)w.last_fec : 6, h->t.gf_exp, h->t.gf_log, rootmul_table(h));
		for(uint32_t r = 0; r < w.num_blocks; r++) {
			int nfec = (r == w.num_blocks - 1) ? (int)w.last_fec : 6;
			if(w.rs_ret[r] < 0) { w.status = VDL2_ERR_FEC_BAD; for(uint32_t q = r + 1; q < w.num_blocks; q++) w.rs_ret[q] = -128; break; }
			if(w.rs_ret[r] > 0) w.fec_corr += w.rs_ret[r] - (6 - nfec);
		}
		if(w.status == VDL2_BURST_OK) unstuff_both(w);
	}
	if(g_unstuff_disagree) return -100;
	*n_frames = w.n_frames; *fec_corr = w.fec_corr;
	for(int r = 0; r < 9; r++) rs_ret9[r] = (int8_t)w.rs_ret[r];
	uint32_t off = 0;
	for(uint32_t k = 0; k < w.n_frames && k < max_frames; k++) {
		if(off + w.flen[k] > cap) return -1;
		memcpy(frames_out + off, w.frames + off, w.flen[k]);
		lens[k] = w.flen[k]; crcs[k] = vdl2_crc16_tab(w.frames + off, w.flen[k], crc_table());
		off += w.flen[k];
	}
	return w.status;
}

/* stand-alone pieces for unit tests */
int hostsim_rs_verify(uint8_t *block255, int fec_octets) {
	static host_tables *h = nullptr;
	if(!h) { h = new host_tables(); memset(h, 0, sizeof(*h)); make_gf(h->t); }
	return vdl2_rs_verify(block255, fec_octets, h->t.gf_exp, h->t.gf_log, rootmul_table(h));
}
/* the warp-cooperative form K3 runs (vdl2_kernels.cu: k3_rs_block), with the 32 lanes emulated by a loop: syndromes
 * as the XOR of the lanes' partial sums, Chien search as the lanes' position masks merged in position order */
int hostsim_rs_verify_lanes(uint8_t *block255, int fec_octets) {
	static host_tables *h = nullptr;
	if(!h) { h = new host_tables(); memset(h, 0, sizeof(*h)); make_gf(h->t); }
	if(fec_octets == 0) return 0;
	uint64_t acc = 0;
	for(uint32_t lane = 0; lane < 32; lane++) acc ^= vdl2_rs_syndrome_partial(block255, lane, h->t.gf_exp, h->t.gf_log, rootmul_table(h));
	if(acc == 0) return 0;
	uint8_t S[6], lambda[7];
	for(int i = 0; i < 6; i++) S[i] = (uint8_t)(acc >> (8 * i));
	const int deg = vdl2_rs_locator(S, fec_octets, h->t.gf_exp, h->t.gf_log, lambda);
	uint32_t masks[32];
	for(uint32_t lane = 0; lane < 32; lane++) masks[lane] = vdl2_rs_chien_lane(lambda, deg, lane, h->t.gf_exp, h->t.gf_log);
	int root[256], count = 0;
	for(uint32_t k = 0; k < 8; k++)
		for(uint32_t lane = 0; lane < 32; lane++)
			if(masks[lane] & (1u << k)) root[count++] = (int)(lane + 1u + 32u * k);
	if(deg != count) return -1;
	return vdl2_rs_forney(block255, S, lambda, deg, root, count, h->t.gf_exp, h->t.gf_log);
}
uint32_t hostsim_header_fix(uint32_t word, uint32_t *syndrome) {
	uint32_t s = vdl2_header_syndrome(word);
	*syndrome = s;
	return word ^ vdl2_header_error_pattern(s);
}
uint32_t hostsim_synd_weight(uint32_t s) { return vdl2_synd_weight(s); }
float hostsim_unwrap_step(float unwrap, float step) { return vdl2_unwrap_step(unwrap, step); }
int hostsim_unwrap_lut(uint32_t *out /*[VDL2_UNWRAP_STATES * 6]*/) {
	vdl2_tables *t = new vdl2_tables();
	int n = make_unwrap_lut(*t);
	memcpy(out, t->unwrap_lut, sizeof(t->unwrap_lut));
	delete t;
	return n;
}
float hostsim_unwrap_lut_step(const uint32_t *lut, uint32_t *row, float step) { return vdl2_unwrap_lut_step(lut, *row, step); }
uint16_t hostsim_crc16(const uint8_t *p, uint32_t n) { return vdl2_crc16(p, n); }
void hostsim_tables(uint32_t rate, float *levels, float *sin_lut, float *cos_lut, float *A, float *B, float *lr_X, float *lr_denom, float *pr_phase) {
	host_tables *h = new host_tables();
	make_tables(*h, rate);
	memcpy(levels, h->t.levels, sizeof(h->t.levels)); memcpy(sin_lut, h->sin_lut, sizeof(h->sin_lut)); memcpy(cos_lut, h->cos_lut, sizeof(h->cos_lut));
	memcpy(A, h->t.A, 12); memcpy(B, h->t.B, 12); memcpy(lr_X, h->t.lr_X, 64); *lr_denom = h->t.lr_denom; memcpy(pr_phase, h->t.pr_phase, 64);
	delete h;
}

}
