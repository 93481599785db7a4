/*
 * tests/hostsim/restart.cpp — TEST-ONLY host walk of the K2 state machine and the K3 burst decoder of
 * dumpvdl2_b200/csrc/vdl2_core.cuh with receiver restarts (vdl2gpu_restart_receiver) applied at given cuts, through the
 * same restart rule the ragged K2 applies (vdl2_chan_restart) and the same treatment of abandoned burst-pool slots as the
 * K3 that runs on restart spans.  Built on hostsim.cpp (its tables and burst-decoder helpers); nothing in the product
 * links or loads it.
 */
#include "hostsim.cpp"

extern "C" {

/* K2 + K3 over one receiver's decimated stream dec[n_dec][n_ch], restarted at each of cuts[0..n_cuts) (ascending decimated
 * sample indices; equal cuts restart twice): segment k (between cut k-1 and cut k) runs on freqs[k * n_ch ..].  The walk
 * goes chunk by chunk as the kernels do - chunks end at every cut and every 1024 samples; K2 restarts the channels at the
 * start of the chunk, K3 then works through the chunk's ready list.  Outputs as hostsim_k2k3, plus pool[0] = slots in the
 * pool, pool[1] = free-list entries at the end, pool[2] = slots still held by channels in a burst, pool[3] = abandoned
 * slots K3 put back.  Returns the pool overflows (or -1 when `out` is too small, -100 on an unstuffer disagreement). */
int hostsim_restart_k2k3(const float *dec, uint32_t n_dec, uint32_t n_ch, const uint32_t *freqs, const uint32_t *cuts, uint32_t n_cuts,
		uint32_t rate, uint8_t *out, uint32_t out_cap, uint32_t *out_used, uint32_t *n_records, vdl2_event_rec *events,
		uint32_t event_cap, uint32_t *n_events, uint32_t *chan_counters /*[n_ch][2]*/, uint32_t *pool_out /*[4]*/) {
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
	env.pr_phase = h->t.pr_phase; env.lr_X = h->t.lr_X; env.lr_denom = h->t.lr_denom; env.max_ppm = 0.f; env.s27 = h->s27; env.unwrap_lut = h->t.unwrap_lut;
	env.pool = pool.data(); env.free_list = free_list.data(); env.ready = ready.data(); env.ctl = &ctl;
	env.events = events; env.event_cap = event_cap; env.trace = events != nullptr;
	std::vector<vdl2_chan> chans(n_ch);
	std::vector<float> rings((size_t)n_ch * VDL2_SYNC_BUFLEN, 0.f);
	for(uint32_t ch = 0; ch < n_ch; ch++) vdl2_chan_init(chans[ch], freqs[ch]);
	*out_used = 0; *n_records = 0;
	uint32_t abandoned = 0;
	vdl2_burst_work *w = new vdl2_burst_work();
	uint32_t seg = 0;
	for(uint32_t base = 0; base < n_dec;) {
		/* restarts due at the start of this chunk (the ragged K2's load, vdl2_kernels.cu: k2_sync_body) */
		while(seg < n_cuts && cuts[seg] == base) {
			seg++;
			for(uint32_t ch = 0; ch < n_ch; ch++) {
				vdl2_chan_restart(chans[ch], env, freqs[(size_t)seg * n_ch + ch]);
				for(int i = 0; i < VDL2_SYNC_BUFLEN; i++) rings[(size_t)ch * VDL2_SYNC_BUFLEN + i] = 0.f;
			}
		}
		uint32_t end = base + 1024 < n_dec ? base + 1024 : n_dec;
		if(seg < n_cuts && cuts[seg] < end) end = cuts[seg];
		for(uint32_t ch = 0; ch < n_ch; ch++)
			for(uint32_t m = base; m < end; m++) {
				const float *d = &dec[((size_t)m * n_ch + ch) * 2];
				vdl2_demod_step_pm(chans[ch], &rings[(size_t)ch * VDL2_SYNC_BUFLEN], 1, env, ch, m, d[0], d[1],
						vdl2_phase_of(d[0], d[1]), vdl2_mag_of(d[0], d[1]), false, 0.f, 0.f);
			}
		/* K3 over the chunk's ready list (k3_burst_fec_abandoned) */
		for(uint32_t b = 0; b < ctl.n_ready; b++) {
			if(ready[b] & VDL2_READY_ABANDONED) {
				free_list[ctl.free_top++] = (int32_t)(ready[b] & ~VDL2_READY_ABANDONED);
				abandoned++;
				continue;
			}
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
		base = end;
	}
	uint32_t held = 0;
	for(uint32_t ch = 0; ch < n_ch; ch++) {
		chan_counters[2 * ch] = chans[ch].cnt_sync; chan_counters[2 * ch + 1] = chans[ch].cnt_hdr_good;
		held += chans[ch].slot >= 0;
	}
	pool_out[0] = n_slots; pool_out[1] = (uint32_t)ctl.free_top; pool_out[2] = held; pool_out[3] = abandoned;
	*n_events = ctl.n_events < event_cap ? ctl.n_events : event_cap;
	int ovf = (int)ctl.pool_overflows;
	delete w; delete h;
	if(g_unstuff_disagree) return -100;
	return ovf;
}

/* the K1 and K2 state create gives a channel (initial_state) and a restart gives it (vdl2_k1_fresh, vdl2_chan_restart):
 * k1[K1_NFIELDS], k2[K2_NFIELDS] of one channel; `restart_from` non-NULL: the K2 fields of a channel in that state
 * restarted, with its pool slot (if any) handed to a scratch ready list */
void hostsim_fresh_state(uint32_t centerfreq, uint32_t freq, uint32_t rate, const uint32_t *restart_from, uint32_t *k1, uint32_t *k2,
		uint32_t *ready_out /*[1]*/, uint32_t *n_ready_out) {
	vdl2_k1_fresh(k1, 1, 0, vdl2_nco_dphi(centerfreq, freq, rate));
	vdl2_chan v;
	vdl2_chan_init(v, freq);
	if(restart_from) {
		/* the planes' fields back into a vdl2_chan (the order of k2_sync_body's load) */
		const uint32_t *s = restart_from;
		union { uint32_t u; float f; } b;
#define LDF(F, X) do { b.u = s[F]; X = b.f; } while(0)
		LDF(K2_PREV_PHI, v.prev_phi); LDF(K2_PREV_DPHI, v.prev_dphi); LDF(K2_DPHI, v.dphi); LDF(K2_PHERR0, v.pherr0);
		LDF(K2_PHERR1, v.pherr1); LDF(K2_PHERR2, v.pherr2); LDF(K2_PPM, v.ppm_error); LDF(K2_MAG_LP, v.mag_lp);
		LDF(K2_MAG_NF, v.mag_nf); LDF(K2_FRAME_PWR, v.frame_pwr);
#undef LDF
		v.ring_pos = (int32_t)s[K2_RING_POS]; v.sclk = (int32_t)s[K2_SCLK]; v.nfcnt = (int32_t)s[K2_NFCNT];
		v.frame_pwr_cnt = (int32_t)s[K2_FRAME_PWR_CNT]; v.state = s[K2_STATE];
		v.acc = (uint64_t)s[K2_ACC_LO] | ((uint64_t)s[K2_ACC_HI] << 32); v.nbits = s[K2_NBITS]; v.need_bits = s[K2_NEED_BITS];
		v.datalen = s[K2_DATALEN]; v.syndrome = s[K2_SYNDROME]; v.slot = (int32_t)s[K2_SLOT]; v.burst_seq = s[K2_BURST_SEQ];
		v.sync_dec_index = (uint64_t)s[K2_SYNC_LO] | ((uint64_t)s[K2_SYNC_HI] << 32); v.freq = s[K2_FREQ];
		v.cnt_sync = s[K2_CNT_SYNC]; v.cnt_hdr_good = s[K2_CNT_HDR_GOOD]; v.pure_run = s[K2_PURE_RUN];
		vdl2_queue_ctl ctl;
		memset(&ctl, 0, sizeof(ctl));
		vdl2_k2_env env;
		memset(&env, 0, sizeof(env));
		env.ready = ready_out; env.ctl = &ctl;
		vdl2_chan_restart(v, env, freq);
		*n_ready_out = ctl.n_ready;
	}
	vdl2_chan_store(v, k2, 1, 0);
}

size_t hostsim_restart_entry_bytes(void) { return sizeof(vdl2_rx_restart); }

}
