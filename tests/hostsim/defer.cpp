/*
 * tests/hostsim/defer.cpp — TEST-ONLY host walk of the K2 default walk (MODE 4) of dumpvdl2_b200/csrc/vdl2_core.cuh in its
 * two forms: data symbols sliced inline, and sliced after the walk (vdl2_defer), as k2_sync_slice<128, true, 4> and
 * k2_sync_slice_ragged do.  Built on hostsim.cpp (its tables); nothing in the product links or loads it.
 */
#include <algorithm>
#include "hostsim.cpp"

/* the kernel's default walk (MODE 4) over one launch of one channel: no magnitude plane, the four attempt magnitudes from
 * the samples; `defer`: data symbols sliced after the walk (vdl2_defer), as k2_sync_slice<128, true, 4> does.  dec and phase
 * point at the channel's sample 0 of the launch, consecutive samples n_ch apart.  stats (defer only, may be null): [0..11]
 * bursts ending on each block offset with the walk going on, [12] ending in the per-sample tail, [13] queued, [14] sliced
 * at once (queue taken), [15] without a pool slot, [16] open bursts completed on a launch's last sample, [17] bursts
 * ending on a launch's last sample but one, [18] open bursts whose last symbol is the next launch's first sample, [19]
 * launches with two burst ends or more walked past, [20] with three or more */
#define DEFER_STATS 23
static void walk_default(vdl2_chan &v, float *ring, const vdl2_k2_env &env, uint32_t ch, uint64_t base, uint32_t n, uint32_t n_ch,
		const float2 *dec, const float *phase, bool defer, uint64_t *stats) {
	vdl2_defer d;
	vdl2_defer_init(d);
	uint32_t m = 0;
	int ends = 0;
	auto count_end = [&](int k) {
		if(!stats) return;
		stats[k]++;
		if(d.last == (int)n - 2) stats[17]++;
		ends++;
		if(v.slot < 0) stats[15]++;
		else stats[d.q_at < 0 ? 13 : 14]++;
	};
	for(; m + VDL2_WALK_BLOCK <= n; m += VDL2_WALK_BLOCK) {
		const size_t o = (size_t)m * n_ch;
		if(defer) {
			vdl2_defer_enter(d, v, (int)m);
			if(d.at >= 0 && d.last < (int)m + VDL2_WALK_BLOCK && d.last + 1 < (int)n) count_end(d.last - (int)m);
			if(vdl2_defer_block<false>(d, v, ring, 1, env, ch, base + m, (int)m, (int)n, dec + o, phase + o, n_ch, dec, phase, n_ch))
				continue;
		}
		vdl2_walk_pref pf;
		const int first = vdl2_walk_first(v);
		for(int t = 0; t < VDL2_WALK_BLOCK; t++) pf.pw[t] = phase[o + (size_t)t * n_ch];
		for(int j = 0; j < 4; j++) {
			const float2 dj = dec[o + (size_t)(first + VDL2_SYNC_SKIP * j) * n_ch];
			pf.mg[j] = vdl2_mag_of(dj.x, dj.y);
		}
		pf.first = first; pf.valid = 1;
		vdl2_walk_block_ring(v, ring, 1, env, ch, base + m, dec + o, phase + o, nullptr, n_ch, pf, false);
	}
	for(; m < n; m++) {
		if(defer) {
			vdl2_defer_enter(d, v, (int)m);
			if(d.at >= 0 && d.last + 1 < (int)n) count_end(12);
			const int next = vdl2_defer_sample(d, v, env, ch, (int)m, (int)n, dec, phase, n_ch);
			if(next >= 0) { m = (uint32_t)next - 1u; continue; }
		}
		const size_t o = (size_t)m * n_ch;
		vdl2_demod_step_pm(v, ring, 1, env, ch, base + m, dec[o].x, dec[o].y, phase[o], vdl2_mag_of(dec[o].x, dec[o].y), false, 0.f, 0.f);
	}
	if(defer) {
		if(stats && d.at >= 0 && d.last == (int)n - 1) stats[16]++;
		if(stats && d.at >= 0 && d.last == (int)n) stats[18]++;
		if(stats && ends >= 2) stats[19]++;
		if(stats && ends >= 3) stats[20]++;
		vdl2_defer_finish(d, v, env, ch, dec, phase, n_ch, (int)n);
	}
}

/* K2 state of a whole context for hostsim_k2_defer_check */
struct k2_sim {
	std::vector<vdl2_burst_slot> pool;
	std::vector<int32_t> free_list;
	std::vector<uint32_t> ready;
	std::vector<vdl2_event_rec> events;
	vdl2_queue_ctl ctl;
	vdl2_k2_env env;
	std::vector<vdl2_chan> chans;
	std::vector<float> rings;
	k2_sim(const host_tables *h, uint32_t n_ch, const uint32_t *freqs, uint32_t n_slots, float max_ppm, uint32_t event_cap)
		: pool(n_slots), free_list(n_slots), ready(n_slots), events(event_cap), chans(n_ch), rings((size_t)n_ch * VDL2_SYNC_BUFLEN, 0.f) {
		memset(pool.data(), 0, sizeof(vdl2_burst_slot) * n_slots);
		memset(events.data(), 0, sizeof(vdl2_event_rec) * event_cap);
		for(uint32_t i = 0; i < n_slots; i++) free_list[i] = (int32_t)i;
		memset(&ctl, 0, sizeof(ctl));
		ctl.free_top = (int32_t)n_slots;
		env.pr_phase = h->t.pr_phase; env.lr_X = h->t.lr_X; env.lr_denom = h->t.lr_denom; env.max_ppm = max_ppm; env.s27 = h->s27;
		env.unwrap_lut = h->t.unwrap_lut; env.pool = pool.data(); env.free_list = free_list.data(); env.ready = ready.data();
		env.ctl = &ctl; env.events = events.data(); env.event_cap = event_cap; env.trace = 1;
		for(uint32_t ch = 0; ch < n_ch; ch++) vdl2_chan_init(chans[ch], freqs[ch]);
	}
};

static bool chan_equal(const vdl2_chan &a, const vdl2_chan &b) {
#define EQF(f) (memcmp(&a.f, &b.f, sizeof(a.f)) == 0)
	return EQF(prev_phi) && EQF(prev_dphi) && EQF(dphi) && EQF(pherr0) && EQF(pherr1) && EQF(pherr2) && EQF(ppm_error) && EQF(mag_lp)
		&& EQF(mag_nf) && EQF(frame_pwr) && EQF(ring_pos) && EQF(sclk) && EQF(nfcnt) && EQF(frame_pwr_cnt) && EQF(state) && EQF(acc)
		&& EQF(nbits) && EQF(need_bits) && EQF(datalen) && EQF(syndrome) && EQF(slot) && EQF(burst_seq) && EQF(sync_dec_index)
		&& EQF(freq) && EQF(cnt_sync) && EQF(cnt_hdr_good) && EQF(pure_run);
#undef EQF
}

/* The default walk twice over one decimated stream fed span by span, channel ch taking counts[span * n_ch + ch] samples
 * (0 included) from where it stands: data symbols sliced inline (as the one-warp variant does) and sliced after the walk
 * (vdl2_defer).  After every span every field of every channel, the rings, the whole pool, the free list, the queue
 * counters, the events and the set of ready slots must be equal; then both return the ready slots to the pool in slot
 * order (as K3 would, in some order).  Returns -1 when they always were, else the index of the first span that differs
 * (*bad_ch: its first differing channel, or -1 when the difference is elsewhere).  stats: DEFER_STATS counters, see
 * walk_default, and [21] channels inside a burst's data given an empty span, [22] given a one-sample span. */
static int defer_check(const float *dec /*[n_dec][n_ch][2]*/, uint32_t n_dec, uint32_t n_ch, const uint32_t *freqs, uint32_t rate,
		float max_ppm, uint32_t n_slots, const uint32_t *counts, uint32_t n_spans, uint64_t *stats, int32_t *bad_ch) {
	host_tables *h = new host_tables();
	make_tables(*h, rate);
	const uint32_t event_cap = 1u << 18;
	k2_sim *a = new k2_sim(h, n_ch, freqs, n_slots, max_ppm, event_cap), *b = new k2_sim(h, n_ch, freqs, n_slots, max_ppm, event_cap);
	std::vector<float> phase((size_t)(n_dec + VDL2_SYNC_BUFLEN) * n_ch, 0.f);
	for(uint32_t m = 0; m < n_dec; m++)
		for(uint32_t ch = 0; ch < n_ch; ch++)
			phase[(size_t)(m + VDL2_SYNC_BUFLEN) * n_ch + ch] = vdl2_phase_of(dec[((size_t)m * n_ch + ch) * 2], dec[((size_t)m * n_ch + ch) * 2 + 1]);
	const float2 *dec2 = reinterpret_cast<const float2 *>(dec);
	memset(stats, 0, DEFER_STATS * sizeof(uint64_t));
	*bad_ch = -1;
	int bad = -1;
	std::vector<uint32_t> pos(n_ch, 0u);
	for(uint32_t li = 0; li < n_spans && bad < 0; li++) {
		const uint32_t *cnt = counts + (size_t)li * n_ch;
		for(uint32_t ch = 0; ch < n_ch; ch++) {
			const vdl2_chan &v = b->chans[ch];
			if((v.state & VDL2_ST_LOCKED) && vdl2_dec_state(v) == VDL2_DEC_DATA) {
				if(cnt[ch] == 0) stats[21]++;
				if(cnt[ch] == 1) stats[22]++;
			}
		}
		for(int k = 0; k < 2; k++) {
			k2_sim &S = k ? *b : *a;
			for(uint32_t ch = 0; ch < n_ch; ch++)
				walk_default(S.chans[ch], &S.rings[(size_t)ch * VDL2_SYNC_BUFLEN], S.env, ch, pos[ch], cnt[ch], n_ch, dec2 + (size_t)pos[ch] * n_ch + ch,
						&phase[((size_t)pos[ch] + VDL2_SYNC_BUFLEN) * n_ch + ch], k == 1, k ? stats : nullptr);
		}
		for(uint32_t ch = 0; ch < n_ch; ch++) pos[ch] += cnt[ch];
		for(uint32_t ch = 0; ch < n_ch && bad < 0; ch++)
			if(!chan_equal(a->chans[ch], b->chans[ch])
					|| memcmp(&a->rings[(size_t)ch * VDL2_SYNC_BUFLEN], &b->rings[(size_t)ch * VDL2_SYNC_BUFLEN], VDL2_SYNC_BUFLEN * sizeof(float))) {
				bad = (int)li;
				*bad_ch = (int32_t)ch;
			}
		std::sort(a->ready.begin(), a->ready.begin() + a->ctl.n_ready);
		std::sort(b->ready.begin(), b->ready.begin() + b->ctl.n_ready);
		if(bad < 0 && (memcmp(&a->ctl, &b->ctl, sizeof(a->ctl)) || memcmp(a->pool.data(), b->pool.data(), sizeof(vdl2_burst_slot) * n_slots)
				|| memcmp(a->free_list.data(), b->free_list.data(), sizeof(int32_t) * n_slots)
				|| memcmp(a->ready.data(), b->ready.data(), sizeof(uint32_t) * a->ctl.n_ready)
				|| memcmp(a->events.data(), b->events.data(), sizeof(vdl2_event_rec) * (a->ctl.n_events < event_cap ? a->ctl.n_events : event_cap))))
			bad = (int)li;
		for(k2_sim *S : {a, b}) {
			for(uint32_t r = 0; r < S->ctl.n_ready; r++) S->free_list[S->ctl.free_top++] = (int32_t)S->ready[r];
			S->ctl.n_ready = 0;
		}
	}
	delete a; delete b; delete h;
	return bad;
}

extern "C" {

/* defer_check with every channel on one launch schedule: launch lengths launches[0..n_launches), repeated, up to n_dec;
 * returns the first launch that differs */
int hostsim_k2_defer_check(const float *dec /*[n_dec][n_ch][2]*/, uint32_t n_dec, uint32_t n_ch, const uint32_t *freqs, uint32_t rate,
		float max_ppm, uint32_t n_slots, const uint32_t *launches, uint32_t n_launches, uint64_t *stats, int32_t *bad_ch) {
	std::vector<uint32_t> counts;
	for(uint32_t base = 0, li = 0; base < n_dec; li++) {
		const uint32_t len = launches[li % n_launches];
		const uint32_t n = n_dec - base < len ? n_dec - base : len;
		counts.insert(counts.end(), n_ch, n);
		base += n;
	}
	return defer_check(dec, n_dec, n_ch, freqs, rate, max_ppm, n_slots, counts.data(), (uint32_t)(counts.size() / n_ch), stats, bad_ch);
}

/* defer_check on per-channel spans: counts [n_spans][n_ch], each channel's counts summing to at most n_dec */
int hostsim_k2_defer_check_spans(const float *dec, uint32_t n_dec, uint32_t n_ch, const uint32_t *freqs, uint32_t rate, float max_ppm,
		uint32_t n_slots, const uint32_t *counts, uint32_t n_spans, uint64_t *stats, int32_t *bad_ch) {
	std::vector<uint64_t> sum(n_ch, 0);
	for(uint32_t li = 0; li < n_spans; li++)
		for(uint32_t ch = 0; ch < n_ch; ch++) sum[ch] += counts[(size_t)li * n_ch + ch];
	for(uint32_t ch = 0; ch < n_ch; ch++)
		if(sum[ch] > n_dec) return -2;
	return defer_check(dec, n_dec, n_ch, freqs, rate, max_ppm, n_slots, counts, n_spans, stats, bad_ch);
}

}
