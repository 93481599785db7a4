/*
 * tests/hostsim/k2_state.cpp — TEST-ONLY host reference of the state a K2 launch leaves behind, for a whole stage of
 * channels: every K2_* field in the plane encoding of vdl2_chan_store, the syncbuf rings, the burst pool, the ready list,
 * the queue counters and the phase history the next launch starts from.  Each launch walks every channel in one of the
 * walk forms of the kernels (hostsim.cpp, defer.cpp); the simplest, the per-sample vdl2_demod_step_pm, is the reference.
 * Also restates the device layout of a stage (vdl2gpu_stage_create) against vdl2_types.h, so that the tests can read
 * the planes of a stage straight from its device memory.  Nothing in the product links or loads it.
 */
#include "defer.cpp"
#include "vdl2gpu.h"

/* walk forms: 0-5 hostsim_walk_launch's use_pre (0 the per-sample walk, 5 the default walk with data symbols sliced
 * inline), 6 the default walk with data symbols sliced after the walk (vdl2_defer) */
#define K2_STATE_DEFERRED 6

struct k2_state {
	host_tables *h;
	k2_sim *S;
	const float2x *dec;                      /* [n_dec][n_ch], the caller's */
	std::vector<float> phase, mag;           /* [160 + n_dec][n_ch] (160 rows of zero history), [n_dec][n_ch] */
	std::vector<uint32_t> pos;               /* per channel: samples walked */
	uint32_t n_dec, n_ch, n_slots;
	int form;
};

static void k2_state_recycle(k2_state *K) {
	/* K3 gives every ready slot back to the free list, in some order: here in slot order, so that every form pops the same
	 * slots in the next launch whatever order its ready list was filled in */
	k2_sim &S = *K->S;
	std::sort(S.ready.begin(), S.ready.begin() + S.ctl.n_ready);
	for(uint32_t r = 0; r < S.ctl.n_ready; r++) S.free_list[S.ctl.free_top++] = (int32_t)S.ready[r];
	S.ctl.n_ready = 0;
}

extern "C" {

void *k2_state_open(const float *dec /*[n_dec][n_ch][2]*/, uint32_t n_dec, uint32_t n_ch, const uint32_t *freqs, uint32_t rate,
		float max_ppm, uint32_t n_slots, int form, int trace) {
	if(form < 0 || form > K2_STATE_DEFERRED) return nullptr;
	k2_state *K = new k2_state();
	K->h = new host_tables();
	make_tables(*K->h, rate);
	K->S = new k2_sim(K->h, n_ch, freqs, n_slots, max_ppm, 1u << 18);
	K->S->env.trace = trace ? 1u : 0u;
	K->dec = reinterpret_cast<const float2x *>(dec);
	K->n_dec = n_dec; K->n_ch = n_ch; K->n_slots = n_slots; K->form = form;
	K->pos.assign(n_ch, 0u);
	K->phase.assign((size_t)(n_dec + VDL2_SYNC_BUFLEN) * n_ch, 0.f);
	K->mag.assign((size_t)n_dec * n_ch, 0.f);
	for(size_t i = 0; i < (size_t)n_dec * n_ch; i++) {
		K->phase[(size_t)VDL2_SYNC_BUFLEN * n_ch + i] = vdl2_phase_of(K->dec[i].x, K->dec[i].y);
		K->mag[i] = vdl2_mag_of(K->dec[i].x, K->dec[i].y);
	}
	return K;
}

/* One launch: the previous launch's ready slots go back to the free list (as K3 gives them back), then channel ch walks
 * the next counts[ch] samples of its stream (counts == nullptr: every channel n).  Returns -1 when a count runs past the
 * stream. */
int k2_state_step(void *hk, const uint32_t *counts, uint32_t n) {
	k2_state *K = static_cast<k2_state *>(hk);
	k2_sim &S = *K->S;
	const size_t n_ch = K->n_ch;
	for(uint32_t ch = 0; ch < K->n_ch; ch++)
		if(K->pos[ch] + (counts ? counts[ch] : n) > K->n_dec) return -1;
	k2_state_recycle(K);
	for(uint32_t ch = 0; ch < K->n_ch; ch++) {
		const uint32_t c = counts ? counts[ch] : n, base = K->pos[ch];
		const size_t o = (size_t)base * n_ch + ch;
		float *ring = &S.rings[(size_t)ch * VDL2_SYNC_BUFLEN];
		const float *phs = &K->phase[o + (size_t)VDL2_SYNC_BUFLEN * n_ch];
		if(K->form == K2_STATE_DEFERRED)
			walk_default(S.chans[ch], ring, S.env, ch, base, c, K->n_ch, K->dec + o, phs, true, nullptr);
		else
			hostsim_walk_launch(K->form, S.chans[ch], ring, S.env, ch, base, c, n_ch, K->dec + o, phs, &K->mag[o]);
		K->pos[ch] += c;
	}
	return 0;
}

/* the state after the last launch, laid out as on the device with a row stride of n_ch: k2 [K2_NFIELDS][n_ch]
 * (vdl2_chan_store), ring [160][n_ch], hist [160][n_ch] the 160 phases before each channel's next sample (the phase
 * plane's history rows), ctl the queue counters */
void k2_state_read(void *hk, uint32_t *k2, float *ring, float *hist, vdl2_queue_ctl *ctl) {
	k2_state *K = static_cast<k2_state *>(hk);
	const size_t n_ch = K->n_ch;
	for(uint32_t ch = 0; ch < K->n_ch; ch++) {
		vdl2_chan_store(K->S->chans[ch], k2, n_ch, ch);
		for(int i = 0; i < VDL2_SYNC_BUFLEN; i++) {
			ring[(size_t)i * n_ch + ch] = K->S->rings[(size_t)ch * VDL2_SYNC_BUFLEN + i];
			hist[(size_t)i * n_ch + ch] = K->phase[((size_t)K->pos[ch] + i) * n_ch + ch];
		}
	}
	*ctl = K->S->ctl;
}

/* the ready list of the last launch, in slot order (a launch fills it in any order): copies of the slots */
uint32_t k2_state_ready(void *hk, vdl2_burst_slot *out, uint32_t cap) {
	k2_state *K = static_cast<k2_state *>(hk);
	k2_sim &S = *K->S;
	std::sort(S.ready.begin(), S.ready.begin() + S.ctl.n_ready);
	for(uint32_t r = 0; r < S.ctl.n_ready && r < cap; r++) out[r] = S.pool[S.ready[r]];
	return S.ctl.n_ready;
}

/* a copy of one pool slot (an open burst's words written so far) */
int k2_state_slot(void *hk, int32_t slot, vdl2_burst_slot *out) {
	k2_state *K = static_cast<k2_state *>(hk);
	if(slot < 0 || (uint32_t)slot >= K->n_slots) return -1;
	*out = K->S->pool[slot];
	return 0;
}

/* phase rows [row0, row0 + n_rows) of the stream with its 160 rows of zero history in front, [n_rows][n_ch] */
void k2_state_phase_rows(void *hk, uint32_t row0, uint32_t n_rows, float *out) {
	k2_state *K = static_cast<k2_state *>(hk);
	memcpy(out, &K->phase[(size_t)row0 * K->n_ch], (size_t)n_rows * K->n_ch * sizeof(float));
}

void k2_state_close(void *hk) {
	k2_state *K = static_cast<k2_state *>(hk);
	delete K->S; delete K->h; delete K;
}

/* sizes the tests parse with: sizeof(vdl2_burst_slot), offsetof(words), K2_NFIELDS, sizeof(vdl2_queue_ctl) */
void k2_state_sizes(uint32_t *out) {
	out[0] = (uint32_t)sizeof(vdl2_burst_slot); out[1] = (uint32_t)offsetof(vdl2_burst_slot, words);
	out[2] = K2_NFIELDS; out[3] = (uint32_t)sizeof(vdl2_queue_ctl);
}

/* The device memory of a stage (vdl2gpu_stage_create), restated: byte offsets of tab, k1, k2, counters, ring, phase, mag,
 * hist_tmp, pool, free_list, ready, ctl, events, and the total (off[13]); each part 256-byte aligned, n_ch rounded up to
 * 32 rows, max(256, 3 n_ch) pool slots, 2^18 events with VDL2GPU_FLAG_TRACE and 1 without.  Returns the pool's slot count. */
uint32_t k2_state_stage_layout(uint32_t n_ch, uint32_t max_dec, uint32_t flags, uint64_t *off) {
	auto al = [](size_t x) { return (x + 255u) & ~(size_t)255u; };
	const size_t n_chp = (n_ch + 31u) & ~31u, n_slots = 3u * n_ch > 256u ? 3u * n_ch : 256u;
	const size_t event_cap = (flags & VDL2GPU_FLAG_TRACE) ? (1u << 18) : 1u;
	const size_t part[13] = {
		sizeof(vdl2_tables), (size_t)K1_NFIELDS * n_chp * 4, (size_t)K2_NFIELDS * n_chp * 4, (size_t)VDL2_NUM_COUNTERS * n_chp * 4,
		(size_t)VDL2_SYNC_BUFLEN * n_chp * 4, (size_t)(max_dec + VDL2_SYNC_BUFLEN) * n_chp * 4, (size_t)max_dec * n_chp * 4,
		(size_t)VDL2_SYNC_BUFLEN * n_chp * 4, n_slots * sizeof(vdl2_burst_slot), n_slots * 4, n_slots * 4, sizeof(vdl2_queue_ctl),
		event_cap * sizeof(vdl2gpu_event) };
	size_t o = 0;
	for(int k = 0; k < 13; k++) { off[k] = o; o += al(part[k]); }
	off[13] = o;
	return (uint32_t)n_slots;
}

}
