/*
 * tests/hostsim/push_rings.cpp — TEST-ONLY host build of the pushed-input ring arithmetic of dumpvdl2_b200/csrc/vdl2_core.cuh
 * (ring layout, free room, the pieces of a write or read across the wrap, a span's take and table, the timestamp anchor),
 * so the CPU suite can step it as the library does.
 */
#include <stdint.h>
#include "vdl2_tables_host.h"
#ifndef __CUDACC__
struct float2 { float x, y; };
#endif
#include "vdl2_core.cuh"

static void inputs(const uint32_t *oversample, const uint32_t *fmt, uint32_t n_rx, vdl2_rx_input *rx) {
	vdl2_rx_span_layout(oversample, fmt, n_rx, rx);
}

extern "C" {

/* every receiver's ring: base[r], cap[r]; returns the bytes of the ring buffer */
uint64_t push_ring_layout(const uint32_t *oversample, const uint32_t *fmt, uint32_t n_rx, uint32_t max_chunk_bytes, uint32_t max_span,
		uint64_t *base, uint64_t *cap) {
	vdl2_rx_input *rx = new vdl2_rx_input[n_rx ? n_rx : 1];
	vdl2_rx_ring *rg = new vdl2_rx_ring[n_rx ? n_rx : 1];
	inputs(oversample, fmt, n_rx, rx);
	const uint64_t total = vdl2_push_ring_layout(rx, n_rx, max_chunk_bytes, max_span, rg);
	for(uint32_t r = 0; r < n_rx; r++) { base[r] = rg[r].base; cap[r] = rg[r].cap; }
	delete[] rg;
	delete[] rx;
	return total;
}

uint64_t push_room(uint64_t cap, uint64_t head, uint64_t freed) { return vdl2_push_room(cap, head, freed); }

/* out = {off0, len0, off1, len1} */
void push_segments(uint64_t cap, uint64_t pos, uint64_t len, uint64_t *out) {
	const vdl2_ring_segs s = vdl2_ring_segments(cap, pos, len);
	out[0] = s.off[0]; out[1] = s.len[0]; out[2] = s.off[1]; out[3] = s.len[1];
}

uint32_t push_take(uint64_t head, uint64_t tail, uint32_t group_bytes, uint32_t max_span) { return vdl2_push_take(head, tail, group_bytes, max_span); }

uint64_t push_realign(uint64_t head, uint32_t bpp) { return vdl2_push_realign(head, bpp); }

/* one pushed span: out[4 * r .. 4 * r + 3] = {off, n, prev_n, dec_base}; advances tail, pos, prev */
void push_span_table(const uint32_t *oversample, const uint32_t *fmt, const uint64_t *cap, uint32_t n_rx, const uint32_t *n, uint64_t *tail,
		uint64_t *pos, uint32_t *prev, uint64_t *out) {
	vdl2_rx_input *rx = new vdl2_rx_input[n_rx ? n_rx : 1];
	vdl2_rx_ring *rg = new vdl2_rx_ring[n_rx ? n_rx : 1];
	vdl2_rx_span *t = new vdl2_rx_span[n_rx ? n_rx : 1];
	inputs(oversample, fmt, n_rx, rx);
	for(uint32_t r = 0; r < n_rx; r++) { rg[r].base = 0; rg[r].cap = cap[r]; }
	vdl2_push_span_table(rx, rg, n_rx, n, tail, pos, prev, t);
	for(uint32_t r = 0; r < n_rx; r++) {
		out[4 * r] = t[r].off; out[4 * r + 1] = t[r].n; out[4 * r + 2] = t[r].prev_n; out[4 * r + 3] = t[r].dec_base;
	}
	delete[] t;
	delete[] rg;
	delete[] rx;
}

uint64_t push_sync_end(uint64_t sync, uint64_t dec_base, uint64_t byte_base, uint32_t group_bytes) {
	return vdl2_push_sync_end(sync, dec_base, byte_base, group_bytes);
}

double push_back_seconds(uint64_t sample_end, uint64_t push_end, uint32_t bpp, uint32_t rate) {
	return vdl2_push_back_seconds(sample_end, push_end, bpp, rate);
}

}
