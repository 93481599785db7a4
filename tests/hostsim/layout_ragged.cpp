/*
 * tests/hostsim/layout_ragged.cpp — TEST-ONLY host build of the ragged-span functions of dumpvdl2_b200/csrc/vdl2_core.cuh
 * (the per-span receiver table and the ragged K1's per-row copy sizes), so the CPU suite can step them as the library does.
 */
#include <stdint.h>
#include "vdl2_tables_host.h"
#ifndef __CUDACC__
struct float2 { float x, y; };
#endif
#include "vdl2_core.cuh"

extern "C" {

/* one span: fills out[4 * r .. 4 * r + 3] = {off, n, prev_n, dec_base} of receiver r and advances pos / prev; returns the
 * span's bytes */
uint64_t ragged_span_table(const uint32_t *oversample, const uint32_t *fmt, uint32_t n_rx, const uint32_t *n, uint64_t *pos,
		uint32_t *prev, uint64_t *out) {
	vdl2_rx_input *rx = new vdl2_rx_input[n_rx ? n_rx : 1];
	vdl2_rx_span *t = new vdl2_rx_span[n_rx ? n_rx : 1];
	vdl2_rx_span_layout(oversample, fmt, n_rx, rx);
	const uint64_t bytes = vdl2_rx_span_table(rx, n_rx, n, pos, prev, t);
	for(uint32_t r = 0; r < n_rx; r++) {
		out[4 * r] = t[r].off; out[4 * r + 1] = t[r].n; out[4 * r + 2] = t[r].prev_n; out[4 * r + 3] = t[r].dec_base;
	}
	delete[] t;
	delete[] rx;
	return bytes;
}

/* row r of the tile at group g0: out[4 * r .. 4 * r + 3] = {groups, samples, bytes, odd} */
void ragged_tile_rows(const uint32_t *n, const uint32_t *oversample, uint32_t n_rx, uint32_t g0, uint32_t TG, uint32_t *out) {
	for(uint32_t r = 0; r < n_rx; r++) {
		const vdl2_rx_tile_row t = vdl2_rx_ragged_row(n[r], g0, TG, oversample[r]);
		out[4 * r] = t.groups; out[4 * r + 1] = t.samples; out[4 * r + 2] = t.bytes; out[4 * r + 3] = t.odd;
	}
}

size_t ragged_span_entry_bytes(void) { return sizeof(vdl2_rx_span); }

}
