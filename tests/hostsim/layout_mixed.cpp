/*
 * tests/hostsim/layout_mixed.cpp — TEST-ONLY host build of the mixed-rate receiver functions of
 * dumpvdl2_b200/csrc/vdl2_core.cuh (span layout, rate classes, tile sizing of the mixed K1), so the CPU suite can check
 * what vdl2gpu_create_mixed_receivers builds and uploads.
 */
#include <stdint.h>
#include "vdl2_tables_host.h"
#ifndef __CUDACC__
struct float2 { float x, y; };
#endif
#include "vdl2_core.cuh"

extern "C" {

uint32_t layout_rx_tile_stride(uint32_t T) { return vdl2_rx_tile_stride(T); }
uint32_t layout_rx_k1_smem_bytes(uint32_t G, uint32_t T) { return vdl2_rx_k1_smem_bytes(G, T); }
uint32_t layout_rx_k1_smem_budget(void) { return VDL2_RX_K1_SMEM_BUDGET; }
uint32_t layout_rx_mixed_tile_groups(uint32_t G, uint32_t os_max) { return vdl2_rx_mixed_tile_groups(G, os_max); }
uint32_t layout_rx_mixed_smem_max(void) { return VDL2_RX_MIXED_SMEM_MAX; }
uint32_t layout_rx_class(uint32_t oversample) { return vdl2_rx_class(oversample); }

/* off[r] = byte offset of receiver r's buffer in a span of n_dec; returns the bytes per decimated sample of the span */
uint64_t layout_rx_span_offsets(const uint32_t *oversample, const uint32_t *fmt, uint32_t n_rx, uint32_t n_dec, uint64_t *off) {
	vdl2_rx_input *rx = new vdl2_rx_input[n_rx ? n_rx : 1];
	const uint64_t per_dec = vdl2_rx_span_layout(oversample, fmt, n_rx, rx);
	for(uint32_t r = 0; r < n_rx; r++) off[r] = vdl2_rx_span_offset(rx, r, n_dec);
	delete[] rx;
	return per_dec;
}

}
