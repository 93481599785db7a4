/*
 * tests/hostsim/layout.cpp — TEST-ONLY host build of the channel-layout functions of
 * dumpvdl2_b200/csrc/vdl2_core.cuh (slot -> channel -> receiver, receivers per K1 block, tile geometry of the
 * receiver-group K1), so the CPU suite can check the tables the multi-receiver context uploads.
 */
#include <stdint.h>
#include "vdl2_tables_host.h"
#ifndef __CUDACC__
struct float2 { float x, y; };
#endif
#include "vdl2_core.cuh"

extern "C" {

int layout_slot_channel(uint32_t slot, uint32_t lanes, uint32_t full_warps, uint32_t n_ch, uint32_t *chan) {
	return vdl2_slot_channel(slot, lanes, full_warps, n_ch, *chan) ? 1 : 0;
}

uint32_t layout_rx_of_channel(uint32_t chan, const uint32_t *rx_first, uint32_t n_rx) { return vdl2_rx_of_channel(chan, rx_first, n_rx); }

uint32_t layout_rx_tables(uint32_t n_blocks, uint32_t lanes, uint32_t full_warps, uint32_t n_ch, const uint32_t *rx_first, uint32_t n_rx,
		uint32_t *slot_rx, uint32_t *block_rx) {
	return vdl2_rx_layout(n_blocks, lanes, full_warps, n_ch, rx_first, n_rx, slot_rx, block_rx);
}

uint32_t layout_rx_tile_samples(uint32_t G, uint32_t oversample) { return vdl2_rx_tile_samples(G, oversample); }
uint32_t layout_rx_tile_stride(uint32_t T) { return vdl2_rx_tile_stride(T); }
uint32_t layout_rx_k1_smem_bytes(uint32_t G, uint32_t T) { return vdl2_rx_k1_smem_bytes(G, T); }
uint32_t layout_rx_k1_smem_budget(void) { return VDL2_RX_K1_SMEM_BUDGET; }

}
