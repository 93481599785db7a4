/*
 * tests/hostsim/update_receivers.cpp — TEST-ONLY host build of the functions of dumpvdl2_b200/csrc/vdl2_core.cuh that map
 * the slots of a new receiver list to the old one (vdl2gpu_update_receivers), so the CPU suite can step them as the library
 * does.
 */
#include <stdint.h>
#include "vdl2_tables_host.h"
#ifndef __CUDACC__
struct float2 { float x, y; };
#endif
#include "vdl2_core.cuh"

extern "C" {

/* slot_from[i] = vdl2_rx_slot_from of new slot i, chan_from[i] = vdl2_rx_chan_from of new channel i (-1 past n_ch), i < n_chp */
void update_slot_map(uint32_t n_chp, uint32_t lanes, uint32_t full_warps, uint32_t n_ch, const uint32_t *rx_first, uint32_t n_rx,
		const int32_t *from, uint32_t old_lanes, uint32_t old_full_warps, const uint32_t *old_first, int32_t *slot_from, int32_t *chan_from) {
	for(uint32_t i = 0; i < n_chp; i++) {
		slot_from[i] = vdl2_rx_slot_from(i, lanes, full_warps, n_ch, rx_first, n_rx, from, old_lanes, old_full_warps, old_first);
		chan_from[i] = i < n_ch ? vdl2_rx_chan_from(i, rx_first, n_rx, from, old_first) : -1;
	}
}

int update_slot_channel(uint32_t slot, uint32_t lanes, uint32_t full_warps, uint32_t n_ch, uint32_t *chan) {
	return vdl2_slot_channel(slot, lanes, full_warps, n_ch, *chan) ? 1 : 0;
}

size_t update_migrate_entry_bytes(void) { return sizeof(vdl2_rx_migrate); }

}
