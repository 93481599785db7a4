/*
 * tests/hostsim/oracle_noise_floor.c — TEST-ONLY: the oracle (oracle/vdl2_oracle.c, compiled unchanged inside this translation
 * unit) plus one reader of what its channel records keep private, every channel's noise-floor filters as they stand now
 * (src/demod.c:238-243).  The channel-level tests compare the device's mag_lp / mag_nf with these.
 */
#include "../../oracle/vdl2_oracle.c"

/* out[k][0] = mag_lp, out[k][1] = mag_nf of channel k (out: [n_channels][2]) */
void vo_noise_floor(const vo_ctx *c, float *out) {
	for(uint32_t k = 0; k < c->n_channels; k++) { out[2 * k] = c->ch[k].mag_lp; out[2 * k + 1] = c->ch[k].mag_nf; }
}
