/* vdl2_kernels.h — kernel parameter blocks and launch prototypes (internal to libvdl2gpu.so). */
#ifndef VDL2_KERNELS_H
#define VDL2_KERNELS_H
#include <stdint.h>
#include <cuda_runtime.h>
#include "vdl2_types.h"

/* Per-chunk values that change from one chunk to the next.  The host writes one of these into pinned memory and the
 * first node of the chunk's CUDA graph copies it to the device, so the captured kernel nodes never need new
 * parameters: kernels given a non-NULL `ca` take these fields from it instead of from their parameter block. */
typedef struct {
	const void *raw;             /* K0 input (device pointer) */
	uint64_t dec_base;           /* absolute index of the chunk's first decimated sample */
	uint32_t n_pairs;            /* complex samples per stream in this chunk */
	uint32_t cnt0;               /* decimation counter on entry */
	uint32_t n_dec;              /* decimated samples this chunk produces */
	uint32_t prev_n_dec;         /* ... and the previous chunk produced (its last 160 phase rows are this chunk's history) */
} vdl2_chunk_args;

/* optional per-block scheduling trace (VDL2GPU_BLOCK_TRACE=1): every block of K1 and K2 appends one record */
typedef struct {
	uint32_t kernel;             /* 1 = K1, 2 = K2 */
	uint32_t block;
	uint32_t smid;
	uint32_t pad;
	uint64_t t_start, t_end;     /* %globaltimer, ns */
} vdl2_block_rec;
typedef struct {
	uint32_t n, cap;
	vdl2_block_rec rec[1];
} vdl2_block_trace;

typedef struct {
	const float2 *samples;       /* K0 output: {re, im} per complex sample; stream s at samples + s * stream_stride */
	uint32_t n_pairs;
	uint32_t oversample;
	uint32_t cnt0;               /* decimation counter on entry (src/demod.c:289,322), same for all channels */
	uint32_t n_ch, n_chp;        /* channels; per-channel array stride = channel SLOTS (n_chp >= n_ch, multiple of 32) */
	uint32_t lanes;              /* channels per warp (1..32) for the first `full_warps` warps, lanes - 1 for the others: the
	                              * channels are dealt out evenly so that the warps of the channel kernels cover every SM
	                              * sub-partition and all live equally long (see create_impl in vdl2_host.cu) */
	uint32_t full_warps;
	float2 *dec;                 /* [n_dec][n_chp] */
	uint32_t *state;             /* [K1_NFIELDS][n_chp] */
	const float4 *lut;           /* 257 x {cos, sin, dcos*2^-16, dsin*2^-16} */
	float a0, a1, a2, b1, b2;
	float one, neg_one, two;     /* run-time 1.0f / -1.0f / 2.0f (see k1_mix_iir_decimate_packed) */
	uint32_t ch_per_stream;      /* independent-streams mode: channels [s*C, (s+1)*C) read stream s; 0 = one stream for all;
	                              * 1 = one stream per channel: `samples` is float2[n_pairs][stream_stride], time-major across streams */
	uint32_t stream_stride;      /* float2 elements between consecutive streams in `samples` (ch_per_stream == 1: per sample row) */
	const vdl2_chunk_args *ca;   /* NULL, or device pointer overriding n_pairs / cnt0 */
	vdl2_block_trace *trace_blocks;
	/* multi-receiver context (vdl2gpu_create_receivers; NULL otherwise): `samples` is float2[n_rx][stream_stride], receiver-major;
	 * slot_rx[slot] = receiver of the slot's channel, block_rx[2 b] / [2 b + 1] = first receiver / number of receivers of
	 * 128-slot block b (vdl2_rx_layout); every tile stages rx_tile samples of each of them, at most rx_max per block */
	const uint32_t *slot_rx;
	const uint32_t *block_rx;
	uint32_t rx_tile, rx_max;
	/* mixed-rate receivers (vdl2gpu_create_mixed_receivers; NULL otherwise): n_pairs (or ca->n_pairs) counts DECIMATED
	 * samples per receiver, receiver r has rx_in[r].oversample x n_pairs samples in its row; slot_cls[slot] = rate class
	 * (vdl2_rx_class) of the slot's receiver, cls_taps[k] = {a0, a1, a2, b1, b2} of class k, cls_mask = the classes present;
	 * every tile stages rx_tile decimation groups of each receiver, rows of vdl2_rx_tile_stride(rx_tile x rx_os_max) */
	const vdl2_rx_input *rx_in;
	const uint8_t *slot_cls;
	float cls_taps[3][5];
	uint32_t cls_mask, rx_os_max;
	/* ragged spans (VDL2GPU_FLAG_RAGGED; NULL otherwise): the span's receiver table (vdl2_rx_span_table); receiver r's row
	 * holds rx_span[r].n x os_r samples, and n_pairs (or ca->n_pairs) is the span's width, the largest n */
	const vdl2_rx_span *rx_span;
	/* ragged spans that restart receivers (vdl2gpu_restart_receiver; NULL on every other span): per slot, whether its
	 * channel starts afresh with this span and its new NCO step (vdl2_rx_restart) */
	const vdl2_rx_restart *rx_restart;
} vdl2_k1_params;

typedef struct {
	const float2 *dec;
	float *phase;                /* [160 + n_dec][n_chp]: rows 0..159 = last 160 phases of the previous chunks */
	float *mag;                  /* [n_dec][n_chp] */
	float *hist_tmp;             /* [160][n_chp] scratch for the history shift of short chunks */
	uint32_t n_dec;
	uint32_t n_ch, n_chp;
	uint32_t lanes, full_warps;  /* channel slot mapping, as in vdl2_k1_params */
	uint64_t dec_base;           /* absolute index of dec[0] */
	uint32_t *state;             /* [K2_NFIELDS][n_chp] */
	float *ring;                 /* [160][n_chp] */
	const vdl2_tables *tables;
	float max_ppm;
	uint32_t s27;
	vdl2_burst_slot *pool;
	int32_t *free_list;
	uint32_t *ready;
	vdl2_queue_ctl *ctl;
	void *events;
	uint32_t event_cap;
	uint32_t trace;
	uint32_t variant;            /* walk variant, see vdl2_launch_k2 */
	uint32_t k2a_mode;           /* 0: libdevice atan2 for every sample; 1: vdl2_phase_fast with the Ziv fall-back */
	const vdl2_chunk_args *ca;   /* NULL, or device pointer overriding n_dec / dec_base */
	vdl2_block_trace *trace_blocks;
	/* ragged spans (NULL otherwise): a lane walks rx_span[slot_rx[slot]].n samples from index rx_span[...].dec_base */
	const uint32_t *slot_rx;
	const vdl2_rx_span *rx_span;
	/* (NULL unless the span restarts receivers) per slot: start the demodulator afresh on frequency rx_restart[slot].freq */
	const vdl2_rx_restart *rx_restart;
} vdl2_k2_params;

/* K2a in its resident form (k2a_phase_mag_warps): warp w computes phase and magnitude of slots [32 w, 32 w + 32) for every
 * decimated sample of the chunk and first carries the last 160 phase rows of the previous chunk's plane over */
typedef struct {
	const float2 *dec;           /* [n_dec][n_chp] */
	float *phase;                /* this chunk's plane [160 + n_dec][n_chp] */
	float *mag;                  /* [n_dec][n_chp], or NULL: the walk (variant 5) takes the magnitudes from the samples itself */
	const float *phase_prev;     /* the previous chunk's plane (the other of the two) */
	uint32_t n_dec, prev_n_dec;
	uint32_t n_ch, n_chp, lanes, full_warps;
	uint32_t mode;               /* 0 libdevice atan2 / IEEE sqrt for every sample, 1 the Ziv-guarded short forms */
	uint32_t split;              /* time slices per chunk: the grid is `split` x (one block per 128 slots) */
	const vdl2_chunk_args *ca;
	/* ragged spans (NULL otherwise): a lane's rows are rx_span[slot_rx[slot]].n, its history the previous plane's rows
	 * [prev_n, prev_n + 160) */
	const uint32_t *slot_rx;
	const vdl2_rx_span *rx_span;
	/* (NULL unless the span restarts receivers) per slot: zero history rows instead of the previous plane's */
	const vdl2_rx_restart *rx_restart;
	/* channel levels (VDL2GPU_FLAG_CHANNEL_LEVELS; NULL otherwise): uint64 [VDL2_CHLV_ROWS][n_chp] then the uint32 peak plane
	 * [n_chp], which the levels form adds every sample it evaluates to (vdl2_core.cuh) */
	uint64_t *chlv;
} vdl2_k2a_params;

typedef struct {
	vdl2_burst_slot *pool;
	int32_t *free_list;
	const uint32_t *ready;
	vdl2_queue_ctl *ctl;
	const vdl2_tables *tables;
	uint8_t *out;                /* device address of the mapped pinned output region (header + records) */
	uint32_t out_cap;            /* bytes available for records */
	uint32_t n_chp;
	uint32_t *counters;          /* [VDL2_NUM_COUNTERS][n_chp] */
	uint32_t abandoned;          /* the ready list may hold slots given up by a restart (VDL2_READY_ABANDONED) */
} vdl2_k3_params;

/* receivers joining and leaving (k_migrate_receivers): the new per-channel planes (stride n_chp) from the old ones (stride
 * old_n_chp), entry i of `map` for slot i and channel i */
typedef struct {
	const vdl2_rx_migrate *map;  /* [n_chp] */
	uint32_t n_chp, old_n_chp;
	const uint32_t *old_k1, *old_k2, *old_counters;
	const float *old_ring;
	const float *old_phase;      /* the old plane the next span would have taken its history rows from */
	uint32_t *k1, *k2, *counters;
	float *ring, *phase;         /* phase: the new plane the next span takes its history rows from */
	const uint64_t *old_chlv;    /* channel levels planes by slot (vdl2_k2a_params.chlv), or NULL */
	uint64_t *chlv;
} vdl2_migrate_params;

#ifdef __cplusplus
extern "C" {
#endif
/* once per device (thread-safe): the shared-memory carve-out every kernel of the chain asks for */
int vdl2_kernels_init_device(int device);
/* Every K0 launcher takes lv: NULL, or the per-input accumulators (vdl2_levels, one per stream or receiver) that the levels
 * form of the kernel adds the chunk's samples to (VDL2GPU_FLAG_INPUT_LEVELS) */
/* n_streams streams of n_pairs samples each: raw stream s at raw + s * raw_stride bytes, output at out2 + s * out_stride float2 */
int vdl2_launch_k0(const void *raw, uint32_t n_pairs, uint32_t fmt, const float *levels, float *out2, uint32_t n_streams,
		uint32_t raw_stride, uint32_t out_stride, const vdl2_chunk_args *ca, vdl2_levels *lv, cudaStream_t st);
/* one stream per channel: raw[s][i] -> out2[i][out_stride] float2, time-major across streams */
int vdl2_launch_k0_lanes(const void *raw, uint32_t n_pairs, uint32_t fmt, const float *levels, float *out2, uint32_t n_streams,
		uint32_t raw_stride, uint32_t out_stride, uint32_t lanes, uint32_t full_warps, const vdl2_chunk_args *ca, vdl2_levels *lv, cudaStream_t st);
/* one row per receiver: row r converts its samples, in format rx[r].fmt, into out2 + r x out_stride float2.  The row
 * source is the first of these that applies:
 *   pushed spans (ring given): span[r].n x rx[r].oversample samples from receiver r's ring (raw + ring[r].base), starting at
 *     ring offset span[r].off and wrapping at ring[r].cap;
 *   ragged spans (span given): span[r].n x rx[r].oversample samples from raw + span[r].off;
 *   mixed-rate receivers: width x rx[r].oversample samples from raw + width x rx[r].off_per_dec.
 * width: the largest span[r].n, or the mixed span's decimated samples (sizes the grid).  When ca is given, mixed and
 * ragged rows take raw from ca->raw, and mixed rows their decimated samples from ca->n_pairs. */
typedef struct {
	const void *raw;             /* the span's bytes, or (pushed spans) the receivers' rings */
	const vdl2_rx_input *rx;
	const vdl2_rx_span *span;    /* ragged and pushed spans, else NULL */
	const vdl2_rx_ring *ring;    /* pushed spans, else NULL */
} vdl2_k0_rows;
int vdl2_launch_k0_rows(const vdl2_k0_rows *r, uint32_t width, uint32_t n_rx, uint32_t os_max, const float *levels, float *out2,
		uint32_t out_stride, const vdl2_chunk_args *ca, vdl2_levels *lv, cudaStream_t st);
int vdl2_launch_k1(const vdl2_k1_params *p, int force_scalar, int variant, cudaStream_t st);
int vdl2_launch_copy_hist(const vdl2_k2_params *p, cudaStream_t st);
int vdl2_launch_k2a(const vdl2_k2_params *p, cudaStream_t st);
int vdl2_launch_k2a_warps(const vdl2_k2a_params *p, cudaStream_t st);
int vdl2_launch_k2(const vdl2_k2_params *p, cudaStream_t st);
int vdl2_launch_k3(const vdl2_k3_params *p, uint32_t grid, cudaStream_t st);
int vdl2_launch_k4(const uint8_t *frames, const uint32_t *offsets, const uint32_t *lens, uint32_t n, uint16_t *out, cudaStream_t st);
int vdl2_launch_rs(uint8_t *blocks, const int32_t *fec_octets, uint32_t n, int32_t *ret, const vdl2_tables *tables, cudaStream_t st);
int vdl2_launch_migrate(const vdl2_migrate_params *p, cudaStream_t st);
/* Spectrum (VDL2GPU_FLAG_SPECTRUM): n_in inputs of the sample plane, input i bringing span[i].n samples after span[i].pend
 * held in acc[i].carry (vdl2_core.cuh).  Input i's sample t is samples[i x stride + t] (row layouts), or, with lanes != 0
 * (one stream per channel, time-major), samples[t x stride + slot of i].  width: the most samples any input brings (sizes
 * the grid). */
int vdl2_launch_spectrum(const float *samples, uint32_t width, uint32_t n_in, uint32_t stride, uint32_t lanes, uint32_t full_warps,
		const vdl2_spec_span *span, const vdl2_spec_tab *tab, vdl2_spec_acc *acc, cudaStream_t st);
#ifdef __cplusplus
}
#endif
#endif
