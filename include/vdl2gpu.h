/*
 * include/vdl2gpu.h — C-ABI of libvdl2gpu.so: the H100 (sm_90a) implementation of dumpvdl2's
 * per-channel DSP hot path (reference src/demod.c + src/decode.c burst part + src/chebyshev.c +
 * src/rs.c + src/libfec + the src/bitstream.c helpers).
 *
 * Plain C: pointers and sizes only, no CUDA or torch types (a cudaStream_t travels as void*).
 * Every entry point returns 0 on success or a negative VDL2GPU_E* code; the library never calls
 * exit().  There is NO CPU fallback: without a CUDA device every call that needs one fails with
 * VDL2GPU_ENODEV.
 *
 * Two front doors (INTEGRATION.md shows the reference-side binding for both):
 *
 *  (1) batch API (this file): one context = one IQ stream fanned out to N channels.  It replaces, as a
 *      unit, what the reference spreads over
 *        process_buf_uchar/process_buf_short   (src/demod.c:339-365)    -> vdl2gpu_submit
 *        N x process_samples threads + barriers (src/demod.c:288-337)   -> kernels K0-K3 on a stream
 *        decode_vdl2_burst -> avlc_decoder_queue_push (src/decode.c:165-194,196-384) -> vdl2gpu_poll/flush callback
 *
 *  (2) drop-in symbols (include/vdl2_dropin.h): the exact names/signatures of src/dumpvdl2.h:371-389 so
 *      that the unmodified front-ends and main() of the reference link against this library.
 */
#ifndef VDL2GPU_H
#define VDL2GPU_H
#include <stddef.h>
#include <stdint.h>
#include <sys/time.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VDL2GPU_ABI_VERSION 2

/* error codes */
enum {
	VDL2GPU_OK = 0,
	VDL2GPU_EINVAL = -1,      /* bad argument */
	VDL2GPU_ENODEV = -2,      /* no usable CUDA device / extension not usable */
	VDL2GPU_ECUDA = -3,       /* CUDA runtime error (vdl2gpu_last_error() has the text) */
	VDL2GPU_ENOMEM = -4,
	VDL2GPU_ETOOBIG = -5,     /* chunk larger than max_chunk_bytes */
	VDL2GPU_EOVERFLOW = -6    /* an internal device queue overflowed; bursts were dropped (see stats) */
};

/* sample formats: reference enum sample_formats (src/dumpvdl2.h:319) */
enum { VDL2GPU_FMT_U8 = 0, VDL2GPU_FMT_S16_LE = 1 };

/* config flags */
enum {
	VDL2GPU_FLAG_TRACE = 1u << 0,        /* record sync/header/burst events (debug, parity tests) */
	VDL2GPU_FLAG_KEEP_DEC = 1u << 1,     /* keep the decimated samples of the last chunk readable (parity tests) */
	VDL2GPU_FLAG_K1_SCALAR = 1u << 2,    /* use the plain per-sample K1 kernel instead of the pipelined one */
	VDL2GPU_FLAG_NO_OVERLAP = 1u << 3,   /* one stream: do not run K0/K1 of chunk c+1 beside K2/K3 of chunk c (profiling) */
	VDL2GPU_FLAG_NO_GRAPH = 1u << 4,     /* launch every kernel individually instead of replaying the per-chunk CUDA graphs */
	VDL2GPU_FLAG_RAGGED = 1u << 5,       /* vdl2gpu_create_mixed_receivers only: every receiver brings its own number of decimated
	                                      * samples to a span (vdl2gpu_submit_ragged); every other create function refuses it */
	VDL2GPU_FLAG_INPUT_LEVELS = 1u << 6, /* measure every input's levels on the device (vdl2gpu_get_input_levels); any create function */
	VDL2GPU_FLAG_CHANNEL_LEVELS = 1u << 7, /* measure every channel's in-band levels on the device (vdl2gpu_get_channel_levels); any
	                                       * create function */
	VDL2GPU_FLAG_SPECTRUM = 1u << 8      /* measure every input's power spectrum on the device (vdl2gpu_get_spectrum); any create
	                                      * function */
};

typedef struct {
	uint32_t sample_rate;        /* Hz; must equal 105000 * oversample (src/dumpvdl2.c:1073) */
	uint32_t oversample;         /* src/dumpvdl2.h:348 */
	uint32_t sample_fmt;         /* VDL2GPU_FMT_* */
	uint32_t centerfreq;         /* Hz */
	uint32_t n_channels;
	const uint32_t *freqs;       /* n_channels channel frequencies, Hz (src/demod.c:379-392) */
	float max_ppm;               /* Config.max_ppm (src/demod.c:192); 0 = off */
	uint32_t max_chunk_bytes;    /* largest len ever passed to submit; 0 = 1 MiB */
	int32_t device;              /* CUDA device ordinal; -1 = current device */
	uint32_t flags;              /* VDL2GPU_FLAG_* */
	uint32_t n_inflight;         /* chunks in flight before submit blocks (back-pressure); 0 = 4 */
	uint32_t n_streams;          /* independent IQ streams (0 = 1).  With S > 1 the n_channels = S x C channels are split
	                              * stream-major: channels [s*C, (s+1)*C) demodulate stream s; C must be a multiple of 32,
	                              * or 1 (one stream per channel: every channel reads its own IQ buffer, as every
	                              * channel thread of the reference does, src/demod.c:302-310) */
	uint32_t reserved[4];
} vdl2gpu_config;

/* One AVLC frame with the metadata the reference attaches in decode_frame (src/decode.c:173-194,
 * struct vdl2_msg_metadata src/output-common.h:31-43).  `data` is valid only during the callback. */
typedef struct {
	uint32_t channel;            /* index into freqs[] */
	uint32_t freq;
	uint32_t burst_seq;          /* per-channel count of bursts that reached the data stage */
	int32_t idx;                 /* frame number within the burst (metadata->idx) */
	const uint8_t *data;         /* frame octets, FCS included, flags excluded */
	uint32_t len;
	uint32_t synd_weight;
	uint32_t datalen_octets;
	int32_t num_fec_corrections;
	float frame_pwr_dbfs, nf_pwr_dbfs, ppm_error;
	float frame_pwr, mag_nf;     /* the raw values the two dBFS figures derive from */
	uint64_t sync_dec_index;     /* decimated-sample index at which preamble sync was declared */
	struct timeval burst_timestamp; /* chunk arrival time + sample offset (the reference calls gettimeofday at sync) */
	uint16_t fcs_residue;        /* crc16 over the frame; 0xF0B8 = good (src/avlc.c:40,177-179) */
	uint16_t fcs_ok;             /* len >= 11 && residue good */
} vdl2gpu_frame;

typedef void (*vdl2gpu_frame_cb)(const vdl2gpu_frame *frame, void *user);

/* per-context counters; names follow the reference's statsd counters (src/statsd.c:33-64) */
typedef struct {
	uint64_t chunks_submitted, chunks_completed;
	uint64_t iq_samples;                 /* complex samples accepted (per stream; a mixed-receivers context: of all receivers; ragged
	                                      * spans: the complex samples actually submitted, sum over r of n_r x oversample_r) */
	uint64_t dec_samples;                /* decimated samples produced per channel (ragged spans: the sum of the span widths, the
	                                      * largest n_r of each span; vdl2gpu_get_receiver_positions has each receiver's count) */
	uint64_t demod_sync_good;            /* demod.sync.good */
	uint64_t decoder_crc_good;           /* decoder.crc.good (header syndrome 0) */
	uint64_t bursts;                     /* bursts that reached DEC_DATA */
	uint64_t burst_errors;               /* bursts dropped in DEC_DATA (any decoder.errors.*) */
	uint64_t blocks_processed, blocks_fec_ok;
	uint64_t msg_good;                   /* decoder.msg.good = frames pushed */
	uint64_t fcs_good, fcs_bad;          /* avlc.frames.good / avlc.errors.bad_fcs (len >= 11 only) */
	uint64_t pool_overflows;             /* bursts lost because the device burst pool was exhausted (must be 0) */
	uint64_t out_overflows;              /* bursts lost because the output region was exhausted (must be 0) */
	uint64_t kernel_launches;            /* kernels launched by this context so far */
	uint64_t out_bytes;                  /* burst-record bytes K3 wrote to host memory (device->host traffic) */
	uint64_t graph_launches;             /* CUDA graph replays (3 per chunk of the nominal shape; 0 with VDL2GPU_FLAG_NO_GRAPH) */
	uint64_t reserved[2];
} vdl2gpu_stats;

/* trace event (VDL2GPU_FLAG_TRACE): same layout as the oracle's vo_event */
typedef struct {
	uint32_t channel, kind;      /* kind: 1 sync, 2 header, 3 burst */
	uint64_t dec_index;
	int32_t i[8];
	float f[8];
} vdl2gpu_event;

typedef struct vdl2gpu_ctx vdl2gpu_ctx;

/* ---- life cycle ---- */
int vdl2gpu_abi_version(void);
int vdl2gpu_device_count(void);
int vdl2gpu_create(const vdl2gpu_config *cfg, vdl2gpu_ctx **out);
/* Many receivers in one context: receiver r has its own tuning and its own channels, exactly as if it were one reference
 * process (vdl2_channel_init(rx[r].centerfreq, freq, ...) per channel, src/demod.c:379-392).  cfg->freqs lists the
 * channels receiver by receiver (receiver r owns the next rx[r].n_channels entries), cfg->n_channels is their sum,
 * cfg->n_streams is 0 or n_rx and cfg->centerfreq is ignored.  Channel numbers (frames, counters, read_dec, events) index
 * cfg->freqs.  All receivers share sample rate and format and advance in lock step: vdl2gpu_submit / vdl2gpu_submit_device
 * take the n_rx buffers of `len` bytes back to back (receiver 0 first); vdl2gpu_submit_planar_s16 is not available.
 * n_rx <= 65535; oversample 20, 10 or 13; VDL2GPU_FLAG_K1_SCALAR is refused. */
typedef struct {
	uint32_t centerfreq;         /* Hz: this receiver's tuning (src/demod.c:385 uses it for every channel of the receiver) */
	uint32_t n_channels;         /* >= 1; this receiver's channels are the next n_channels entries of cfg->freqs */
} vdl2gpu_receiver;
int vdl2gpu_create_receivers(const vdl2gpu_config *cfg, const vdl2gpu_receiver *rx, uint32_t n_rx, vdl2gpu_ctx **out);
/* Receivers of different sample rates and formats in one context (e.g. RTL-SDR dongles, cu8 at 1.05 Msps, next to
 * SDRplay devices, cs16 at 2.1 Msps): as vdl2gpu_create_receivers, but receiver r samples at 105000 x rx[r].oversample
 * in format rx[r].sample_fmt, and its filter taps and NCO steps are those of one reference process at that rate.
 * cfg->sample_rate, oversample, sample_fmt and centerfreq must be 0 (they are per receiver here), cfg->n_streams is 0 or
 * n_rx, n_rx <= 65535, VDL2GPU_FLAG_K1_SCALAR is refused.  The receivers advance in lock step in DECIMATED samples:
 * feed the context with vdl2gpu_submit_span / vdl2gpu_submit_span_device (vdl2gpu_submit, vdl2gpu_submit_device and
 * vdl2gpu_submit_planar_s16 return VDL2GPU_EINVAL).  max_chunk_bytes bounds the buffer of any one receiver in a span:
 * n_dec <= max_chunk_bytes / max over r of (oversample_r x bytes per complex sample_r).  vdl2gpu_get_tables returns
 * VDL2GPU_EINVAL (there is no single rate); stats.iq_samples counts the complex samples of all receivers.  Listing the
 * receivers grouped by rate keeps the 32 channels of a K1 warp on one rate, which runs faster than interleaved rates.
 * With VDL2GPU_FLAG_RAGGED in cfg->flags the receivers do not advance in lock step: every receiver brings its own number
 * of decimated samples to each span (vdl2gpu_submit_ragged); a uniform fleet gets ragged spans by describing itself here. */
typedef struct {
	uint32_t centerfreq;         /* Hz */
	uint32_t n_channels;         /* >= 1; the next n_channels entries of cfg->freqs */
	uint32_t oversample;         /* 10, 13 or 20: this receiver samples at 105000 x oversample */
	uint32_t sample_fmt;         /* VDL2GPU_FMT_U8 or VDL2GPU_FMT_S16_LE */
} vdl2gpu_receiver_ex;
int vdl2gpu_create_mixed_receivers(const vdl2gpu_config *cfg, const vdl2gpu_receiver_ex *rx, uint32_t n_rx, vdl2gpu_ctx **out);
int vdl2gpu_destroy(vdl2gpu_ctx *ctx);
const char *vdl2gpu_strerror(int code);
const char *vdl2gpu_last_error(void);

/* ---- data path ---- */
/* == process_buf_uchar / process_buf_short (src/demod.c:339-365): `iq` is interleaved I,Q, `len` is in BYTES,
 * the caller may reuse `iq` as soon as the call returns.  Asynchronous: copies into a pinned staging ring,
 * enqueues H2D + kernels.  Blocks only when n_inflight chunks are pending (the reference's back-pressure).
 * With n_streams = S > 1, `iq` holds S buffers of `len` bytes back to back (stream 0 first) and `len` is the size of ONE. */
int vdl2gpu_submit(vdl2gpu_ctx *ctx, const void *iq, uint32_t len);
/* Ingest adaptor for front-ends that deliver I and Q as separate int16 arrays (SDRplay: src/sdrplay.c:72-134,
 * src/sdrplay3.c): n_pairs values each; replaces the host-side interleave + process_buf_short.  The context must
 * have been created with VDL2GPU_FMT_S16_LE. */
int vdl2gpu_submit_planar_s16(vdl2gpu_ctx *ctx, const int16_t *xi, const int16_t *xq, uint32_t n_pairs);
/* Same, but `dev_iq` already lives in this GPU's memory (e.g. the receive buffer of an NCCL broadcast).
 * `producer_stream` (cudaStream_t, may be NULL = legacy default stream) is the stream on which the buffer
 * was produced; the library orders its work after it.  The buffer may be overwritten once
 * vdl2gpu_wait_input_consumed() has been enqueued on the stream that overwrites it. */
int vdl2gpu_submit_device(vdl2gpu_ctx *ctx, const void *dev_iq, uint32_t len, void *producer_stream);
/* One span of n_dec decimated samples for every receiver of a receivers context (vdl2gpu_create_mixed_receivers or
 * vdl2gpu_create_receivers): receiver r contributes n_dec x oversample_r complex samples in its own format, and the n_rx
 * buffers lie back to back, receiver 0 first, so receiver r's buffer starts n_dec x sum over q < r of
 * (oversample_q x bytes per complex sample_q) bytes in (a 64-bit offset).  n_dec == 0 is a no-op; a span longer than
 * max_chunk_bytes allows returns VDL2GPU_ETOOBIG.  On a vdl2gpu_create_receivers context this is vdl2gpu_submit /
 * vdl2gpu_submit_device with len = n_dec x oversample x bytes per complex sample; other contexts return VDL2GPU_EINVAL.
 * Same buffer and stream rules as vdl2gpu_submit / vdl2gpu_submit_device. */
int vdl2gpu_submit_span(vdl2gpu_ctx *ctx, const void *iq, uint32_t n_dec);
int vdl2gpu_submit_span_device(vdl2gpu_ctx *ctx, const void *dev_iq, uint32_t n_dec, void *producer_stream);
/* Ragged spans (a context made by vdl2gpu_create_mixed_receivers with VDL2GPU_FLAG_RAGGED): receiver r brings its own
 * n_dec[r] >= 0 decimated samples to the span, i.e. n_dec[r] x oversample_r complex samples in its own format, and the
 * counts may differ from receiver to receiver and from span to span (0 for any number of spans, fewer than 12 or 160, ...).
 * Receivers need not be paced against each other: every receiver decodes exactly what one reference process at its rate
 * decodes from the concatenation of everything that receiver brought, however the streams were cut.  The n_rx buffers lie
 * back to back, receiver 0 first: receiver r's starts sum over q < r of n_dec[q] x oversample_q x bytes per complex
 * sample_q bytes in (a 64-bit offset).  All counts 0 is a no-op; a count above the largest span max_chunk_bytes allows for
 * that receiver returns VDL2GPU_ETOOBIG; on any other context these calls return VDL2GPU_EINVAL.  Same buffer and stream
 * rules as vdl2gpu_submit_span / vdl2gpu_submit_span_device, which on a ragged context are these calls with all counts
 * equal.  Frames' sync_dec_index, trace events' dec_index and burst timestamps count in the receiver's own decimated
 * samples; a burst's timestamp is the span's arrival time moved back by the distance from its sync sample to the end of
 * its receiver's samples in the span.  vdl2gpu_read_dec returns the span's width (largest count) in rows, of which only
 * the first n_dec[r] are defined for the channels of receiver r. */
int vdl2gpu_submit_ragged(vdl2gpu_ctx *ctx, const void *iq, const uint32_t *n_dec /* [n_rx] */);
int vdl2gpu_submit_ragged_device(vdl2gpu_ctx *ctx, const void *dev_iq, const uint32_t *n_dec /* [n_rx], host memory */,
		void *producer_stream);
/* Pushed input on a ragged mixed-receivers context (VDL2GPU_FLAG_RAGGED): the per-receiver form of the reference's
 * process_buf_uchar / process_buf_short, one call per device callback.  Any other context returns VDL2GPU_EINVAL.
 *
 * vdl2gpu_push(ctx, r, iq, len) queues len bytes of receiver r, in its own format, inside the library.  len may be any
 * length up to max_chunk_bytes (more: VDL2GPU_ETOOBIG; 0: a no-op); a buffer may end inside a decimation group or inside a
 * complex sample.  Each receiver decodes exactly what one reference process at its rate decodes from the concatenation of
 * every byte pushed for it, however the stream was cut, up to the last whole decimation group that has gone into a span.
 * The caller may reuse iq as soon as the call returns.  VDL2GPU_EINVAL, before the device is touched, for a NULL context,
 * r >= n_rx, iq NULL with len > 0, or any context but a ragged mixed-receivers one.
 *   - The bytes go to pinned host memory and are copied at once into the receiver's ring in device memory, on a copy stream
 *     of the context, so the copy engine moves them while the GPU computes.
 *   - Back-pressure, as in the reference: a push blocks while its receiver's ring lacks room.  Room comes back when spans
 *     already in flight have converted their samples (nothing is needed from the caller for that) and when
 *     vdl2gpu_submit_pushed takes queued bytes into spans.  A push of up to max_chunk_bytes that follows a
 *     vdl2gpu_submit_pushed never waits for the caller, only for the GPU: a single thread that alternates pushes and
 *     vdl2gpu_submit_pushed cannot deadlock.
 *   - Memory: the first push allocates every receiver's ring, max_chunk_bytes + (max_span + 1) x oversample_r x bytes per
 *     complex sample_r bytes (rounded up to 16), in device memory and again in pinned host memory; contexts that never push
 *     pay nothing.  For 2048 receivers at the default 1 MiB that is up to about 4 GiB of each (a cs16 receiver at oversample
 *     20: 2 MiB).  An allocation failure is returned by that first push.
 *   - Each push records its arrival time (gettimeofday at entry) for the burst timestamps below.
 *
 * vdl2gpu_submit_pushed(ctx) reads every receiver's queue once, when it is entered, and submits ragged spans until every
 * whole decimation group queued at that moment is in a span.  Bytes pushed during the call wait for the next call, so the
 * call returns however fast other threads keep pushing, and a control loop of submit_pushed and poll keeps delivering
 * frames.  Each span takes min(whole groups left of that snapshot, max_span) from every receiver, so a receiver far behind
 * catches up over several spans.  Returns the number of spans submitted (0 when nothing was queued: a no-op that leaves restarts pending)
 * or a negative error.  Frames come out through vdl2gpu_poll / vdl2gpu_flush as for any span (vdl2gpu_flush forms no
 * spans).  Positions, stats.iq_samples, dec_samples and chunks_submitted count exactly as for vdl2gpu_submit_ragged spans
 * of the same counts.
 *
 * Burst timestamps of pushed spans: the arrival time of the push that carried the last input sample of the burst's sync
 * decimation group, moved back by the input samples that push carried after that sample, at the receiver's own rate (the
 * receiver's analogue of the reference stamping at processing time; it does not depend on when vdl2gpu_submit_pushed runs).
 *
 * Threads: vdl2gpu_push may run concurrently for different receivers, and concurrently with vdl2gpu_submit_pushed,
 * vdl2gpu_poll, vdl2gpu_flush and vdl2gpu_get_stats on the one control thread.  Two pushes of the same receiver are
 * serialised, in an unspecified order: keep one thread per receiver.  No push may run during vdl2gpu_update_receivers or
 * vdl2gpu_destroy, and no push of receiver r during vdl2gpu_restart_receiver(ctx, r, ...).
 *
 * With the other calls:
 *   - vdl2gpu_submit_ragged*, vdl2gpu_submit_span* return VDL2GPU_EINVAL while any receiver has pushed bytes not yet in a
 *     span (stream order); with nothing queued the two ways of feeding may alternate.
 *   - vdl2gpu_restart_receiver(r) drops r's pushed bytes not yet in a span, a split sample included (the old process is
 *     killed at the call); the restart applies at the next span as always, and bytes pushed after the call belong to the
 *     new process.  Call vdl2gpu_submit_pushed first to have the queued groups decoded.
 *   - vdl2gpu_update_receivers also refuses (VDL2GPU_EINVAL) while any receiver has a whole group queued.  A kept receiver
 *     carries its partial group (fewer than oversample_r samples, or a split sample) and its arrival records to its new
 *     index; a removed receiver's bytes are dropped; a new receiver starts empty.  Once anything has been pushed, the call
 *     allocates the new list's rings before it frees the old ones, so for the call's duration the device and the pinned
 *     host memory briefly hold both sets of rings (up to about 2 x 4 GiB of each for 2048 receivers at the default
 *     max_chunk_bytes), on top of the rebuild described below. */
int vdl2gpu_push(vdl2gpu_ctx *ctx, uint32_t r, const void *iq, uint32_t len);
int vdl2gpu_submit_pushed(vdl2gpu_ctx *ctx);
/* out[r] = decimated samples of receiver r accepted so far, for the first n_rx receivers of a receivers context (with ragged
 * spans: the sum of receiver r's counts, which shows which receiver lags; in lock step all receivers are equal) */
int vdl2gpu_get_receiver_positions(vdl2gpu_ctx *ctx, uint64_t *out, uint32_t n_rx);
/* Restart receiver r of a ragged mixed-receivers context (VDL2GPU_FLAG_RAGGED) at the start of the next span that runs:
 * from that span on, its channels decode exactly what a freshly started reference process tuned to (centerfreq, freqs)
 * decodes from the samples the receiver brings from then on.  centerfreq 0 keeps the receiver's centre; freqs NULL keeps
 * its channel frequencies, otherwise it holds rx[r].n_channels entries (the channel count, oversample and format stay).
 * For a front-end whose receiver reconnects, re-enumerates with a gap in its stream, is swapped for another device, or is
 * moved to other frequencies; every other receiver keeps its demodulator state and its bursts in flight.
 *   - Any of the four span calls applies it; an all-zero ragged span is a no-op and leaves it pending.  Several receivers
 *     may restart in the same span; restarting one twice before a span runs keeps the last tuning.  The receiver may
 *     bring any count to that span, 0 included.
 *   - Its position (vdl2gpu_get_receiver_positions), frames' sync_dec_index, trace dec_index and burst timestamps keep
 *     counting in its own decimated samples; burst_seq keeps counting, so (channel, burst_seq, idx) never repeats, and the
 *     per-channel counters are the sums over the old and the new process.
 *   - The old process is treated as killed at the restart point: a burst already complete is delivered normally (with
 *     the old frequency); a burst still in progress is dropped without a frame, a trace event or a counter change.
 * Returns VDL2GPU_EINVAL, before the device is touched, for a NULL context, r >= n_rx, or any context but a ragged
 * mixed-receivers one. */
int vdl2gpu_restart_receiver(vdl2gpu_ctx *ctx, uint32_t r, uint32_t centerfreq, const uint32_t *freqs);
/* Replace the receivers of a drained ragged mixed-receivers context (VDL2GPU_FLAG_RAGGED) with rx[0..n_rx): receivers
 * join, leave, move within the list, or are swapped for a device of another kind (remove it and add the new one), and
 * every other receiver carries on as if nothing had happened.  freqs lists the channels receiver by receiver, as for
 * vdl2gpu_create_mixed_receivers.
 *   - from[i] >= 0: entry i continues old receiver from[i] and repeats its current description (centre, channel count,
 *     oversample, format and channel frequencies, after any restarts; a retune is vdl2gpu_restart_receiver's job).  Each
 *     old receiver appears at most once; those not listed are removed.
 *   - from[i] == -1: a new receiver, which decodes what a freshly started reference process decodes from what it brings:
 *     position 0, burst_seq 0, zero counters.
 *   - A kept receiver keeps its demodulator state, its burst in progress (delivered later under its new channel numbers),
 *     its position (vdl2gpu_get_receiver_positions), sync_dec_index, timestamps, burst_seq and counters, and a restart
 *     still pending applies with the next span.  A removed receiver's burst in progress is dropped without a frame, a trace
 *     event or a counter change, and its counters are gone (read them first).
 *   - Only on a drained context (vdl2gpu_chunks_in_flight == 0, as after vdl2gpu_flush): frames delivered before the call
 *     carry the old channel numbers and frames delivered after it the new ones.  Trace events not yet read still carry the
 *     old numbers.  vdl2gpu_read_dec has no rows until a span runs.  max_span follows the create rule for the new list: a
 *     receiver with more bytes per decimated sample than any before shortens the longest allowed span.
 *   - The context is rebuilt: the new buffers are allocated before the old ones are freed, so the device briefly holds both
 *     (about 2 x 9 GB for 2048 receivers x 8 channels at the default max_chunk_bytes), and the next spans recapture their
 *     CUDA graphs.
 * Returns VDL2GPU_EINVAL for a NULL context, any context but a ragged mixed-receivers one, spans in flight, a bad from[]
 * (out of range, repeated, or a changed description), and the receiver checks of vdl2gpu_create_mixed_receivers (none,
 * more than 65535, oversample, format, no channels); VDL2GPU_ETOOBIG past the kernels' 32-bit element index.  Refusals
 * touch neither the context nor the device; a CUDA or allocation failure during the rebuild leaves the context as it was. */
int vdl2gpu_update_receivers(vdl2gpu_ctx *ctx, const vdl2gpu_receiver_ex *rx, const int32_t *from, uint32_t n_rx,
		const uint32_t *freqs);
int vdl2gpu_wait_input_consumed(vdl2gpu_ctx *ctx, void *stream);
/* Make `stream` (cudaStream_t) wait for all device work enqueued by this context so far (for timing with
 * events recorded on the caller's stream, and for ordering consumers of device-side results). */
int vdl2gpu_stream_wait(vdl2gpu_ctx *ctx, void *stream);
/* Deliver the frames of every chunk that has finished, in (chunk, channel, burst, idx) order.  Returns the
 * number of frames delivered or a negative error.  cb may be NULL (frames are dropped, counters kept). */
int vdl2gpu_poll(vdl2gpu_ctx *ctx, vdl2gpu_frame_cb cb, void *user);
/* Chunks submitted whose frames have not been harvested yet (0 right after a poll = everything delivered). */
int vdl2gpu_chunks_in_flight(vdl2gpu_ctx *ctx);
/* Block until everything submitted so far has been processed, then deliver like poll. */
int vdl2gpu_flush(vdl2gpu_ctx *ctx, vdl2gpu_frame_cb cb, void *user);
int vdl2gpu_get_stats(vdl2gpu_ctx *ctx, vdl2gpu_stats *out);
/* per-channel counters, 9 x uint64 per channel in the order: sync_good, hdr_crc_good, bursts, burst_err,
 * blocks_processed, blocks_fec_ok, msg_good, fcs_good, fcs_bad.  Implies a flush of device work. */
int vdl2gpu_get_channel_counters(vdl2gpu_ctx *ctx, uint64_t *out, uint32_t n_channels);

/* Input levels (VDL2GPU_FLAG_INPUT_LEVELS): exact integer figures of every raw sample an input has brought, for telling a
 * dead or disconnected receiver, a gain set too high or a DC spike from a quiet sky without waiting for traffic.  A
 * component's integer code c is, for cu8, c = 2v - 255 (c / 255 is exactly the reference's (v - 127.5) / 127.5,
 * src/demod.c:349-354) and, for cs16, c = v (c / 32768, src/demod.c:361-363).  A sample is clipped when its I or Q sits on
 * a rail: cu8 v = 0 or 255, cs16 v = -32768 or 32767.  Mean power in dBFS is 10 log10(pow / (samples x full_scale^2)),
 * with pow = pow_hi x 2^64 + pow_lo; the DC offsets are sum_i / (samples x full_scale) and sum_q / (samples x full_scale). */
typedef struct {
	uint64_t samples;            /* complex samples measured */
	int64_t sum_i, sum_q;        /* sum of c over the I and over the Q components */
	uint64_t pow_lo, pow_hi;     /* sum of (c_I^2 + c_Q^2), one unsigned 128-bit integer */
	uint64_t clipped;            /* complex samples with I or Q on a rail */
	uint32_t peak;               /* largest |c| of any component */
	uint32_t full_scale;         /* 255 (cu8) or 32768 (cs16) */
} vdl2gpu_input_levels;          /* 56 bytes */
/* out[k] = the levels of input k for k < n.  Inputs: a fan-out context has one, an n_streams context n_streams, a
 * receivers context (vdl2gpu_create_receivers, vdl2gpu_create_mixed_receivers) one per receiver, in receiver order.
 *   - Cumulative from create (for a receiver added by vdl2gpu_update_receivers: from when it joined), over every sample of
 *     every chunk or span submitted before the call; the call waits for that work, as vdl2gpu_get_channel_counters does.
 *     Host, device and planar submits count alike.
 *   - Pushed input counts once it enters a span: positions[r] x oversample_r complex samples for receiver r.  Bytes still
 *     queued, and bytes a restart drops, are not counted.  vdl2gpu_restart_receiver keeps counting, as the per-channel
 *     counters do.  vdl2gpu_update_receivers: a kept receiver carries its levels to its new index, a new receiver starts
 *     at zero, a removed receiver's levels are gone.
 *   - The integers are exact and do not depend on how the stream was cut (chunk, span and push lengths, ragged counts),
 *     n_inflight, graphs or trace.  The sum of squares never wraps.
 *   - Frames, metadata, counters, trace events and vdl2gpu_stats are the same with the flag on or off.  A context without
 *     the flag allocates and launches nothing for it.
 * Runs on the control thread, concurrently with vdl2gpu_push (which does not touch the figures).  VDL2GPU_EINVAL (with
 * vdl2gpu_last_error) for a NULL context or output, n larger than the number of inputs, or a context created without
 * VDL2GPU_FLAG_INPUT_LEVELS.  Not available through the stage stubs or the drop-in symbols. */
int vdl2gpu_get_input_levels(vdl2gpu_ctx *ctx, vdl2gpu_input_levels *out, uint32_t n);

/* Channel levels (VDL2GPU_FLAG_CHANNEL_LEVELS): what every channel hears in its band, for telling a raised noise floor or a
 * parked carrier from a quiet sky on a channel that sends no frames.  p = fl32(fl32(re x re) + fl32(im x im)), without FMA,
 * of a decimated sample is the reference's symbol power (src/demod.c:266): 10 log10(p) is on the dBFS scale of a frame's
 * frame_pwr_dbfs.  Its bin comes from the biased exponent E of p alone, b = min(max(E - 90, 0), 39): bins 3.01 dB wide
 * covering -108.4 to +6.0 dBFS.  q = (uint64)(p x 2^48), truncated; p < 2^15 for every decimated sample, so q fits. */
typedef struct {
	uint64_t hist[40];           /* decimated samples by octave of p: [0] p < 2^-36 (zeros included),
	                              * [b] 2^(b-37) <= p < 2^(b-36) for b = 1..38, [39] p >= 2^2; their sum is the sample count */
	uint64_t pow_lo, pow_hi;     /* sum over those samples of q, one unsigned 128-bit integer */
	float peak_pow;              /* largest p */
	float mag_lp, mag_nf;        /* the channel's noise-floor filters as they stand now (src/demod.c:238-243) */
	float nf_pwr_dbfs;           /* 20 log10f(mag_nf + 0.001f), computed as for a frame's nf_pwr_dbfs */
} vdl2gpu_channel_levels;        /* 352 bytes */
/* out[k] = the levels of channel k (its index into cfg->freqs) for k < n.
 *   - Cumulative from create (for a channel added by vdl2gpu_update_receivers: from when it joined), over every decimated
 *     sample of every chunk or span submitted before the call; the call waits for that work.  Take windows by
 *     differencing two reads.
 *   - The integers and peak_pow are exact and do not depend on chunk, span or push lengths, ragged counts, n_inflight,
 *     graphs, trace or how the phase pass is cut in time (VDL2GPU_K2A_SPLIT, VDL2GPU_STAGES=3).  Ragged spans count only
 *     the rows a receiver brought.
 *   - vdl2gpu_restart_receiver: hist, power and peak keep counting, as the per-channel counters do; mag_lp and mag_nf are
 *     the new process's, which starts at 0 and 2.0 as the reference's does (src/demod.c:383).
 *   - vdl2gpu_update_receivers: a kept channel carries its levels to its new index, a new channel starts at zero, a
 *     removed channel's levels are gone.
 *   - Frames, metadata, counters, trace events and vdl2gpu_stats are the same with the flag on or off.  A context without
 *     the flag allocates and launches nothing for it.
 * Runs on the control thread, concurrently with vdl2gpu_push.  VDL2GPU_EINVAL (with vdl2gpu_last_error) for a NULL context
 * or output, n larger than the number of channels, or a context created without VDL2GPU_FLAG_CHANNEL_LEVELS.  Not
 * available through the stage stubs or the drop-in symbols. */
int vdl2gpu_get_channel_levels(vdl2gpu_ctx *ctx, vdl2gpu_channel_levels *out, uint32_t n);

/* Spectrum (VDL2GPU_FLAG_SPECTRUM): the power spectrum of every input in VDL2GPU_SPECTRUM_BINS bins, for seeing what lies
 * between and beside the configured channels: an interferer, a DC spike, a receiver tuned off, traffic on a slot not yet
 * configured, a filter edge.  Inputs are numbered as for vdl2gpu_get_input_levels.
 *   - Segment j of an input is its complex samples [1024 j, 1024 (j + 1)), counted from create (for a receiver added by
 *     vdl2gpu_update_receivers: from when it joined; after vdl2gpu_restart_receiver: from the restart).  A segment counts
 *     once its last sample has been in a chunk or span that ran; the samples of the segment not yet complete (at most 1023)
 *     wait on the device.
 *   - Per segment, with x_n the float the reference makes of sample n (cu8 c / 255, cs16 v / 32768): y_n = fl32(x_n w_n),
 *     w the periodic Hann window 0.5 - 0.5 cos(2 pi n / 1024) rounded to float; a radix-2 FFT with float twiddles, every
 *     product and sum rounded on its own; p_k = fl32(fl32(re^2) + fl32(im^2)).  Bin k (stored order) is the frequency
 *     centre + (k - 512) fs / 1024, fs = 105000 x the input's oversample: bin 512 is the centre.
 *   - pow[k] = pow_hi[k] x 2^64 + pow_lo[k] is the exact sum over segments of (uint64)(p_k x 2^40); peak[k] the largest p_k
 *     (peak hold).  A full-scale complex tone on a bin gives p = 512^2, so the mean power in dBFS is
 *     10 log10(pow / 2^40 / segments / 512^2).
 *   - The figures do not depend on how the stream was cut (chunk, span and push lengths, ragged counts), n_inflight, graphs,
 *     trace or VDL2GPU_FLAG_NO_OVERLAP.  Pushed input counts once it enters a span; bytes still queued, or dropped by a
 *     restart, never count.
 *   - vdl2gpu_restart_receiver zeroes the receiver's spectrum and drops its waiting samples at the span the restart applies
 *     to: a retune changes what every bin means.  Read the old figures first (this call waits for everything submitted).
 *     vdl2gpu_update_receivers: a kept receiver carries its figures and waiting samples to its new index, a new receiver
 *     starts at zero, a removed receiver's figures are gone.
 *   - Frames, metadata, counters, trace events, vdl2gpu_stats and both levels are the same with the flag on or off.  A
 *     context without the flag allocates and launches nothing for it.  With it, a context holds 28 KB of device memory per
 *     input (the sums, the peaks and the waiting samples), about 460 MB at 16384 one-channel receivers. */
#define VDL2GPU_SPECTRUM_BINS 1024
typedef struct {
	uint64_t segments;                              /* complete segments counted */
	uint32_t pending;                               /* samples of the incomplete segment held on the device, 0..1023 */
	uint32_t reserved;
	uint64_t pow_lo[VDL2GPU_SPECTRUM_BINS];         /* sum of (uint64)(p_k 2^40), one unsigned 128-bit integer per bin */
	uint64_t pow_hi[VDL2GPU_SPECTRUM_BINS];
	float peak[VDL2GPU_SPECTRUM_BINS];              /* largest p_k */
} vdl2gpu_spectrum;                                 /* 20496 bytes */
/* out[k] = the spectrum of input first + k for k < n, after everything submitted so far has run.  Runs on the control
 * thread, concurrently with vdl2gpu_push.  VDL2GPU_EINVAL (with vdl2gpu_last_error) for a NULL context or output, a range
 * past the inputs, or a context created without VDL2GPU_FLAG_SPECTRUM.  Not available through the stage stubs or the
 * drop-in symbols. */
int vdl2gpu_get_spectrum(vdl2gpu_ctx *ctx, uint32_t first, uint32_t n, vdl2gpu_spectrum *out);

/* ---- multi-GPU ingest (one process per GPU; global channel k is demodulated on GPU k mod N, the reference's
 * channel threads share nothing but the read-only sample buffer: src/dumpvdl2.c:117-135, src/demod.c:50,300-301).
 * Rank 0 owns the IQ source; vdl2gpu_mg_* fans every step's chunks out into a double-buffered receive area on every
 * rank and feeds the rank's context from it (vdl2gpu_submit_device), either with ncclBroadcast (libnccl is dlopen()ed)
 * or, with no kernel at all, with copy-engine peer copies into CUDA-IPC-mapped buffers ordered by stream memory
 * operations.  The caller carries the small opaque blobs between the processes (MPI, sockets, ...).  Typical sequence:
 *
 *     uint8_t id[VDL2GPU_MG_ID_BYTES];              // NCCL mode only
 *     if(rank == 0) vdl2gpu_mg_unique_id(id, sizeof id);   bcast(id);
 *     vdl2gpu_mg_create(ctx, rank, world, mode, id, step_bytes, &mg);
 *     // copy-engine mode only:  vdl2gpu_mg_export(mg, blob, n);  allgather(blob -> all);  vdl2gpu_mg_import(mg, all, world * n);
 *     half = vdl2gpu_mg_stage(mg, pieces, sizes, n_pieces, host?, step_bytes);          // step 0
 *     for(;;) {
 *         next = vdl2gpu_mg_stage(mg, ...);          // step s+1 travels while step s is demodulated
 *         vdl2gpu_mg_submit(mg, half, chunks_per_step, chunk_bytes);
 *         vdl2gpu_poll(ctx, frame_cb, user);
 *         half = next;
 *     }
 * ---- */
enum { VDL2GPU_MG_NCCL = 0, VDL2GPU_MG_COPY_ENGINE = 1 };
#define VDL2GPU_MG_ID_BYTES 128
typedef struct vdl2gpu_mg vdl2gpu_mg;
int vdl2gpu_mg_unique_id(uint8_t *id, size_t cap);      /* rank 0: ncclGetUniqueId */
int vdl2gpu_mg_create(vdl2gpu_ctx *ctx, int rank, int world, int mode, const uint8_t *nccl_id /* NULL in copy-engine mode */,
		uint32_t stage_bytes /* bytes of one step, at most */, vdl2gpu_mg **out);
size_t vdl2gpu_mg_blob_bytes(void);
int vdl2gpu_mg_export(vdl2gpu_mg *mg, uint8_t *blob, size_t cap);
int vdl2gpu_mg_import(vdl2gpu_mg *mg, const uint8_t *all_blobs, size_t bytes);
/* rank 0: the pieces (device pointers, or pinned host pointers with src_is_host) that make up the step, `total` bytes;
 * other ranks: n_src = 0, same total.  Returns the half (0/1) for vdl2gpu_mg_submit or a negative error.  Asynchronous. */
int vdl2gpu_mg_stage(vdl2gpu_mg *mg, const void *const *src, const uint32_t *src_bytes, uint32_t n_src, int src_is_host, uint32_t total);
int vdl2gpu_mg_submit(vdl2gpu_mg *mg, int half, uint32_t n_chunks, uint32_t chunk_bytes);
int vdl2gpu_mg_mode(vdl2gpu_mg *mg);
int vdl2gpu_mg_destroy(vdl2gpu_mg *mg);

/* One frame in the reference's raw-frame archive format (2-octet big-endian record length + proto3
 * dumpvdl2.raw_avlc_frame, proto/dumpvdl2.proto:25-48, as written by src/fmtr-binary.c + src/output-file.c:181-189):
 * records written back to back replay through an unmodified `dumpvdl2 --raw-frames-file`.
 * Returns the record size in octets, or a negative error.  Host-only helper (no device work). */
int vdl2gpu_serialize_raw_frame(const vdl2gpu_frame *frame, const char *station_id, uint8_t *out, size_t cap);

/* ---- introspection for parity tests / profiling ---- */
/* tables the kernels use, computed by the library's own host code (restating src/demod.c:349-377,367-370,84-96) */
int vdl2gpu_get_tables(vdl2gpu_ctx *ctx, float levels[256], float sin_lut[257], float cos_lut[257],
		float A[3], float B[3], float lr_X[16], float *lr_denom, float pr_phase[16]);
/* decimated samples of the most recent chunk (VDL2GPU_FLAG_KEEP_DEC): out[n_dec][n_channels][2] floats.
 * *n_dec receives the count; cap_floats is the capacity of out.  Synchronises. */
int vdl2gpu_read_dec(vdl2gpu_ctx *ctx, float *out, size_t cap_floats, uint32_t *n_dec);
/* drain trace events (VDL2GPU_FLAG_TRACE).  Synchronises.  Returns the number copied (0: none left).  The device buffer
 * holds 2^20 events and restarts whenever it has been drained; if it filled up in between, the stored events are
 * delivered first and the following call returns VDL2GPU_EOVERFLOW once (the count of lost events in vdl2gpu_last_error). */
int vdl2gpu_read_events(vdl2gpu_ctx *ctx, vdl2gpu_event *out, uint32_t cap);
/* device time (ms) spent in each kernel for the chunks completed so far, measured with CUDA events on
 * the library's streams when timing was enabled with vdl2gpu_enable_timing(ctx, 1).
 * Order: K0, K1, K2a, K2 (+history copy), K3 (+finish). */
int vdl2gpu_enable_timing(vdl2gpu_ctx *ctx, int on);
int vdl2gpu_get_kernel_ms(vdl2gpu_ctx *ctx, double ms[5], uint64_t launches[5]);
/* stage boundaries of the timed chunks harvested so far, 8 floats per chunk: chunk number, then ms since
 * vdl2gpu_enable_timing(ctx, 1) of: front (K0+K1) start, K1 end, K2a start, K2a end, K2 start, K2|K3, K3 end (with graph
 * replay K3 counts into K2).  Returns the number of rows copied. */
int vdl2gpu_get_timeline(vdl2gpu_ctx *ctx, float *out, uint32_t cap_rows);
/* diagnostic (context created with VDL2GPU_BLOCK_TRACE=1 in the environment): where and when every block of K1 / K2 ran,
 * 6 x uint64 per record {kernel (1 K1, 2 K2), block, SM id, 0, start ns, end ns}.  Synchronises. */
int vdl2gpu_debug_block_trace(vdl2gpu_ctx *ctx, uint64_t *out, uint32_t cap_records);

/* ---- raw launch stubs (extern "C", plain pointers; used by the micro-parity tests and by hosts that
 *      manage device memory themselves).  All pointers are DEVICE pointers unless stated otherwise; `stream` is a
 *      cudaStream_t.  The launch stubs only enqueue kernels: no allocation, no synchronisation.
 *      (vdl2gpu_launch_rs_verify builds its GF tables on the first call on a device.) ---- */
/* K0: raw cu8/cs16 -> float samples {re, im} per complex sample, the reference's sbuf (src/demod.c:339-365:
 * process_buf_uchar / process_buf_short).  levels256 = the 256-entry table of process_buf_uchar_init
 * (src/demod.c:349-354), only read for VDL2GPU_FMT_U8. */
int vdl2gpu_launch_convert(const void *raw, uint32_t n_pairs, uint32_t sample_fmt, const float *levels256,
		float *samples_out /* [n_pairs][2] */, void *stream);
/* K4: FCS residue of n frames stored back to back (src/crc.c:21-64 as used at src/avlc.c:177) */
int vdl2gpu_launch_fcs_crc16(const uint8_t *frames, const uint32_t *offsets, const uint32_t *lens,
		uint32_t n_frames, uint16_t *residues_out, void *stream);
/* RS(255,249) errors-and-erasures decode of n blocks in place (src/rs.c:32-49); fec_octets[i] in {0,2,4,6} */
int vdl2gpu_launch_rs_verify(uint8_t *blocks /* [n][255] */, const int32_t *fec_octets, uint32_t n_blocks,
		int32_t *ret_out, void *stream);

/* K2a: phase_out[i] = (float)atan2((double)im, (double)re) and mag_out[i] = hypotf(re, im) of n_elems decimated
 * samples dec[n_elems][2] (src/demod.c:232,238,256); the phase is atan2 correctly rounded to double, narrowed.
 * exact_libm = 0: the short double-precision evaluation with a Ziv rounding test the pipeline uses, and the full
 * evaluation where that test fails; 1: the full evaluation for every element (no fast path).  Same floats either way. */
int vdl2gpu_launch_phase_mag(const float *dec, uint32_t n_elems, float *phase_out, float *mag_out, int exact_libm, void *stream);

/* ---- stage stubs: the three per-channel stages one at a time, on device memory the caller owns.
 * A vdl2gpu_stage is the device-resident state of n_channels vdl2_channel_t's (src/dumpvdl2.h:321-352) plus the
 * read-only tables, laid out inside ONE block of device memory that the caller allocates (256-byte aligned,
 * vdl2gpu_stage_device_bytes() bytes).  vdl2gpu_stage_create fills it (synchronous copies, no allocation); the three
 * launch stubs below then only enqueue kernels on `stream`.  Decimated samples travel between K1 and K2 in a caller
 * buffer dec[n_dec][row_stride][2] floats, row_stride = vdl2gpu_stage_row_stride(n_channels) (channels padded to 32).
 * Config fields used: sample_rate, oversample, centerfreq, n_channels, freqs, max_ppm, flags (TRACE, K1_SCALAR). ---- */
typedef struct vdl2gpu_stage vdl2gpu_stage;
size_t vdl2gpu_stage_device_bytes(uint32_t n_channels, uint32_t max_dec, uint32_t flags);
uint32_t vdl2gpu_stage_row_stride(uint32_t n_channels);
int vdl2gpu_stage_create(const vdl2gpu_config *cfg, uint32_t max_dec /* decimated samples per launch, at most */,
		void *device_mem, size_t device_bytes, vdl2gpu_stage **out);
int vdl2gpu_stage_destroy(vdl2gpu_stage *stage);
/* device address of the stage's cu8 level table, for vdl2gpu_launch_convert */
int vdl2gpu_stage_levels(vdl2gpu_stage *stage, const float **levels256_dev);
/* K1: NCO mix + 2-pole Chebyshev IIR + decimation == the sample loop of process_samples (src/demod.c:288-337, with
 * sincosf_lut :58-72, multiply :200-203, chebyshev_lpf_2pole :74-79) for every channel.  Filter, NCO and decimation
 * state persist in the stage across calls.  *n_dec_out (host) receives the number of rows written to dec_out. */
int vdl2gpu_launch_mix_iir_decimate(vdl2gpu_stage *stage, const float *samples /* [n_pairs][2] */, uint32_t n_pairs,
		float *dec_out /* [n_dec][row_stride][2] */, uint32_t *n_dec_out, void *stream);
/* K2a + K2: demod() (src/demod.c:222-286: phase ring, got_sync :105-198, D8PSK slicing) and the header part of
 * decode_vdl2_burst (src/decode.c:198-258) over n_dec decimated samples of every channel; completed bursts are
 * queued inside the stage for vdl2gpu_launch_burst_fec. */
int vdl2gpu_launch_sync_slice(vdl2gpu_stage *stage, const float *dec /* [n_dec][row_stride][2] */, uint32_t n_dec, void *stream);
/* K3 (+K4): the data part of decode_vdl2_burst (src/decode.c:259-380: descramble, de-interleave, RS, HDLC unstuff)
 * and the FCS residue of every frame, for all queued bursts.  `region` (device memory, or mapped pinned host memory;
 * 16-byte aligned) receives a 32-byte header followed by the burst records; copy it to the host and hand it to
 * vdl2gpu_parse_records. */
int vdl2gpu_launch_burst_fec(vdl2gpu_stage *stage, uint8_t *region, uint32_t region_bytes, void *stream);
/* HOST helper: records of one region -> frames in (channel, burst, idx) order through cb (`data` valid during the
 * callback).  decimated_rate = sample_rate / oversample.  Returns the number of frames or a negative error. */
int vdl2gpu_parse_records(const uint8_t *region_host, uint32_t region_bytes, uint32_t decimated_rate,
		vdl2gpu_frame_cb cb, void *user);
/* trace events of the stage (VDL2GPU_FLAG_TRACE).  Synchronises the device. */
int vdl2gpu_stage_read_events(vdl2gpu_stage *stage, vdl2gpu_event *out, uint32_t cap);
/* Feeding K3 directly, for tests of the burst decoder that choose every burst themselves.
 * vdl2gpu_stage_queue_bursts queues n bursts in the stage exactly as K2 hands them over, so that the next
 * vdl2gpu_launch_burst_fec decodes them: it pops n burst-pool slots from the stage's device free list, writes each slot's
 * metadata and only its first ceil(nbits / 32) words (later words keep what an earlier burst left in the slot, as after
 * K2), and queues the slots in call order; burst i gets burst_seq = i.  Synchronous.  Returns VDL2GPU_EINVAL if bursts are
 * already queued, a channel is out of range or nbits > 16843, and VDL2GPU_ETOOBIG if n exceeds the free slots (a stage has
 * max(256, 3 x n_channels) slots; every launch of vdl2gpu_launch_burst_fec gives the slots it decoded back).
 * vdl2gpu_stage_read_counters copies the per-channel counters, 9 x uint64 per channel in the order of
 * vdl2gpu_get_channel_counters, to `out` (host, n_channels x 9).  Synchronises the device. */
typedef struct {
	uint32_t channel;            /* < n_channels */
	uint32_t datalen_bits;       /* transmission length from the header (src/decode.c:222) */
	uint32_t nbits;              /* bits in words[], the 25 header bits included */
	uint32_t syndrome;           /* header syndrome */
	float frame_pwr, mag_nf, ppm_error;
	uint32_t freq;
	uint64_t sync_dec_index;
	const uint32_t *words;       /* HOST memory: the still-scrambled bits, bit i = words[i / 32] >> (31 - i % 32) & 1, the rest
	                              * of the last word zero */
} vdl2gpu_burst;                 /* 48 bytes */
int vdl2gpu_stage_queue_bursts(vdl2gpu_stage *stage, const vdl2gpu_burst *bursts, uint32_t n);
int vdl2gpu_stage_read_counters(vdl2gpu_stage *stage, uint64_t *out);

#ifdef __cplusplus
}
#endif
#endif
