/*
 * vdl2_host.cu — host runtime of libvdl2gpu.so: start-up tables, device-resident channel state, the
 * pinned staging ring, stream-ordered kernel chain per IQ chunk, and harvesting of burst records into
 * avlc_decoder_queue_push-shaped frames.  C-ABI in include/vdl2gpu.h.
 *
 * Host arithmetic for the start-up tables restates the reference's init code read strictly
 * (compiled with -ffp-contract=off, no fast-math); citations are file:line under /root/reference.
 * There is no CPU implementation of the sample path in this library: every data-path entry point
 * needs a CUDA device and fails with VDL2GPU_ENODEV / VDL2GPU_ECUDA otherwise.
 */
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/time.h>
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <vector>
#include "../../include/vdl2gpu.h"
#include "vdl2_core.cuh"
#include "vdl2_kernels.h"
#include "vdl2_types.h"
#include "vdl2_tables_host.h"

static thread_local char g_last_error[512] = "";

extern "C" void vdl2gpu_set_last_error(const char *msg) {          /* for the other translation units of the library */
	snprintf(g_last_error, sizeof(g_last_error), "%s", msg ? msg : "");
}

static int fail_cuda(cudaError_t e, const char *what, int line) {
	snprintf(g_last_error, sizeof(g_last_error), "%s failed at vdl2_host.cu:%d: %s", what, line, cudaGetErrorString(e));
	return (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) ? VDL2GPU_ENODEV : VDL2GPU_ECUDA;
}
#define CU(call) do { cudaError_t e_ = (call); if(e_ != cudaSuccess) return fail_cuda(e_, #call, __LINE__); } while(0)
#define KL(call) do { int e_ = (call); if(e_ != 0) return fail_cuda((cudaError_t)e_, #call, __LINE__); } while(0)

/* One owner per CUDA resource: a handle releases what it holds when it is reset, moved onto or destroyed, and a null
 * handle releases nothing.  It reads as the raw handle; put() releases the old one and hands a creating call the address
 * to fill, as in CU(cudaMalloc(x.put(), bytes)). */
template<typename T, typename Release>
class owned {
	T h_ = nullptr;
public:
	owned() = default;
	owned(owned &&o) noexcept : h_(o.h_) { o.h_ = nullptr; }
	owned &operator=(owned &&o) noexcept { if(this != &o) { reset(); h_ = o.h_; o.h_ = nullptr; } return *this; }
	~owned() { reset(); }
	void reset() { if(h_) Release()(h_); h_ = nullptr; }
	T *put() { reset(); return &h_; }
	T get() const { return h_; }
	operator T() const { return h_; }
	T operator->() const { return h_; }
};
struct free_dev { void operator()(void *p) const { cudaFree(p); } };
struct free_host { void operator()(void *p) const { cudaFreeHost(p); } };
struct destroy_event { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct destroy_stream { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
struct destroy_graph_exec { void operator()(cudaGraphExec_t g) const { cudaGraphExecDestroy(g); } };
template<typename T> using dev_mem = owned<T *, free_dev>;
template<typename T> using host_mem = owned<T *, free_host>;          /* cudaHostAlloc */
using event_h = owned<cudaEvent_t, destroy_event>;
using stream_h = owned<cudaStream_t, destroy_stream>;
using graph_exec_h = owned<cudaGraphExec_t, destroy_graph_exec>;

/* ------------------------------------------------------------------------------------------------
 * context
 * ---------------------------------------------------------------------------------------------- */
/* frames harvested but not yet delivered; their octets live in per-chunk blobs (one copy per chunk) */
struct pending_frame {
	vdl2gpu_frame f;
	uint32_t blob, offset;
};

struct chunk_slot {
	host_mem<uint8_t> h_raw; dev_mem<uint8_t> d_raw;
	host_mem<uint8_t> h_out; uint8_t *d_out = nullptr;  /* mapped: d_out is h_out's device address */
	event_h done;
	event_h tk[8];                                      /* front: 0,1,2  mid: 3,6  back: 7,4,5 */
	bool busy = false, timed = false;
	uint64_t seq = 0;
	/* per-chunk arguments (pinned host copy, device copy made by the first node of the front graph) and the three
	 * CUDA graphs of this slot per decimated-sample buffer: front {args copy, K0, K1}, K2a, back {K2, history, K3, finish} */
	host_mem<vdl2_chunk_args> h_args; dev_mem<vdl2_chunk_args> d_args;
	/* ragged spans: the span's receiver table (vdl2_rx_span_table; pinned host copy, device copy made with the arguments) */
	host_mem<vdl2_rx_span> h_span; dev_mem<vdl2_rx_span> d_span;
	/* ragged spans that restart receivers (vdl2gpu_restart_receiver): per channel slot, whether it starts afresh with this
	 * span and its new tuning (pinned host copy, device copy made with the span's table); such a span takes the direct
	 * path, so the graphs of ordinary spans never see the table */
	host_mem<vdl2_rx_restart> h_restart; dev_mem<vdl2_rx_restart> d_restart;
	bool restart = false;
	/* pushed spans (vdl2gpu_submit_pushed): K0 reads the receivers' rings; k0_done is recorded after it (ragged contexts) */
	bool pushed = false;
	event_h k0_done;
	/* spectrum (VDL2GPU_FLAG_SPECTRUM): per input, the samples it holds and brings to this chunk (pinned host copy, device
	 * copy made right before the spectrum kernel) */
	host_mem<vdl2_spec_span> h_spec; dev_mem<vdl2_spec_span> d_spec;
	graph_exec_h g_front[6], g_k2a[6], g_back[6];      /* index = chunk number mod 6 (dec buffer, plane) */
	uint32_t graph_pairs[6] = { 0 };
	uint64_t first_pair = 0, dec_base = 0;
	uint32_t n_pairs = 0, n_dec = 0;
	struct timeval arrival = { 0, 0 };
};

/* Pushed input of one receiver (vdl2gpu_push).  Stream positions as in vdl2_core.cuh: head, tail, freed.  A fence says
 * that once `ev` has completed, every byte before `pos` has been read by whatever copy or K0 needed it. */
struct ring_fence { cudaEvent_t ev; uint64_t pos; };
struct push_rec { uint64_t end; double t; };                /* a push: the stream position it ended at, its arrival time */
struct span_anchor { uint64_t dec_base, byte_base; uint32_t n; };   /* a pushed span took groups [dec_base, + n) from byte_base on */
struct push_rx {
	std::mutex m;                                       /* head, tail, freed, fences, recs (pushes of this receiver and the control thread) */
	std::condition_variable room;                       /* a push waiting for the control thread to take its queue into spans */
	uint64_t head = 0, tail = 0, freed = 0;
	std::deque<ring_fence> fences;
	std::deque<push_rec> recs;
	std::deque<span_anchor> anchors;                    /* (control thread only) */
};

/* the pushed-input rings of one receiver list (ragged contexts, allocated by the first vdl2gpu_push): the receivers' rings
 * (vdl2_push_ring_layout) in device memory, their pinned host mirror and table, and per receiver its queue state */
struct push_rings {
	dev_mem<uint8_t> d_rings;
	host_mem<uint8_t> h_rings;
	std::vector<vdl2_rx_ring> rings;
	dev_mem<vdl2_rx_ring> d_ring_tab;
	std::vector<std::unique_ptr<push_rx>> push;
};

/* The part of a context that follows from its channels and receivers (setup_layout): vdl2gpu_update_receivers builds a new
 * one and swaps it in whole. */
struct ctx_layout {
	std::vector<uint32_t> freqs;
	uint32_t n_ch = 0, n_chp = 0, max_pairs = 0, max_dec = 0, n_slots = 0, out_cap = 0;
	uint32_t lanes = 32, full_warps = 0xFFFFFFFFu;      /* channel slot mapping (see setup_layout) */
	uint32_t n_streams = 1;                             /* inputs: streams, or receivers */
	dev_mem<uint32_t> d_slot_rx, d_block_rx;            /* receivers: vdl2_rx_layout tables */
	uint32_t rx_tile = 0, rx_max = 0;                   /* receivers: samples per staged tile, most receivers of one K1 block */
	/* mixed-rate receivers (vdl2gpu_create_mixed_receivers): every receiver has its own oversample factor and format, and
	 * the chain counts DECIMATED samples (n_pairs of a chunk = n_dec of a span, decimation counter always 0); rx_tile is
	 * then the decimation groups of a staged tile */
	std::vector<vdl2_rx_input> rx_in;                   /* per receiver: oversample, format, byte offset per decimated sample */
	dev_mem<vdl2_rx_input> d_rx_in;
	dev_mem<uint8_t> d_slot_cls;                        /* slot -> rate class (vdl2_rx_class) of its receiver */
	uint64_t span_bytes_per_dec = 0, span_pairs_per_dec = 0;   /* sums over the receivers of os x bytes per sample, of os */
	uint32_t max_span = 0, rx_os_max = 0, cls_mask = 0;  /* largest n_dec of a span; largest oversample; rate classes present */
	float cls_taps[3][5] = {};                          /* {a0, a1, a2, b1, b2} per rate class (10, 13, 20) */
	/* ragged spans (VDL2GPU_FLAG_RAGGED on a mixed context): every receiver brings its own count n_r to a span; the chain then
	 * counts the span's width (the largest n_r) and each kernel lane takes its receiver's entry of the span's table */
	std::vector<uint64_t> rx_pos;                       /* per receiver: decimated samples accepted so far */
	std::vector<uint32_t> rx_prev;                      /* per receiver: its count in the previous span */
	std::vector<uint32_t> ch_rx;                        /* per channel: its receiver (burst timestamps) */
	/* restarts (vdl2gpu_restart_receiver): every receiver's current centre and first channel, and the receivers whose
	 * restart waits for the next span that runs */
	std::vector<uint32_t> rx_centre, rx_first;
	std::vector<uint8_t> rx_restart_pending;
	uint32_t n_restart_pending = 0;
	dev_mem<float2> d_samples;
	dev_mem<float2> d_dec3[3];
	dev_mem<float> d_phase2[2], d_mag2[2];
	dev_mem<uint32_t> d_k1, d_k2, d_counters, d_ready;
	dev_mem<float> d_ring;
	dev_mem<vdl2_burst_slot> d_pool;
	dev_mem<int32_t> d_free;
	dev_mem<vdl2_queue_ctl> d_ctl;
	/* input levels (VDL2GPU_FLAG_INPUT_LEVELS; NULL otherwise): one accumulator per input (stream or receiver), which the
	 * levels form of K0 adds every converted sample to */
	dev_mem<vdl2_levels> d_levels;
	/* channel levels (VDL2GPU_FLAG_CHANNEL_LEVELS; NULL otherwise): the per-slot planes the levels form of K2a adds every
	 * decimated sample to, uint64 [VDL2_CHLV_ROWS][n_chp] then the uint32 peak plane [n_chp] */
	dev_mem<uint64_t> d_chlv;
	/* spectrum (VDL2GPU_FLAG_SPECTRUM; NULL / empty otherwise): per input its accumulators and waiting samples, the window and
	 * twiddle tables, and per input its position on its segment grid (samples since the grid's origin: create, joining,
	 * restart); inputs whose figures a restart zeroes at the start of the next span */
	dev_mem<vdl2_spec_acc> d_spec;
	dev_mem<vdl2_spec_tab> d_spec_tab;
	std::vector<uint64_t> spec_pos;
	std::vector<uint32_t> spec_zero;
	std::vector<chunk_slot> chunks;
};

struct vdl2gpu_ctx : ctx_layout, push_rings {
	/* the config create was given, max_chunk_bytes and n_inflight defaulted; its channel fields (freqs, n_channels,
	 * n_streams) are create's input only: the layout holds the current ones */
	vdl2gpu_config cfg;
	int device = 0;
	/* `stream` (front) carries H2D + K0 + K1 of chunk c+1 while `s_back` carries K2a/K2/K3 of chunk c.  Both stages
	 * are latency-bound with one warp per SM sub-partition at 16 k channels, so co-residency raises issue-slot use.
	 * This only works because every kernel of the chain requests the SAME
	 * shared-memory carve-out (vdl2_kernels.cu): with per-kernel defaults the SMs drain to re-partition L1/shared
	 * memory and the overlap is a 1.7x slow-down.  VDL2GPU_FLAG_NO_OVERLAP puts everything on one stream.
	 * s_back and s_mid alias `stream`, back_stream or mid_stream, whichever create made for them. */
	stream_h stream, back_stream, mid_stream;
	cudaStream_t s_mid = nullptr, s_back = nullptr;
	/* three stages, three chunks in flight: K0+K1 of chunk c+2 (front), K2a of chunk c+1 (mid), K2+K3 of chunk c (back).
	 * dec is triple-buffered (written by K1, read by K2a and K2), the phase / magnitude planes alternate (written by K2a,
	 * read by K2; K2a of chunk c takes its 160 history rows from the other plane, i.e. from chunk c-1). */
	event_h ev_k1_done[3], ev_back_done[3], ev_k2a_done[2];
	uint64_t chunk_seq = 0;
	event_h ev_input_ready, ev_input_consumed;
	uint32_t event_cap = 0;
	uint64_t events_dropped = 0;                        /* trace events lost to a full buffer, not yet reported by vdl2gpu_read_events */
	int n_sms = 0;                                      /* read from the device at create */
	uint32_t ch_per_stream = 0;                         /* independent-streams mode: n_streams > 1, channels [s*C, (s+1)*C) on stream s */
	bool lane_streams = false;                          /* C == 1: samples kept time-major across streams, one lane per stream in K1 */
	bool receivers = false;                             /* vdl2gpu_create_receivers: n_streams receivers, each with its own centre and channels */
	bool mixed = false;                                 /* vdl2gpu_create_mixed_receivers (see ctx_layout) */
	bool ragged = false;                                /* VDL2GPU_FLAG_RAGGED (see ctx_layout) */
	uint32_t raw_bytes = 0;                             /* size of each slot's raw staging buffers (allocated on the first host submit) */
	int k1_variant = 2, k2_variant = 5, k2a_mode = 1;   /* A/B knobs (VDL2GPU_K1_VARIANT, VDL2GPU_K2_VARIANT, VDL2GPU_K2A), read at create */
	bool use_graphs = true;
	uint32_t k2a_split = 64;                            /* time slices of the K2a grid (VDL2GPU_K2A_SPLIT) */
	int stages = 2;                                     /* 2: K2a runs alone between K1 of chunk c and K1 of chunk c+1 (default, see run_chain);
	                                                     * 3: K2a of chunk c+1 beside K1 of chunk c+2 and K2 of chunk c (VDL2GPU_STAGES=3) */
	uint64_t overflows_reported = 0;
	host_tables tab;
	dev_mem<vdl2_tables> d_tab;
	dev_mem<vdl2gpu_event> d_events;
	std::deque<uint32_t> inflight;
	uint32_t next_slot = 0;
	uint32_t decim_cnt = 0, last_n_dec = 0;
	uint64_t total_pairs = 0, total_dec = 0;
	uint32_t events_read = 0;
	bool timing = false;
	double k_ms[5] = { 0, 0, 0, 0, 0 };                 /* K0, K1, K2a, K2 (+history copy), K3 (+finish) */
	uint64_t k_launches[5] = { 0, 0, 0, 0, 0 };
	dev_mem<vdl2_block_trace> d_block_trace;            /* VDL2GPU_BLOCK_TRACE=1: per-block scheduling records of K1 / K2 */
	uint32_t block_trace_cap = 0;
	uint32_t graph_nominal = 0;                         /* chunk shape (n_pairs) the graphs are kept for */
	event_h ev_t0;                                      /* origin of the timeline (recorded by vdl2gpu_enable_timing) */
	std::vector<float> timeline;                        /* 8 floats per timed chunk: chunk number, then the 7 stage boundaries in ms since ev_t0 */
	vdl2gpu_stats stats;
	std::vector<pending_frame> pending;
	std::vector<std::vector<uint8_t>> blobs;
	event_h ev_drain;
	/* pushed input: the rings are push_rings; here the copy stream every push issues its copies on, the event a restart
	 * records there when it drops queued bytes, and whether the rings exist */
	std::mutex push_alloc;
	std::atomic<bool> push_ready{false};
	stream_h s_copy;
	event_h ev_copied, ev_dropped;
};

static void initial_state(const vdl2gpu_config &cfg, const uint32_t *freqs, const uint32_t *centres, const uint32_t *rates, uint32_t n_ch,
		uint32_t n_chp, uint32_t lanes, uint32_t full_warps, std::vector<uint32_t> &k1, std::vector<uint32_t> &k2);
/* channel -> slot: the first full_warps warps hold `lanes` channels each, the others lanes - 1 */
static inline uint32_t slot_of(uint32_t ch, uint32_t lanes, uint32_t full_warps) { return vdl2_channel_slot(ch, lanes, full_warps); }
/* the noise floor in dBFS, of a frame and of vdl2gpu_get_channel_levels (src/decode.c:181) */
static inline float nf_pwr_dbfs(float mag_nf) { return 20.0f * log10f(mag_nf + 0.001f); }

extern "C" int vdl2gpu_abi_version(void) { return VDL2GPU_ABI_VERSION; }

extern "C" int vdl2gpu_device_count(void) {
	int n = 0;
	if(cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
	return n;
}

extern "C" const char *vdl2gpu_last_error(void) { return g_last_error; }

extern "C" const char *vdl2gpu_strerror(int code) {
	switch(code) {
		case VDL2GPU_OK: return "ok";
		case VDL2GPU_EINVAL: return "invalid argument";
		case VDL2GPU_ENODEV: return "no usable CUDA device";
		case VDL2GPU_ECUDA: return "CUDA runtime error";
		case VDL2GPU_ENOMEM: return "out of memory";
		case VDL2GPU_ETOOBIG: return "chunk larger than max_chunk_bytes";
		case VDL2GPU_EOVERFLOW: return "device queue overflow, bursts dropped";
		default: return "unknown error";
	}
}

static int free_ctx(vdl2gpu_ctx *c) {
	if(!c) return VDL2GPU_OK;
	cudaSetDevice(c->device);
	/* nothing runs once every stream is idle: the handles may then go in any order */
	if(c->stream) cudaStreamSynchronize(c->stream);
	if(c->s_mid) cudaStreamSynchronize(c->s_mid);
	if(c->s_back) cudaStreamSynchronize(c->s_back);
	if(c->s_copy) cudaStreamSynchronize(c->s_copy);
	delete c;
	return VDL2GPU_OK;
}

/* The part of a context that follows from its channels and receivers: the channel slot mapping, span and chunk sizes,
 * burst-pool size, output capacity, receiver tables, per-receiver host records, and every device buffer and chunk slot
 * sized by them, built into the empty layout L.  Create and vdl2gpu_update_receivers both build it here, so the two cannot
 * drift apart.  The checks come first: an EINVAL or ETOOBIG return has touched no device.  The contents of the state
 * planes, the free list and the queue control block are left to the caller.  cfg: the channels, the inputs (n_streams,
 * resolved as in create_impl), the flags, max_chunk_bytes and n_inflight with create's defaults, and for a single-rate
 * context its sample format and oversample factor; rx / n_rx / rx_ex and the context kind as for create_impl; n_sms: the
 * device's SMs.  The pool holds at least min_slots slots. */
static int setup_layout(ctx_layout &L, const vdl2gpu_config &cfg, const vdl2gpu_receiver *rx, uint32_t n_rx,
		const vdl2gpu_receiver_ex *rx_ex, bool receivers, bool mixed, bool ragged, bool lane_streams, int n_sms,
		uint32_t min_slots, const char *what) {
	L.freqs.assign(cfg.freqs, cfg.freqs + cfg.n_channels);
	L.n_ch = cfg.n_channels;
	L.n_chp = (L.n_ch + 31u) & ~31u;
	L.n_streams = cfg.n_streams;
	/* Slot mapping.  K1 and K2 run four-warp blocks, one warp per SM sub-partition, and a chunk's K2 overlaps the next
	 * chunk's K1.  The block scheduler places a new block on the SM with the most free resources: when a grid leaves SMs
	 * empty (128 blocks on 132 SMs at 16384 channels), the OTHER kernel's blocks pile up on those SMs two and three deep
	 * instead of sitting beside the first kernel's blocks, one per SM, and run two to three times slower (measured with
	 * the per-block trace, tools/block_trace.py).  So when the channels fill more than half of the machine's
	 * sub-partitions, they are dealt out evenly over ALL of them: every warp holds floor or ceil of n_ch / (4 x SMs)
	 * channels instead of 32 (31 or 32 at 16384 channels on 132 SMs), each of the two kernels launches exactly one block
	 * per SM, every block lives for the whole kernel, and every SM looks the same to the scheduler. */
	if(receivers || cfg.n_streams <= 1 || cfg.n_streams == cfg.n_channels) {
		const uint32_t warps_all = 4u * (uint32_t)n_sms;
		if(L.n_ch > 16u * warps_all && L.n_ch <= 32u * warps_all) {
			const char *e = getenv("VDL2GPU_BALANCE");
			if(!e || atoi(e)) {
				L.lanes = (L.n_ch + warps_all - 1u) / warps_all;
				L.full_warps = L.n_ch - (L.lanes - 1u) * warps_all;       /* warps with `lanes` channels; the rest have lanes - 1 */
				L.n_chp = warps_all * 32u;
			}
		}
	}
	const uint32_t max_bytes = cfg.max_chunk_bytes;
	if(mixed) {
		/* the largest span: every receiver's buffer within max_chunk_bytes; the plane's row stride holds the longest row */
		uint32_t bpd_max = 0;
		for(uint32_t r = 0; r < n_rx; r++) {
			bpd_max = std::max(bpd_max, rx_ex[r].oversample * (rx_ex[r].sample_fmt == VDL2GPU_FMT_S16_LE ? 4u : 2u));
			L.rx_os_max = std::max(L.rx_os_max, rx_ex[r].oversample);
		}
		L.max_span = max_bytes / bpd_max;
		if(L.max_span == 0) {
			snprintf(g_last_error, sizeof(g_last_error), "%s: max_chunk_bytes (%u) holds less than one decimated sample of a receiver (%u bytes)",
					what, max_bytes, bpd_max);
			return VDL2GPU_EINVAL;
		}
		L.max_pairs = (L.max_span * L.rx_os_max + 1u) & ~1u;       /* even row stride: every row of the plane starts 16-byte aligned */
		L.max_dec = L.max_span + 2;
	} else {
		L.max_pairs = max_bytes / (cfg.sample_fmt == VDL2GPU_FMT_S16_LE ? 4u : 2u);
		if(receivers) L.max_pairs = (L.max_pairs + 1u) & ~1u;     /* even row stride: every receiver row of the plane starts 16-byte aligned */
		L.max_dec = L.max_pairs / cfg.oversample + 2;
	}
	if((uint64_t)(L.max_dec + VDL2_SYNC_BUFLEN) * L.n_chp >= (1ull << 32)) {
		snprintf(g_last_error, sizeof(g_last_error), "%u channels x %u decimated samples per chunk exceed the 32-bit element index of the kernels; "
				"use a smaller max_chunk_bytes or shard the channels", L.n_ch, L.max_dec);
		return VDL2GPU_ETOOBIG;
	}
	L.n_slots = std::max(std::max(256u, 3u * L.n_ch), min_slots);
	L.out_cap = std::max(4u << 20, L.n_ch * 512u);

	/* receiver tables (host side) */
	std::vector<uint32_t> slot_rx, block_rx;
	std::vector<uint8_t> slot_cls;
	if(receivers) {
		/* the slot -> receiver tables K1 stages by */
		std::vector<uint32_t> rx_first(n_rx + 1, 0);
		for(uint32_t r = 0; r < n_rx; r++) rx_first[r + 1] = rx_first[r] + rx[r].n_channels;
		const uint32_t n_blocks = (L.n_chp + VDL2_RX_K1_BLOCK - 1) / VDL2_RX_K1_BLOCK;
		slot_rx.resize((size_t)n_blocks * VDL2_RX_K1_BLOCK); block_rx.resize(2 * (size_t)n_blocks);
		L.rx_max = vdl2_rx_layout(n_blocks, L.lanes, L.full_warps, L.n_ch, rx_first.data(), n_rx, slot_rx.data(), block_rx.data());
		L.rx_tile = mixed ? vdl2_rx_mixed_tile_groups(L.rx_max, L.rx_os_max) : vdl2_rx_tile_samples(L.rx_max, cfg.oversample);
		if(mixed) {
			/* per receiver: oversample, format, place in a span; per slot: rate class; per class: the filter taps of
			 * input_lpf_init(105000 x os) (src/demod.c:367-370) */
			std::vector<uint32_t> os(n_rx), fmt(n_rx);
			for(uint32_t r = 0; r < n_rx; r++) { os[r] = rx_ex[r].oversample; fmt[r] = rx_ex[r].sample_fmt; }
			L.rx_in.resize(n_rx);
			L.span_bytes_per_dec = vdl2_rx_span_layout(os.data(), fmt.data(), n_rx, L.rx_in.data());
			for(uint32_t r = 0; r < n_rx; r++) {
				L.span_pairs_per_dec += os[r];
				L.cls_mask |= 1u << vdl2_rx_class(os[r]);
			}
			static const uint32_t class_os[3] = { 10, 13, 20 };
			for(int k = 0; k < 3; k++) {
				float A[3], B[3];
				make_lpf((uint32_t)VDL2_SYMBOL_RATE * VDL2_SPS * class_os[k], A, B);
				L.cls_taps[k][0] = A[0]; L.cls_taps[k][1] = A[1]; L.cls_taps[k][2] = A[2]; L.cls_taps[k][3] = B[1]; L.cls_taps[k][4] = B[2];
			}
			slot_cls.resize(slot_rx.size());
			for(size_t s = 0; s < slot_rx.size(); s++) slot_cls[s] = (uint8_t)vdl2_rx_class(os[slot_rx[s]]);
		}
		if(ragged) {
			L.rx_pos.assign(n_rx, 0);
			L.rx_prev.assign(n_rx, 0);
			L.ch_rx.resize(L.n_ch);
			for(uint32_t r = 0; r < n_rx; r++) std::fill(L.ch_rx.begin() + rx_first[r], L.ch_rx.begin() + rx_first[r + 1], r);
			L.rx_first = rx_first;
			L.rx_centre.resize(n_rx);
			for(uint32_t r = 0; r < n_rx; r++) L.rx_centre[r] = rx[r].centerfreq;
			L.rx_restart_pending.assign(n_rx, 0);
			L.n_restart_pending = 0;
		}
	}

	/* device buffers */
	if(lane_streams) CU(cudaMalloc(L.d_samples.put(), (size_t)L.max_pairs * L.n_chp * sizeof(float2)));
	else CU(cudaMalloc(L.d_samples.put(), (size_t)L.n_streams * L.max_pairs * sizeof(float2)));
	for(int i = 0; i < 3; i++) {
		CU(cudaMalloc(L.d_dec3[i].put(), (size_t)L.max_dec * L.n_chp * sizeof(float2)));
		CU(cudaMemset(L.d_dec3[i], 0, (size_t)L.max_dec * L.n_chp * sizeof(float2)));
	}
	for(int i = 0; i < 2; i++) {
		CU(cudaMalloc(L.d_phase2[i].put(), (size_t)(L.max_dec + VDL2_SYNC_BUFLEN) * L.n_chp * sizeof(float)));
		CU(cudaMemset(L.d_phase2[i], 0, (size_t)(L.max_dec + VDL2_SYNC_BUFLEN) * L.n_chp * sizeof(float)));
		CU(cudaMalloc(L.d_mag2[i].put(), (size_t)L.max_dec * L.n_chp * sizeof(float)));
	}
	CU(cudaMalloc(L.d_k1.put(), (size_t)K1_NFIELDS * L.n_chp * 4));
	CU(cudaMalloc(L.d_k2.put(), (size_t)K2_NFIELDS * L.n_chp * 4));
	CU(cudaMalloc(L.d_counters.put(), (size_t)VDL2_NUM_COUNTERS * L.n_chp * 4));
	CU(cudaMalloc(L.d_ring.put(), (size_t)VDL2_SYNC_BUFLEN * L.n_chp * 4));
	CU(cudaMalloc(L.d_pool.put(), (size_t)L.n_slots * sizeof(vdl2_burst_slot)));
	CU(cudaMalloc(L.d_free.put(), (size_t)L.n_slots * 4));
	CU(cudaMalloc(L.d_ready.put(), (size_t)L.n_slots * 4));
	CU(cudaMalloc(L.d_ctl.put(), sizeof(vdl2_queue_ctl)));
	CU(cudaMemset(L.d_counters, 0, (size_t)VDL2_NUM_COUNTERS * L.n_chp * 4));
	CU(cudaMemset(L.d_ring, 0, (size_t)VDL2_SYNC_BUFLEN * L.n_chp * 4));
	CU(cudaMemset(L.d_pool, 0, (size_t)L.n_slots * sizeof(vdl2_burst_slot)));
	if(receivers) {
		CU(cudaMalloc(L.d_slot_rx.put(), slot_rx.size() * 4));
		CU(cudaMalloc(L.d_block_rx.put(), block_rx.size() * 4));
		CU(cudaMemcpy(L.d_slot_rx, slot_rx.data(), slot_rx.size() * 4, cudaMemcpyHostToDevice));
		CU(cudaMemcpy(L.d_block_rx, block_rx.data(), block_rx.size() * 4, cudaMemcpyHostToDevice));
	}
	if(cfg.flags & VDL2GPU_FLAG_INPUT_LEVELS) {
		CU(cudaMalloc(L.d_levels.put(), (size_t)L.n_streams * sizeof(vdl2_levels)));
		CU(cudaMemset(L.d_levels, 0, (size_t)L.n_streams * sizeof(vdl2_levels)));
	}
	if(cfg.flags & VDL2GPU_FLAG_CHANNEL_LEVELS) {
		const size_t bytes = (size_t)VDL2_CHLV_ROWS * L.n_chp * 8 + (size_t)L.n_chp * 4;
		CU(cudaMalloc(L.d_chlv.put(), bytes));
		CU(cudaMemset(L.d_chlv, 0, bytes));
	}
	if(cfg.flags & VDL2GPU_FLAG_SPECTRUM) {
		CU(cudaMalloc(L.d_spec.put(), (size_t)L.n_streams * sizeof(vdl2_spec_acc)));
		CU(cudaMemset(L.d_spec, 0, (size_t)L.n_streams * sizeof(vdl2_spec_acc)));
		std::unique_ptr<vdl2_spec_tab> tab(new vdl2_spec_tab);
		vdl2_spec_make_tab(tab.get());
		CU(cudaMalloc(L.d_spec_tab.put(), sizeof(vdl2_spec_tab)));
		CU(cudaMemcpy(L.d_spec_tab, tab.get(), sizeof(vdl2_spec_tab), cudaMemcpyHostToDevice));
		L.spec_pos.assign(L.n_streams, 0);
		L.spec_zero.clear();
	}
	if(mixed) {
		CU(cudaMalloc(L.d_rx_in.put(), L.rx_in.size() * sizeof(vdl2_rx_input)));
		CU(cudaMalloc(L.d_slot_cls.put(), slot_cls.size()));
		CU(cudaMemcpy(L.d_rx_in, L.rx_in.data(), L.rx_in.size() * sizeof(vdl2_rx_input), cudaMemcpyHostToDevice));
		CU(cudaMemcpy(L.d_slot_cls, slot_cls.data(), slot_cls.size(), cudaMemcpyHostToDevice));
	}

	L.chunks.resize(cfg.n_inflight);
	for(auto &s : L.chunks) {
		/* h_raw / d_raw (max_chunk_bytes x n_streams each) are allocated by the first vdl2gpu_submit: hosts that only
		 * use vdl2gpu_submit_device never need them */
		CU(cudaHostAlloc((void **)s.h_args.put(), sizeof(vdl2_chunk_args), cudaHostAllocDefault));
		CU(cudaMalloc(s.d_args.put(), sizeof(vdl2_chunk_args)));
		if(ragged) {
			CU(cudaHostAlloc((void **)s.h_span.put(), (size_t)n_rx * sizeof(vdl2_rx_span), cudaHostAllocDefault));
			CU(cudaMalloc(s.d_span.put(), (size_t)n_rx * sizeof(vdl2_rx_span)));
			CU(cudaHostAlloc((void **)s.h_restart.put(), (size_t)L.n_chp * sizeof(vdl2_rx_restart), cudaHostAllocDefault));
			CU(cudaMalloc(s.d_restart.put(), (size_t)L.n_chp * sizeof(vdl2_rx_restart)));
			CU(cudaEventCreateWithFlags(s.k0_done.put(), cudaEventDisableTiming));
		}
		CU(cudaHostAlloc((void **)s.h_out.put(), sizeof(vdl2_out_header) + L.out_cap, cudaHostAllocMapped));
		CU(cudaHostGetDevicePointer((void **)&s.d_out, s.h_out, 0));
		if(L.d_spec) {
			CU(cudaHostAlloc((void **)s.h_spec.put(), (size_t)L.n_streams * sizeof(vdl2_spec_span), cudaHostAllocDefault));
			CU(cudaMalloc(s.d_spec.put(), (size_t)L.n_streams * sizeof(vdl2_spec_span)));
		}
		memset(s.h_out, 0, sizeof(vdl2_out_header));
		CU(cudaEventCreateWithFlags(s.done.put(), cudaEventDisableTiming));
		for(auto &ev : s.tk) CU(cudaEventCreate(ev.put()));
	}
	return VDL2GPU_OK;
}

/* rx / n_rx: the receivers of a multi-receiver context (vdl2gpu_create_receivers, validated there), NULL / 0 otherwise;
 * rx_ex: the same receivers with their oversample factors and formats (vdl2gpu_create_mixed_receivers), NULL otherwise */
static int create_impl(const vdl2gpu_config *cfg, vdl2gpu_ctx *c, const vdl2gpu_receiver *rx = nullptr, uint32_t n_rx = 0,
		const vdl2gpu_receiver_ex *rx_ex = nullptr) {
	int ndev = 0;
	cudaError_t e = cudaGetDeviceCount(&ndev);
	if(e != cudaSuccess || ndev == 0) {
		cudaGetLastError();
		snprintf(g_last_error, sizeof(g_last_error), "no CUDA device (%s); libvdl2gpu has no CPU fallback",
				e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
		return VDL2GPU_ENODEV;
	}
	if(cfg->device >= 0) { c->device = cfg->device; CU(cudaSetDevice(c->device)); }
	else CU(cudaGetDevice(&c->device));
	cudaDeviceProp prop;
	CU(cudaGetDeviceProperties(&prop, c->device));
	if(prop.major != 9 || prop.minor != 0) {        /* sm_90a code loads on compute capability 9.0 only */
		snprintf(g_last_error, sizeof(g_last_error), "device %d is sm_%d%d; this library carries sm_90a code only", c->device, prop.major, prop.minor);
		return VDL2GPU_ENODEV;
	}
	KL(vdl2_kernels_init_device(c->device));             /* per device: function attributes do not carry over */
	c->cfg = *cfg;
	c->receivers = rx != nullptr;
	c->mixed = rx_ex != nullptr;
	c->ragged = c->mixed && (cfg->flags & VDL2GPU_FLAG_RAGGED);
	const uint32_t n_streams = c->receivers ? n_rx : cfg->n_streams ? cfg->n_streams : 1u;
	c->cfg.n_streams = n_streams;
	c->lane_streams = !c->receivers && n_streams > 1 && n_streams == cfg->n_channels;     /* one stream per channel */
	if(c->lane_streams) {
		c->ch_per_stream = 1;
	} else if(n_streams > 1 && !c->receivers) {         /* (receivers: any channel count each, see the receiver tables below) */
		if(cfg->n_channels % n_streams != 0 || (cfg->n_channels / n_streams) % 32u != 0) {
			snprintf(g_last_error, sizeof(g_last_error), "independent-streams mode needs n_channels = n_streams x C with C = 1 or a multiple of 32 (got %u channels, %u streams)",
					cfg->n_channels, n_streams);
			return VDL2GPU_EINVAL;
		}
		c->ch_per_stream = cfg->n_channels / n_streams;
	}
	{
		const char *e;
		if((e = getenv("VDL2GPU_K1_VARIANT"))) c->k1_variant = atoi(e);
		if((e = getenv("VDL2GPU_K2_VARIANT"))) c->k2_variant = atoi(e);
		if((e = getenv("VDL2GPU_K2A"))) c->k2a_mode = atoi(e);
		if((e = getenv("VDL2GPU_NO_GRAPH")) && atoi(e)) c->use_graphs = false;
		if((e = getenv("VDL2GPU_BLOCK_TRACE")) && atoi(e)) c->block_trace_cap = 1u << 16;
		if((e = getenv("VDL2GPU_STAGES")) && atoi(e) == 3) { c->stages = 3; c->k2a_split = 3; }
		if((e = getenv("VDL2GPU_K2A_SPLIT")) && atoi(e) >= 1 && atoi(e) <= 256) c->k2a_split = (uint32_t)atoi(e);
	}
	if(cfg->flags & (VDL2GPU_FLAG_NO_GRAPH | VDL2GPU_FLAG_TRACE)) c->use_graphs = false;
	c->n_sms = prop.multiProcessorCount;
	c->cfg.max_chunk_bytes = cfg->max_chunk_bytes ? cfg->max_chunk_bytes : (1u << 20);
	c->cfg.n_inflight = cfg->n_inflight ? cfg->n_inflight : 4u;
	c->event_cap = (cfg->flags & VDL2GPU_FLAG_TRACE) ? (1u << 20) : 1u;
	ctx_layout L;
	int rc = setup_layout(L, c->cfg, rx, n_rx, rx_ex, c->receivers, c->mixed, c->ragged, c->lane_streams, c->n_sms, 0,
			c->mixed ? "vdl2gpu_create_mixed_receivers" : c->receivers ? "vdl2gpu_create_receivers" : "vdl2gpu_create");
	if(rc) return rc;
	static_cast<ctx_layout &>(*c) = std::move(L);
	c->cfg.freqs = nullptr;                             /* the caller's array: the layout holds a copy */
	/* (mixed receivers: the rate only enters the filter taps of these tables, which the mixed K1 takes per rate class) */
	make_tables(c->tab, c->mixed ? (uint32_t)VDL2_SYMBOL_RATE * VDL2_SPS * c->rx_os_max : cfg->sample_rate);
	memset(&c->stats, 0, sizeof(c->stats));

	/* equal (default) priorities: raising either stage's priority slowed the pair down (tools/probe_overlap.py) */
	CU(cudaStreamCreateWithFlags(c->stream.put(), cudaStreamNonBlocking));
	if(cfg->flags & VDL2GPU_FLAG_NO_OVERLAP) { c->s_back = c->stream; c->s_mid = c->stream; }
	else {
		CU(cudaStreamCreateWithFlags(c->back_stream.put(), cudaStreamNonBlocking));
		c->s_back = c->back_stream;
		if(c->stages == 3) CU(cudaStreamCreateWithFlags(c->mid_stream.put(), cudaStreamNonBlocking));
		c->s_mid = c->stages == 3 ? c->mid_stream : c->back_stream;
	}
	for(int i = 0; i < 2; i++) CU(cudaEventCreateWithFlags(c->ev_k2a_done[i].put(), cudaEventDisableTiming));
	for(int i = 0; i < 3; i++) {
		CU(cudaEventCreateWithFlags(c->ev_k1_done[i].put(), cudaEventDisableTiming));
		CU(cudaEventCreateWithFlags(c->ev_back_done[i].put(), cudaEventDisableTiming));
	}
	CU(cudaEventCreateWithFlags(c->ev_input_ready.put(), cudaEventDisableTiming));
	CU(cudaEventCreateWithFlags(c->ev_input_consumed.put(), cudaEventDisableTiming));
	CU(cudaEventCreateWithFlags(c->ev_drain.put(), cudaEventDisableTiming));
	if(c->block_trace_cap) {
		const size_t bytes = sizeof(vdl2_block_trace) + (size_t)c->block_trace_cap * sizeof(vdl2_block_rec);
		CU(cudaMalloc(c->d_block_trace.put(), bytes));
		CU(cudaMemset(c->d_block_trace, 0, bytes));
		CU(cudaMemcpy(&c->d_block_trace->cap, &c->block_trace_cap, 4, cudaMemcpyHostToDevice));
	}
	CU(cudaMalloc(c->d_tab.put(), sizeof(vdl2_tables)));
	CU(cudaMemcpy(c->d_tab, &c->tab.t, sizeof(vdl2_tables), cudaMemcpyHostToDevice));
	CU(cudaMalloc(c->d_events.put(), (size_t)c->event_cap * sizeof(vdl2gpu_event)));

	std::vector<uint32_t> k1, k2, centres, rates;
	if(c->receivers) {
		/* every channel mixes against its own receiver's centre (src/demod.c:385) */
		for(uint32_t r = 0; r < n_rx; r++) {
			centres.insert(centres.end(), rx[r].n_channels, rx[r].centerfreq);
			if(c->mixed) rates.insert(rates.end(), rx[r].n_channels, (uint32_t)VDL2_SYMBOL_RATE * VDL2_SPS * rx_ex[r].oversample);
		}
	}
	initial_state(c->cfg, c->freqs.data(), c->receivers ? centres.data() : nullptr, c->mixed ? rates.data() : nullptr, c->n_ch, c->n_chp,
			c->lanes, c->full_warps, k1, k2);
	CU(cudaMemcpy(c->d_k1, k1.data(), k1.size() * 4, cudaMemcpyHostToDevice));
	CU(cudaMemcpy(c->d_k2, k2.data(), k2.size() * 4, cudaMemcpyHostToDevice));
	std::vector<int32_t> fl(c->n_slots);
	for(uint32_t i = 0; i < c->n_slots; i++) fl[i] = (int32_t)i;
	CU(cudaMemcpy(c->d_free, fl.data(), fl.size() * 4, cudaMemcpyHostToDevice));
	vdl2_queue_ctl ctl;
	memset(&ctl, 0, sizeof(ctl));
	ctl.free_top = (int32_t)c->n_slots;
	CU(cudaMemcpy(c->d_ctl, &ctl, sizeof(ctl), cudaMemcpyHostToDevice));
	return VDL2GPU_OK;
}

/* VDL2GPU_FLAG_RAGGED outside vdl2gpu_create_mixed_receivers: refused rather than ignored, since ignoring it would give the
 * caller lock-step spans they did not ask for */
static int refuse_ragged(const char *what) {
	snprintf(g_last_error, sizeof(g_last_error), "%s: VDL2GPU_FLAG_RAGGED needs vdl2gpu_create_mixed_receivers "
			"(a uniform fleet gets ragged spans by describing itself there)", what);
	return VDL2GPU_EINVAL;
}

extern "C" int vdl2gpu_create(const vdl2gpu_config *cfg, vdl2gpu_ctx **out) {
	if(!cfg || !out || !cfg->freqs || cfg->n_channels == 0 || cfg->oversample == 0 || cfg->sample_fmt > 1
			|| cfg->sample_rate != (uint32_t)VDL2_SYMBOL_RATE * VDL2_SPS * cfg->oversample) {
		snprintf(g_last_error, sizeof(g_last_error), "bad vdl2gpu_config (sample_rate must be 105000*oversample)");
		return VDL2GPU_EINVAL;
	}
	if(cfg->flags & VDL2GPU_FLAG_RAGGED) return refuse_ragged("vdl2gpu_create");
	vdl2gpu_ctx *c = new vdl2gpu_ctx();
	int rc = create_impl(cfg, c);
	if(rc != VDL2GPU_OK) { free_ctx(c); *out = nullptr; return rc; }
	*out = c;
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_create_receivers(const vdl2gpu_config *cfg, const vdl2gpu_receiver *rx, uint32_t n_rx, vdl2gpu_ctx **out) {
	const char *why = nullptr;
	uint64_t sum = 0;
	if(!cfg || !out || !cfg->freqs || cfg->n_channels == 0 || cfg->oversample == 0 || cfg->sample_fmt > 1
			|| cfg->sample_rate != (uint32_t)VDL2_SYMBOL_RATE * VDL2_SPS * cfg->oversample) why = "bad vdl2gpu_config (sample_rate must be 105000*oversample)";
	else if(!rx || n_rx == 0) why = "no receivers";
	else if(n_rx > 65535u) why = "more than 65535 receivers (one K0 grid row each)";
	else if(cfg->n_streams != 0 && cfg->n_streams != n_rx) why = "n_streams must be 0 or the number of receivers";
	else if(cfg->oversample != 20 && cfg->oversample != 10 && cfg->oversample != 13) why = "receivers need oversample 20, 10 or 13 (the rates the receiver-group K1 is built for)";
	else if(cfg->flags & VDL2GPU_FLAG_K1_SCALAR) why = "VDL2GPU_FLAG_K1_SCALAR is not available with receivers";
	else if(cfg->flags & VDL2GPU_FLAG_RAGGED) {
		if(out) *out = nullptr;
		return refuse_ragged("vdl2gpu_create_receivers");
	} else {
		for(uint32_t r = 0; r < n_rx && !why; r++) {
			if(rx[r].n_channels == 0) why = "a receiver has no channels";
			sum += rx[r].n_channels;
		}
		if(!why && sum != cfg->n_channels) why = "the receivers' channel counts do not add up to n_channels";
	}
	if(why) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_create_receivers: %s", why);
		if(out) *out = nullptr;
		return VDL2GPU_EINVAL;
	}
	vdl2gpu_ctx *c = new vdl2gpu_ctx();
	int rc = create_impl(cfg, c, rx, n_rx);
	if(rc != VDL2GPU_OK) { free_ctx(c); *out = nullptr; return rc; }
	*out = c;
	return VDL2GPU_OK;
}

/* the checks of a mixed receiver list shared by vdl2gpu_create_mixed_receivers and vdl2gpu_update_receivers: the list's
 * length, then every receiver (the reason goes to buf; *sum = the channels of the list) */
static const char *mixed_count_error(const vdl2gpu_receiver_ex *rx, uint32_t n_rx) {
	if(!rx || n_rx == 0) return "no receivers";
	if(n_rx > 65535u) return "more than 65535 receivers (one K0 grid row each)";
	return nullptr;
}

static const char *mixed_list_error(const vdl2gpu_receiver_ex *rx, uint32_t n_rx, char *buf, size_t cap, uint64_t *sum) {
	*sum = 0;
	for(uint32_t r = 0; r < n_rx; r++) {
		if(rx[r].n_channels == 0) { snprintf(buf, cap, "receiver %u has no channels", r); return buf; }
		if(rx[r].oversample != 10 && rx[r].oversample != 13 && rx[r].oversample != 20) {
			snprintf(buf, cap, "receiver %u: oversample %u (10, 13 or 20 only)", r, rx[r].oversample); return buf;
		}
		if(rx[r].sample_fmt > 1) {
			snprintf(buf, cap, "receiver %u: sample format %u (VDL2GPU_FMT_U8 or VDL2GPU_FMT_S16_LE only)", r, rx[r].sample_fmt); return buf;
		}
		*sum += rx[r].n_channels;
	}
	return nullptr;
}

extern "C" int vdl2gpu_create_mixed_receivers(const vdl2gpu_config *cfg, const vdl2gpu_receiver_ex *rx, uint32_t n_rx, vdl2gpu_ctx **out) {
	const char *why = nullptr;
	char buf[160];
	uint64_t sum = 0;
	if(!cfg || !out || !cfg->freqs || cfg->n_channels == 0) why = "bad vdl2gpu_config (no channels)";
	else if(cfg->sample_rate || cfg->oversample || cfg->sample_fmt || cfg->centerfreq)
		why = "cfg->sample_rate, oversample, sample_fmt and centerfreq must be 0 (they are per receiver)";
	else if((why = mixed_count_error(rx, n_rx))) {}
	else if(cfg->n_streams != 0 && cfg->n_streams != n_rx) why = "n_streams must be 0 or the number of receivers";
	else if(cfg->flags & VDL2GPU_FLAG_K1_SCALAR) why = "VDL2GPU_FLAG_K1_SCALAR is not available with receivers";
	else {
		why = mixed_list_error(rx, n_rx, buf, sizeof(buf), &sum);
		if(!why && sum != cfg->n_channels) why = "the receivers' channel counts do not add up to n_channels";
	}
	if(why) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_create_mixed_receivers: %s", why);
		if(out) *out = nullptr;
		return VDL2GPU_EINVAL;
	}
	std::vector<vdl2gpu_receiver> base(n_rx);
	for(uint32_t r = 0; r < n_rx; r++) { base[r].centerfreq = rx[r].centerfreq; base[r].n_channels = rx[r].n_channels; }
	vdl2gpu_ctx *c = new vdl2gpu_ctx();
	int rc = create_impl(cfg, c, base.data(), n_rx, rx);
	if(rc != VDL2GPU_OK) { free_ctx(c); *out = nullptr; return rc; }
	*out = c;
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_destroy(vdl2gpu_ctx *ctx) { return free_ctx(ctx); }

/* ------------------------------------------------------------------------------------------------
 * harvesting: burst records (mapped pinned memory) -> frames
 * ---------------------------------------------------------------------------------------------- */
static uint32_t synd_weight_of(uint32_t syn) {       /* src/decode.c:98-100 */
	static const uint8_t w[32] = { 0, 1, 1, 2, 1, 2, 1, 1, 1, 1, 1, 1, 1, 2, 1, 1, 1, 1, 2, 1, 2, 1, 1, 2, 1, 1, 1, 1, 1, 1, 1, 1 };
	return w[syn & 31u];
}

/* burst records (region = vdl2_out_header + records) -> frames.  Offsets in the pending frames are relative to the
 * first record.  `dec_end` / `arrival` place the burst in time (see burst_timestamp below); with ragged spans `span` (the
 * span's receiver table) and `ch_rx` (channel -> receiver) give each channel its own receiver's end position instead. */
typedef std::function<bool(uint32_t channel, uint64_t sync, double &ts)> stamp_fn;

static void parse_region(const uint8_t *region, uint32_t out_cap, double rate, struct timeval arrival, uint64_t dec_end,
		uint32_t blob_id, std::vector<pending_frame> &pending, vdl2gpu_stats &stats, const vdl2_rx_span *span = nullptr,
		const uint32_t *ch_rx = nullptr, const stamp_fn *stamp = nullptr) {
	vdl2_out_header h;
	memcpy(&h, region, sizeof(h));
	const uint8_t *base = region + sizeof(vdl2_out_header);
	const uint32_t used = std::min(h.bytes_used, out_cap);
	stats.out_bytes += h.bytes_used;            /* out_bytes: record bytes written by K3 (D2H traffic) */
	std::vector<const vdl2_burst_record *> recs;
	recs.reserve(h.n_records);
	uint32_t off = 0;
	for(uint32_t k = 0; k < h.n_records && off + sizeof(vdl2_burst_record) <= used; k++) {
		const vdl2_burst_record *r = reinterpret_cast<const vdl2_burst_record *>(base + off);
		if(r->rec_bytes < sizeof(vdl2_burst_record) || off + r->rec_bytes > used) break;
		recs.push_back(r);
		off += r->rec_bytes;
	}
	std::sort(recs.begin(), recs.end(), [](const vdl2_burst_record *a, const vdl2_burst_record *b) {
		return a->channel != b->channel ? a->channel < b->channel : a->burst_seq < b->burst_seq;
	});
	stats.pool_overflows = h.pool_overflows;
	stats.out_overflows = h.out_overflows;
	for(const vdl2_burst_record *r : recs) {
		stats.bursts++;
		if(r->status != VDL2_BURST_OK) stats.burst_errors++;
		for(uint32_t q = 0; q < r->num_blocks && q < VDL2_MAX_BLOCKS; q++)
			if(r->rs_ret[q] != -128) { stats.blocks_processed++; if(r->rs_ret[q] >= 0) stats.blocks_fec_ok++; }
		const uint32_t *tab = reinterpret_cast<const uint32_t *>(reinterpret_cast<const uint8_t *>(r) + sizeof(vdl2_burst_record));
		const uint8_t *bytes = reinterpret_cast<const uint8_t *>(tab + r->n_frames);
		uint32_t foff = 0;
		const uint64_t sync_idx = (uint64_t)r->sync_lo | ((uint64_t)r->sync_hi << 32);
		uint64_t end = dec_end;
		if(span) { const vdl2_rx_span &e = span[ch_rx[r->channel]]; end = e.dec_base + e.n; }
		for(uint32_t k = 0; k < r->n_frames; k++) {
			const uint32_t len = tab[k] & 0xFFFFu, crc = tab[k] >> 16;
			pending_frame pf;
			memset(&pf.f, 0, sizeof(pf.f));
			pf.blob = blob_id;
			pf.offset = (uint32_t)((bytes + foff) - base);
			foff += len;
			pf.f.channel = r->channel; pf.f.freq = r->freq; pf.f.burst_seq = r->burst_seq; pf.f.idx = (int32_t)k;
			pf.f.len = len;
			pf.f.synd_weight = synd_weight_of(r->syndrome);
			pf.f.datalen_octets = r->datalen_bits / 8 + ((r->datalen_bits % 8) != 0);
			pf.f.num_fec_corrections = r->num_fec_corrections;
			pf.f.frame_pwr = r->frame_pwr; pf.f.mag_nf = r->mag_nf;
			pf.f.frame_pwr_dbfs = 10.0f * log10f(r->frame_pwr);                  /* src/decode.c:180 */
			pf.f.nf_pwr_dbfs = nf_pwr_dbfs(r->mag_nf);
			pf.f.ppm_error = r->ppm_error;
			pf.f.sync_dec_index = sync_idx;
			/* the reference stamps gettimeofday() at sync (src/demod.c:246); here: arrival time of the chunk
			 * being processed when the burst completed, moved back by the distance to the sync sample */
			double back = end > sync_idx ? ((double)end - (double)sync_idx) / rate : 0.0;
			double ts = (double)arrival.tv_sec + 1e-6 * (double)arrival.tv_usec - back;
			/* pushed spans: from the arrival of the push that carried the sync group (push_stamp) */
			if(stamp) (*stamp)(r->channel, sync_idx, ts);
			pf.f.burst_timestamp.tv_sec = (time_t)floor(ts);
			pf.f.burst_timestamp.tv_usec = (suseconds_t)((ts - floor(ts)) * 1e6);
			pf.f.fcs_residue = (uint16_t)crc;
			pf.f.fcs_ok = (len >= 11 && crc == 0xF0B8u) ? 1 : 0;
			stats.msg_good++;
			if(len >= 11) { if(crc == 0xF0B8u) stats.fcs_good++; else stats.fcs_bad++; }
			pending.push_back(pf);
		}
	}
}

/* Timestamp of a burst of a pushed span whose sync lies in decimation group `sync` of channel chan's receiver: the
 * arrival time of the push that carried the group's last input sample, moved back by the input samples that push carried
 * after it.  False when the group was not taken from pushed bytes (the span-end rule of parse_region then stands). */
static bool push_stamp(vdl2gpu_ctx *c, uint32_t chan, uint64_t sync, double &ts) {
	const uint32_t r = c->ch_rx[chan];
	push_rx &q = *c->push[r];
	const vdl2_rx_input &in = c->rx_in[r];
	const uint32_t bpp = in.fmt == VDL2GPU_FMT_S16_LE ? 4u : 2u;
	auto a = std::upper_bound(q.anchors.begin(), q.anchors.end(), sync, [](uint64_t v, const span_anchor &x) { return v < x.dec_base; });
	if(a == q.anchors.begin()) return false;
	--a;
	if(sync >= a->dec_base + a->n) return false;
	const uint64_t end = vdl2_push_sync_end(sync, a->dec_base, a->byte_base, in.oversample * bpp);
	std::lock_guard<std::mutex> lk(q.m);
	auto p = std::lower_bound(q.recs.begin(), q.recs.end(), end, [](const push_rec &x, uint64_t v) { return x.end < v; });
	if(p == q.recs.end()) return false;
	ts = p->t - vdl2_push_back_seconds(end, p->end, bpp, (uint32_t)VDL2_SYMBOL_RATE * VDL2_SPS * in.oversample);
	return true;
}

static void harvest(vdl2gpu_ctx *c, chunk_slot &s) {
	if(s.timed) {
		static const int from[5] = { 0, 1, 3, 7, 4 }, to[5] = { 1, 2, 6, 4, 5 };   /* K0, K1 front stream; K2a middle stream; K2, K3 back stream */
		for(int k = 0; k < 5; k++) {
			float ms = 0.f;
			if(cudaEventElapsedTime(&ms, s.tk[from[k]], s.tk[to[k]]) == cudaSuccess) { c->k_ms[k] += ms; c->k_launches[k]++; }
		}
		if(c->ev_t0 && c->timeline.size() < 8u * 4096u) {
			static const int order[7] = { 0, 2, 3, 6, 7, 4, 5 };   /* front start, K1 end, K2a start, K2a end, K2 start, K2|K3, K3 end */
			c->timeline.push_back((float)s.seq);
			for(int k = 0; k < 7; k++) {
				float ms = -1.f;
				if(cudaEventElapsedTime(&ms, c->ev_t0, s.tk[order[k]]) != cudaSuccess) { cudaGetLastError(); ms = -1.f; }
				c->timeline.push_back(ms);
			}
		}
		s.timed = false;
	}
	/* one copy out of the mapped region (header + the bytes K3 used), so the region can be handed back to the device at once */
	const uint8_t *out = s.h_out;
	const vdl2_out_header *h = reinterpret_cast<const vdl2_out_header *>(out);
	const uint32_t used = std::min(h->bytes_used, c->out_cap);
	c->blobs.emplace_back(out, out + sizeof(vdl2_out_header) + used);
	const uint32_t blob_id = (uint32_t)c->blobs.size() - 1;
	/* decimated samples per second (105000 for every receiver of a mixed context, whose config carries no rate) */
	const double rate = c->mixed ? (double)VDL2_SYMBOL_RATE * VDL2_SPS : (double)c->cfg.sample_rate / (double)c->cfg.oversample;
	stamp_fn stamp;
	if(s.pushed) stamp = [c](uint32_t chan, uint64_t sync, double &ts) { return push_stamp(c, chan, sync, ts); };
	parse_region(c->blobs.back().data(), c->out_cap, rate, s.arrival, s.dec_base + s.n_dec, blob_id, c->pending, c->stats,
			c->ragged ? s.h_span.get() : nullptr, c->ch_rx.data(), s.pushed ? &stamp : nullptr);
	c->stats.chunks_completed++;
	s.busy = false;
}

static int deliver(vdl2gpu_ctx *c, vdl2gpu_frame_cb cb, void *user) {
	int n = (int)c->pending.size();
	/* bursts dropped on the device (burst pool or output region exhausted) are an error the caller must see, once per
	 * increase; the frames that did arrive are still delivered first */
	const uint64_t ov = c->stats.pool_overflows + c->stats.out_overflows;
	if(ov > c->overflows_reported) {
		snprintf(g_last_error, sizeof(g_last_error), "%llu burst(s) dropped on the device: burst pool overflows %llu, output region overflows %llu",
				(unsigned long long)(ov - c->overflows_reported), (unsigned long long)c->stats.pool_overflows, (unsigned long long)c->stats.out_overflows);
		c->overflows_reported = ov;
		n = VDL2GPU_EOVERFLOW;
	}
	if(cb) {
		for(auto &pf : c->pending) {
			pf.f.data = c->blobs[pf.blob].data() + sizeof(vdl2_out_header) + pf.offset;
			cb(&pf.f, user);
		}
	}
	c->pending.clear();
	c->blobs.clear();
	return n;
}

/* ------------------------------------------------------------------------------------------------
 * data path
 * ---------------------------------------------------------------------------------------------- */
static int ensure_raw(vdl2gpu_ctx *c, chunk_slot &s) {
	if(s.h_raw) return VDL2GPU_OK;
	const size_t bytes = (size_t)c->cfg.max_chunk_bytes * c->n_streams;
	if(bytes >= ((size_t)1 << 32)) {          /* the host path stages all streams of a chunk in one pinned buffer */
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_submit: n_streams x max_chunk_bytes must stay below 4 GiB (use vdl2gpu_submit_device)");
		return VDL2GPU_ETOOBIG;
	}
	CU(cudaHostAlloc((void **)s.h_raw.put(), bytes, cudaHostAllocDefault));
	CU(cudaMalloc(s.d_raw.put(), bytes));
	return VDL2GPU_OK;
}

static int acquire_slot(vdl2gpu_ctx *c, chunk_slot **out) {
	chunk_slot &s = c->chunks[c->next_slot];
	if(s.busy) {
		/* back-pressure: the producer blocks until the oldest chunk has drained (cf. the demods_ready
		 * barrier in src/demod.c:342) */
		CU(cudaEventSynchronize(s.done));
		harvest(c, s);
		if(!c->inflight.empty() && c->inflight.front() == c->next_slot) c->inflight.pop_front();
	}
	s.pushed = false;
	*out = &s;
	return VDL2GPU_OK;
}

/* parameter blocks of one chunk (number `seq`).  With `ca` the per-chunk values come from the device copy of the chunk
 * arguments (graph replay); the sizes given here then only size the grids. */
static void fill_params(vdl2gpu_ctx *c, chunk_slot &s, uint64_t seq, uint32_t n_pairs, uint32_t cnt0, uint32_t n_dec, uint32_t prev_n_dec,
		uint64_t dec_base, const vdl2_chunk_args *ca, vdl2_k1_params &p1, vdl2_k2a_params &pa, vdl2_k2_params &p2, vdl2_k3_params &p3) {
	float2 *d_dec = c->d_dec3[seq % 3u];
	const int pb = (int)(seq & 1u);
	p1.samples = c->d_samples; p1.n_pairs = n_pairs; p1.oversample = c->cfg.oversample; p1.cnt0 = cnt0;
	p1.n_ch = c->n_ch; p1.n_chp = c->n_chp; p1.lanes = c->lanes; p1.full_warps = c->full_warps; p1.dec = d_dec; p1.state = c->d_k1;
	p1.lut = reinterpret_cast<const float4 *>(c->d_tab->lut);
	p1.a0 = c->tab.t.A[0]; p1.a1 = c->tab.t.A[1]; p1.a2 = c->tab.t.A[2]; p1.b1 = c->tab.t.B[1]; p1.b2 = c->tab.t.B[2];
	p1.one = 1.0f; p1.neg_one = -1.0f; p1.two = 2.0f;
	p1.trace_blocks = c->d_block_trace; p2.trace_blocks = c->d_block_trace;
	p1.ch_per_stream = c->ch_per_stream; p1.stream_stride = c->lane_streams ? c->n_chp : c->max_pairs; p1.ca = ca;
	p1.slot_rx = c->d_slot_rx; p1.block_rx = c->d_block_rx; p1.rx_tile = c->rx_tile; p1.rx_max = c->rx_max;
	p1.rx_in = c->d_rx_in; p1.slot_cls = c->d_slot_cls; p1.cls_mask = c->cls_mask; p1.rx_os_max = c->rx_os_max;
	memcpy(p1.cls_taps, c->cls_taps, sizeof(p1.cls_taps));
	/* the default walk (variant 5) computes the four magnitudes a block needs from the staged samples: no magnitude plane */
	const bool need_mag = (c->k2_variant & 0xFF) >= 0 && (c->k2_variant & 0xFF) <= 4;
	pa.dec = d_dec; pa.phase = c->d_phase2[pb]; pa.mag = need_mag ? c->d_mag2[pb].get() : nullptr; pa.phase_prev = c->d_phase2[pb ^ 1];
	pa.n_dec = n_dec; pa.prev_n_dec = prev_n_dec; pa.n_ch = c->n_ch; pa.n_chp = c->n_chp; pa.lanes = c->lanes; pa.full_warps = c->full_warps;
	pa.mode = (uint32_t)c->k2a_mode; pa.split = c->k2a_split; pa.ca = ca; pa.chlv = c->d_chlv;
	p2.dec = d_dec; p2.phase = c->d_phase2[pb]; p2.mag = c->d_mag2[pb]; p2.hist_tmp = nullptr; p2.n_dec = n_dec; p2.n_ch = c->n_ch; p2.n_chp = c->n_chp;
	p2.lanes = c->lanes; p2.full_warps = c->full_warps; p2.dec_base = dec_base;
	p2.state = c->d_k2; p2.ring = c->d_ring; p2.tables = c->d_tab; p2.max_ppm = c->cfg.max_ppm; p2.s27 = c->tab.s27;
	p2.pool = c->d_pool; p2.free_list = c->d_free; p2.ready = c->d_ready; p2.ctl = c->d_ctl;
	p2.events = c->d_events; p2.event_cap = c->event_cap; p2.trace = (c->cfg.flags & VDL2GPU_FLAG_TRACE) ? 1u : 0u;
	p2.variant = (uint32_t)c->k2_variant; p2.k2a_mode = (uint32_t)c->k2a_mode; p2.ca = ca;
	p1.rx_span = s.d_span; pa.slot_rx = c->d_slot_rx; pa.rx_span = s.d_span; p2.slot_rx = c->d_slot_rx; p2.rx_span = s.d_span;   /* (NULL unless ragged) */
	/* the restart table only on a span that restarts receivers, which is never captured (NULL in every graph) */
	const vdl2_rx_restart *rs = (s.restart && !ca) ? s.d_restart.get() : nullptr;
	p1.rx_restart = rs; pa.rx_restart = rs; p2.rx_restart = rs;
	p3.pool = c->d_pool; p3.free_list = c->d_free; p3.ready = c->d_ready; p3.ctl = c->d_ctl; p3.tables = c->d_tab;
	p3.out = s.d_out; p3.out_cap = c->out_cap; p3.n_chp = c->n_chp; p3.counters = c->d_counters; p3.abandoned = rs ? 1u : 0u;
}

#define K3_GRID (132u * 16u)      /* 16 resident blocks on each of the 132 SMs of an H100: ~1.7 bursts per block per chunk at the bench traffic */

/* One CUDA graph per stage, captured once per (slot, chunk number mod 6 = dec buffer and plane) for the chunk shape
 * (n_pairs) and replayed: a chunk then costs three graph launches and a handful of event calls instead of seven kernel
 * launches.  Everything that differs between two chunks of the same shape (input pointer, decimation phase, sample
 * counts, absolute sample index) travels in the chunk-argument block the front graph copies to the device first. */
template<typename F>
static int capture_one(cudaStream_t st, graph_exec_h &out, F body) {
	cudaGraph_t g = nullptr;
	CU(cudaStreamBeginCapture(st, cudaStreamCaptureModeRelaxed));
	int rc = body();
	cudaError_t e = cudaStreamEndCapture(st, &g);
	if(rc != 0 || e != cudaSuccess) { if(g) cudaGraphDestroy(g); cudaGetLastError(); return rc ? rc : fail_cuda(e, "cudaStreamEndCapture", __LINE__); }
	e = cudaGraphInstantiate(out.put(), g, 0);
	cudaGraphDestroy(g);
	if(e != cudaSuccess) return fail_cuda(e, "cudaGraphInstantiate", __LINE__);
	return VDL2GPU_OK;
}

/* input samples per decimated sample as the chain counts them: a mixed-rate context counts decimated samples directly */
static inline uint32_t chain_os(const vdl2gpu_ctx *c) { return c->mixed ? 1u : c->cfg.oversample; }

/* K0 of a chunk into the sample plane: one row per receiver (mixed-rate receivers; ragged spans, whose table gives the
 * counts, and pushed spans, which read the receivers' rings), one column per stream (one stream per channel) or one row
 * per stream.  n_pairs: samples per stream, or the span's decimated samples (its width when ragged).  ca: graph capture. */
static int launch_k0(vdl2gpu_ctx *c, const chunk_slot &s, const void *raw, uint32_t n_pairs, uint32_t fmt, const vdl2_chunk_args *ca) {
	float *out = reinterpret_cast<float *>(c->d_samples.get());
	const uint32_t bpp = c->cfg.sample_fmt == VDL2GPU_FMT_S16_LE ? 4u : 2u;
	if(c->mixed) {
		const vdl2_k0_rows rows = { s.pushed ? c->d_rings : raw, c->d_rx_in, s.d_span, s.pushed ? c->d_ring_tab.get() : nullptr };
		KL(vdl2_launch_k0_rows(&rows, n_pairs, c->n_streams, c->rx_os_max, c->d_tab->levels, out, c->max_pairs, ca, c->d_levels, c->stream));
	} else if(c->lane_streams) KL(vdl2_launch_k0_lanes(raw, n_pairs, fmt, c->d_tab->levels, out, c->n_streams, n_pairs * bpp, c->n_chp,
			c->lanes, c->full_warps, ca, c->d_levels, c->stream));
	else KL(vdl2_launch_k0(raw, n_pairs, fmt, c->d_tab->levels, out, c->n_streams, n_pairs * bpp, c->max_pairs, ca, c->d_levels, c->stream));
	return VDL2GPU_OK;
}

/* Spectrum of the chunk just converted: it reads the sample plane after K0 and before the next chunk's K0 rewrites it, in
 * the front stream's own order, behind K1.  There it runs while K2 of the previous chunk still holds its one block per SM,
 * and before K2a, so the lock step of K2 and K1 launched together into an empty machine after K2a is left as it was. */
static int launch_spectrum(vdl2gpu_ctx *c, chunk_slot &s, uint32_t n_pairs) {
	CU(cudaMemcpyAsync(s.d_spec, s.h_spec, c->n_streams * sizeof(vdl2_spec_span), cudaMemcpyHostToDevice, c->stream));
	KL(vdl2_launch_spectrum(reinterpret_cast<const float *>(c->d_samples.get()), c->mixed ? n_pairs * c->rx_os_max : n_pairs, c->n_streams,
			c->lane_streams ? c->n_chp : c->max_pairs, c->lane_streams ? c->lanes : 0u, c->full_warps, s.d_spec, c->d_spec_tab, c->d_spec,
			c->stream));
	return VDL2GPU_OK;
}

/* every input's entry of the chunk's segment grid (the samples K0 puts in its row or column), its position advanced */
static void fill_spectrum(vdl2gpu_ctx *c, chunk_slot &s, uint32_t n_pairs) {
	for(uint32_t i = 0; i < c->n_streams; i++) {
		const uint32_t n = c->ragged ? s.h_span[i].n * c->rx_in[i].oversample : c->mixed ? n_pairs * c->rx_in[i].oversample : n_pairs;
		s.h_spec[i] = vdl2_spec_step(c->spec_pos[i], n);
	}
}

/* Front stage of a chunk on the front stream: K0, K1 and the spectrum.  ca: captured into the front graph (the chunk's
 * values then come from the device copy of its arguments), NULL on the direct path. */
static int launch_front(vdl2gpu_ctx *c, chunk_slot &s, const void *raw, uint32_t n_pairs, uint32_t k0_fmt, const vdl2_k1_params &p1,
		const vdl2_chunk_args *ca) {
	/* only a replay needs the chunk's arguments on the device */
	if(ca) CU(cudaMemcpyAsync(s.d_args, s.h_args, sizeof(vdl2_chunk_args), cudaMemcpyHostToDevice, c->stream));
	if(c->ragged) CU(cudaMemcpyAsync(s.d_span, s.h_span, c->n_streams * sizeof(vdl2_rx_span), cudaMemcpyHostToDevice, c->stream));
	/* restart spans and pushed spans are never captured */
	if(!ca && s.restart) CU(cudaMemcpyAsync(s.d_restart, s.h_restart, c->n_chp * sizeof(vdl2_rx_restart), cudaMemcpyHostToDevice, c->stream));
	int rc = launch_k0(c, s, raw, n_pairs, k0_fmt, ca);
	if(rc) return rc;
	if(!ca && s.pushed) CU(cudaEventRecord(s.k0_done, c->stream));     /* the rings' bytes of this span are read */
	/* the direct path times K0 and K1 apart; a replayed front graph is timed as a whole (run_chain) */
	const bool timed = !ca && s.timed;
	if(timed) CU(cudaEventRecord(s.tk[1], c->stream));
	KL(vdl2_launch_k1(&p1, (c->cfg.flags & VDL2GPU_FLAG_K1_SCALAR) ? 1 : 0, c->k1_variant, c->stream));
	if(timed) CU(cudaEventRecord(s.tk[2], c->stream));
	if(c->d_spec) {
		if(!ca) {       /* a restart span (never captured) zeroes its restarting receivers' figures first */
			for(uint32_t r : c->spec_zero) CU(cudaMemsetAsync(c->d_spec + r, 0, sizeof(vdl2_spec_acc), c->stream));
			c->spec_zero.clear();
		}
		rc = launch_spectrum(c, s, n_pairs);
		if(rc) return rc;
	}
	return VDL2GPU_OK;
}

/* Back stage of a chunk on the back stream: K2, K3.  tk_k2 (or NULL) is recorded between them: the direct path times them
 * apart, a replayed back graph as a whole. */
static int launch_back(vdl2gpu_ctx *c, const vdl2_k2_params &p2, const vdl2_k3_params &p3, cudaEvent_t tk_k2) {
	KL(vdl2_launch_k2(&p2, c->s_back));
	if(tk_k2) CU(cudaEventRecord(tk_k2, c->s_back));
	KL(vdl2_launch_k3(&p3, K3_GRID, c->s_back));
	return VDL2GPU_OK;
}

static int ensure_graphs(vdl2gpu_ctx *c, chunk_slot &s, uint64_t seq, uint32_t n_pairs, uint32_t k0_fmt) {
	const int k = (int)(seq % 6u);
	if(s.g_front[k] && s.graph_pairs[k] == n_pairs) return VDL2GPU_OK;
	s.g_front[k].reset(); s.g_k2a[k].reset(); s.g_back[k].reset();
	vdl2_k1_params p1; vdl2_k2a_params pa; vdl2_k2_params p2; vdl2_k3_params p3;
	const uint32_t os = chain_os(c);
	fill_params(c, s, seq, n_pairs, 0, (os - 1 + n_pairs) / os, 0, 0, s.d_args, p1, pa, p2, p3);
	int rc = capture_one(c->stream, s.g_front[k], [&] { return launch_front(c, s, nullptr, n_pairs, k0_fmt, p1, s.d_args); });
	if(rc == 0) rc = capture_one(c->s_mid, s.g_k2a[k], [&] { KL(vdl2_launch_k2a_warps(&pa, c->s_mid)); return 0; });
	if(rc == 0) rc = capture_one(c->s_back, s.g_back[k], [&] { return launch_back(c, p2, p3, nullptr); });
	if(rc == 0) s.graph_pairs[k] = n_pairs;
	return rc;
}

/* n_pairs: complex samples per stream; in a mixed-rate context, decimated samples per receiver (the span's n_dec) */
static int run_chain(vdl2gpu_ctx *c, chunk_slot &s, const void *d_raw, uint32_t n_pairs, uint32_t k0_fmt = 0xFFFFFFFFu) {
	const uint32_t os = chain_os(c);
	const bool planar = k0_fmt != 0xFFFFFFFFu;
	if(!planar) k0_fmt = c->cfg.sample_fmt;
	s.first_pair = c->total_pairs;
	s.n_pairs = n_pairs;
	s.dec_base = c->total_dec;
	s.n_dec = (c->decim_cnt + n_pairs) / os;
	gettimeofday(&s.arrival, NULL);
	s.timed = c->timing;
	const uint64_t seq = c->chunk_seq;
	const int db = (int)(seq % 3u), pb = (int)(seq & 1u), gk = (int)(seq % 6u);
	const bool overlap = c->s_back != c->stream;
	s.seq = seq;
	bool graph = c->use_graphs && !planar && overlap && !s.pushed;     /* pushed spans take the direct path */
	if(graph && c->graph_nominal == 0) c->graph_nominal = n_pairs;
	graph = graph && n_pairs == c->graph_nominal;            /* odd-sized chunks (the tail of a file) take the direct path */
	graph = graph && !s.restart;                             /* ... and so do spans that restart receivers */
	if(graph && ensure_graphs(c, s, seq, n_pairs, k0_fmt) != VDL2GPU_OK) { c->use_graphs = false; graph = false; }
	vdl2_k1_params p1; vdl2_k2a_params pa; vdl2_k2_params p2; vdl2_k3_params p3;
	fill_params(c, s, seq, n_pairs, c->decim_cnt, s.n_dec, c->last_n_dec, s.dec_base, nullptr, p1, pa, p2, p3);
	if(c->d_spec) fill_spectrum(c, s, n_pairs);
	if(graph) {
		s.h_args->raw = d_raw; s.h_args->dec_base = s.dec_base; s.h_args->n_pairs = n_pairs; s.h_args->cnt0 = c->decim_cnt;
		s.h_args->n_dec = s.n_dec; s.h_args->prev_n_dec = c->last_n_dec;
	}
	/* ---- front stage: K0, K1 -> dec[db] (free once K2 of chunk c-3 is done) ---- */
	if(seq >= 3) CU(cudaStreamWaitEvent(c->stream, c->ev_back_done[db], 0));
	/* Two-stage schedule (default): K1 of this chunk starts when K2a of the previous chunk has finished.  K2a is a short
	 * full-occupancy pass; when it ends the GPU is empty, and K2 of chunk c-1 and K1 of chunk c are then launched into that
	 * empty machine together, one block per SM each - the only arrangement in which the block scheduler was found to keep
	 * the two long kernels side by side on every SM, launch after launch (see the slot mapping in create_impl). */
	if(c->stages == 2 && seq >= 1 && overlap) CU(cudaStreamWaitEvent(c->stream, c->ev_k2a_done[pb ^ 1], 0));
	if(s.timed) CU(cudaEventRecord(s.tk[0], c->stream));
	if(graph) {
		/* timed as a whole: the spectrum falls inside "K1" */
		if(s.timed) CU(cudaEventRecord(s.tk[1], c->stream));
		CU(cudaGraphLaunch(s.g_front[gk], c->stream));
		if(s.timed) CU(cudaEventRecord(s.tk[2], c->stream));
	} else {
		int rc = launch_front(c, s, d_raw, n_pairs, k0_fmt, p1, nullptr);
		if(rc) return rc;
	}
	CU(cudaEventRecord(c->ev_input_consumed, c->stream));
	CU(cudaEventRecord(c->ev_k1_done[db], c->stream));
	/* ---- middle stage: K2a -> plane[pb] (free once K2 of chunk c-2 is done), history from plane[pb ^ 1] (chunk c-1, same stream) ---- */
	CU(cudaStreamWaitEvent(c->s_mid, c->ev_k1_done[db], 0));
	if(seq >= 2 && overlap) CU(cudaStreamWaitEvent(c->s_mid, c->ev_back_done[(seq - 2) % 3u], 0));
	if(s.timed) CU(cudaEventRecord(s.tk[3], c->s_mid));
	if(graph) CU(cudaGraphLaunch(s.g_k2a[gk], c->s_mid));
	else KL(vdl2_launch_k2a_warps(&pa, c->s_mid));
	if(s.timed) CU(cudaEventRecord(s.tk[6], c->s_mid));
	CU(cudaEventRecord(c->ev_k2a_done[pb], c->s_mid));
	/* ---- back stage: K2, K3 ---- */
	CU(cudaStreamWaitEvent(c->s_back, c->ev_k2a_done[pb], 0));
	if(s.timed) CU(cudaEventRecord(s.tk[7], c->s_back));
	if(graph) {
		CU(cudaGraphLaunch(s.g_back[gk], c->s_back));
		if(s.timed) CU(cudaEventRecord(s.tk[4], c->s_back));
		c->stats.graph_launches += 3;
	} else {
		int rc = launch_back(c, p2, p3, s.timed ? s.tk[4].get() : nullptr);
		if(rc) return rc;
	}
	if(s.timed) CU(cudaEventRecord(s.tk[5], c->s_back));
	CU(cudaEventRecord(c->ev_back_done[db], c->s_back));
	CU(cudaEventRecord(s.done, c->s_back));
	c->chunk_seq++;
	s.busy = true;
	c->inflight.push_back(c->next_slot);
	c->next_slot = (c->next_slot + 1) % (uint32_t)c->chunks.size();
	c->decim_cnt = (c->decim_cnt + n_pairs) % os;
	c->total_pairs += n_pairs;
	c->total_dec += s.n_dec;
	c->last_n_dec = s.n_dec;
	c->stats.chunks_submitted++;
	if(c->ragged) for(uint32_t r = 0; r < c->n_streams; r++) c->stats.iq_samples += (uint64_t)s.h_span[r].n * c->rx_in[r].oversample;
	else c->stats.iq_samples += c->mixed ? (uint64_t)n_pairs * c->span_pairs_per_dec : n_pairs;
	c->stats.dec_samples += s.n_dec;
	c->stats.kernel_launches += (n_pairs ? 2 : 0) + 1 + (s.n_dec ? 1 : 0) + 2;
	return VDL2GPU_OK;
}

/* the byte-length submits have no meaning for receivers of different rates: their buffers differ in length */
static int refuse_mixed(const char *what) {
	snprintf(g_last_error, sizeof(g_last_error), "%s: a mixed-receivers context takes spans of decimated samples (vdl2gpu_submit_span, vdl2gpu_submit_span_device)", what);
	return VDL2GPU_EINVAL;
}

extern "C" int vdl2gpu_submit(vdl2gpu_ctx *c, const void *iq, uint32_t len) {
	if(!c || (!iq && len)) return VDL2GPU_EINVAL;
	if(c->mixed) return refuse_mixed("vdl2gpu_submit");
	if(len == 0) return VDL2GPU_OK;                                   /* src/demod.c:341,358 */
	if(len > c->cfg.max_chunk_bytes) return VDL2GPU_ETOOBIG;
	const uint32_t bpp = c->cfg.sample_fmt == VDL2GPU_FMT_S16_LE ? 4u : 2u;
	const uint32_t n_pairs = len / bpp;
	if(n_pairs == 0) return VDL2GPU_OK;
	CU(cudaSetDevice(c->device));
	chunk_slot *s;
	int rc = acquire_slot(c, &s);
	if(rc) return rc;
	rc = ensure_raw(c, *s);
	if(rc) return rc;
	/* n_streams buffers of `len` bytes back to back; a ragged tail (len not a multiple of the sample size) is dropped
	 * per stream, so the streams are repacked at n_pairs * bpp */
	const size_t used = (size_t)n_pairs * bpp;
	for(uint32_t st = 0; st < c->n_streams; st++)
		memcpy(s->h_raw + st * used, static_cast<const uint8_t *>(iq) + (size_t)st * len, used);
	CU(cudaMemcpyAsync(s->d_raw, s->h_raw, used * c->n_streams, cudaMemcpyHostToDevice, c->stream));
	return run_chain(c, *s, s->d_raw, n_pairs);
}

extern "C" int vdl2gpu_submit_planar_s16(vdl2gpu_ctx *c, const int16_t *xi, const int16_t *xq, uint32_t n_pairs) {
	if(!c || ((!xi || !xq) && n_pairs)) return VDL2GPU_EINVAL;
	if(c->mixed) return refuse_mixed("vdl2gpu_submit_planar_s16");
	if(c->cfg.sample_fmt != VDL2GPU_FMT_S16_LE || c->n_streams != 1 || c->receivers) return VDL2GPU_EINVAL;
	if(n_pairs == 0) return VDL2GPU_OK;
	if((uint64_t)n_pairs * 4u > c->cfg.max_chunk_bytes) return VDL2GPU_ETOOBIG;
	CU(cudaSetDevice(c->device));
	chunk_slot *s;
	int rc = acquire_slot(c, &s);
	if(rc) return rc;
	rc = ensure_raw(c, *s);
	if(rc) return rc;
	memcpy(s->h_raw, xi, (size_t)n_pairs * 2);
	memcpy(s->h_raw + (size_t)n_pairs * 2, xq, (size_t)n_pairs * 2);
	CU(cudaMemcpyAsync(s->d_raw, s->h_raw, (size_t)n_pairs * 4, cudaMemcpyHostToDevice, c->stream));
	return run_chain(c, *s, s->d_raw, n_pairs, 2u);
}

/* src/fmtr-binary.c + src/output-file.c:181-189: one raw frame in the reference's archive format, i.e. a 2-octet
 * big-endian length (its own two octets included) followed by the proto3 message dumpvdl2.raw_avlc_frame
 * (proto/dumpvdl2.proto:25-48).  Files made of these records replay through an unmodified
 * `dumpvdl2 --raw-frames-file` (src/input-raw_frames_file.c:33-75).  Returns the record size or a negative error. */
static size_t pb_varint(uint8_t *o, uint64_t v) { size_t n = 0; do { uint8_t b = v & 0x7Fu; v >>= 7; o[n++] = (uint8_t)(b | (v ? 0x80u : 0u)); } while(v); return n; }
static size_t pb_u32_field(uint8_t *o, int field, uint32_t v) { if(!v) return 0; size_t n = pb_varint(o, (uint64_t)field << 3); return n + pb_varint(o + n, v); }
static size_t pb_i64_field(uint8_t *o, int field, int64_t v) { if(!v) return 0; size_t n = pb_varint(o, (uint64_t)field << 3); return n + pb_varint(o + n, (uint64_t)v); }
static size_t pb_f32_field(uint8_t *o, int field, float v) { uint32_t u; memcpy(&u, &v, 4); if(!u) return 0; size_t n = pb_varint(o, ((uint64_t)field << 3) | 5u); memcpy(o + n, &u, 4); return n + 4; }

extern "C" int vdl2gpu_serialize_raw_frame(const vdl2gpu_frame *f, const char *station_id, uint8_t *out, size_t cap) {
	if(!f || !out || (f->len && !f->data)) return VDL2GPU_EINVAL;
	uint8_t ts[24], md[96 + 256];
	size_t nts = 0, nmd = 0;
	nts += pb_i64_field(ts + nts, 1, (int64_t)f->burst_timestamp.tv_sec);
	nts += pb_i64_field(ts + nts, 2, (int64_t)f->burst_timestamp.tv_usec);
	size_t sl = station_id ? strlen(station_id) : 0;
	if(sl > 255) sl = 255;                                          /* STATION_ID_LEN_MAX, src/dumpvdl2.h:193 */
	if(sl) { nmd += pb_varint(md + nmd, (1u << 3) | 2u); nmd += pb_varint(md + nmd, sl); memcpy(md + nmd, station_id, sl); nmd += sl; }
	nmd += pb_u32_field(md + nmd, 2, f->freq);
	nmd += pb_u32_field(md + nmd, 3, f->synd_weight);
	nmd += pb_u32_field(md + nmd, 4, f->datalen_octets);
	nmd += pb_f32_field(md + nmd, 5, f->frame_pwr_dbfs);
	nmd += pb_f32_field(md + nmd, 6, f->nf_pwr_dbfs);
	nmd += pb_f32_field(md + nmd, 7, f->ppm_error);
	nmd += pb_i64_field(md + nmd, 8, 1);                            /* metadata version, src/decode.c:177 */
	nmd += pb_i64_field(md + nmd, 9, (int64_t)f->num_fec_corrections);
	nmd += pb_i64_field(md + nmd, 10, (int64_t)f->idx);
	nmd += pb_varint(md + nmd, (11u << 3) | 2u); nmd += pb_varint(md + nmd, nts); memcpy(md + nmd, ts, nts); nmd += nts;
	uint8_t hdr[16];
	size_t nh = pb_varint(hdr, (1u << 3) | 2u); nh += pb_varint(hdr + nh, nmd);
	uint8_t dh[16];
	size_t nd = f->len ? pb_varint(dh, (2u << 3) | 2u) : 0;
	if(f->len) nd += pb_varint(dh + nd, f->len);
	const size_t total = 2 + nh + nmd + nd + f->len;
	if(total > 65535 || total > cap) return VDL2GPU_ETOOBIG;         /* OUT_BINARY_FRAME_LEN_MAX, src/output-file.h:26 */
	uint8_t *o = out;
	*o++ = (uint8_t)(total >> 8); *o++ = (uint8_t)total;
	memcpy(o, hdr, nh); o += nh; memcpy(o, md, nmd); o += nmd;
	memcpy(o, dh, nd); o += nd; if(f->len) memcpy(o, f->data, f->len);
	return (int)total;
}

extern "C" int vdl2gpu_submit_device(vdl2gpu_ctx *c, const void *dev_iq, uint32_t len, void *producer_stream) {
	if(!c || (!dev_iq && len)) return VDL2GPU_EINVAL;
	if(c->mixed) return refuse_mixed("vdl2gpu_submit_device");
	if(len == 0) return VDL2GPU_OK;
	if(len > c->cfg.max_chunk_bytes) return VDL2GPU_ETOOBIG;
	const uint32_t bpp = c->cfg.sample_fmt == VDL2GPU_FMT_S16_LE ? 4u : 2u;
	const uint32_t n_pairs = len / bpp;
	if(n_pairs == 0) return VDL2GPU_OK;
	if(c->n_streams > 1 && len % bpp != 0) return VDL2GPU_EINVAL;     /* streams are `len` bytes apart in dev_iq */
	CU(cudaSetDevice(c->device));
	chunk_slot *s;
	int rc = acquire_slot(c, &s);
	if(rc) return rc;
	CU(cudaEventRecord(c->ev_input_ready, (cudaStream_t)producer_stream));
	CU(cudaStreamWaitEvent(c->stream, c->ev_input_ready, 0));
	return run_chain(c, *s, dev_iq, n_pairs);
}

/* spans: the common checks of the two submits.  Returns 1 for a mixed-rate context (go on), 0 after forwarding a uniform
 * receivers context's span as `*len` bytes per receiver (the caller submits it), or a negative error. */
static int span_check(vdl2gpu_ctx *c, const void *iq, uint32_t n_dec, const char *what, uint32_t *len) {
	if(!c || (!iq && n_dec)) return VDL2GPU_EINVAL;
	if(!c->receivers) {
		snprintf(g_last_error, sizeof(g_last_error), "%s: spans need a receivers context (vdl2gpu_create_mixed_receivers or vdl2gpu_create_receivers)", what);
		return VDL2GPU_EINVAL;
	}
	if(c->mixed) {
		if(n_dec > c->max_span) {
			snprintf(g_last_error, sizeof(g_last_error), "%s: %u decimated samples per span, at most %u fit max_chunk_bytes", what, n_dec, c->max_span);
			return VDL2GPU_ETOOBIG;
		}
		return 1;
	}
	const uint64_t bytes = (uint64_t)n_dec * c->cfg.oversample * (c->cfg.sample_fmt == VDL2GPU_FMT_S16_LE ? 4u : 2u);
	if(bytes > c->cfg.max_chunk_bytes) return VDL2GPU_ETOOBIG;
	*len = (uint32_t)bytes;
	return 0;
}

/* the restart table of the span about to run in slot s (its previous chunk has been harvested): every receiver with a
 * restart pending restarts at the start of this span, with its current tuning */
static void fill_restarts(vdl2gpu_ctx *c, chunk_slot &s) {
	s.restart = c->n_restart_pending != 0;
	if(!s.restart) return;
	memset(s.h_restart, 0, (size_t)c->n_chp * sizeof(vdl2_rx_restart));
	for(uint32_t r = 0; r < c->n_streams; r++) {
		if(!c->rx_restart_pending[r]) continue;
		const uint32_t rate = (uint32_t)VDL2_SYMBOL_RATE * VDL2_SPS * c->rx_in[r].oversample;
		for(uint32_t chan = c->rx_first[r]; chan < c->rx_first[r + 1]; chan++) {
			vdl2_rx_restart &e = s.h_restart[slot_of(chan, c->lanes, c->full_warps)];
			e.restart = 1u;
			e.dphi = vdl2_nco_dphi(c->rx_centre[r], c->freqs[chan], rate);
			e.freq = c->freqs[chan];
		}
		if(c->d_spec) { c->spec_pos[r] = 0; c->spec_zero.push_back(r); }    /* a new segment grid from this span on */
		c->rx_restart_pending[r] = 0;
	}
	c->n_restart_pending = 0;
}

/* bytes per decimation group of receiver r of a mixed context */
static inline uint32_t group_bytes(const vdl2gpu_ctx *c, uint32_t r) {
	return c->rx_in[r].oversample * (c->rx_in[r].fmt == VDL2GPU_FMT_S16_LE ? 4u : 2u);
}

/* whether any receiver has pushed bytes not yet in a span (whole_group: at least one whole decimation group of them) */
static bool push_queued(vdl2gpu_ctx *c, bool whole_group) {
	if(!c->push_ready) return false;
	for(uint32_t r = 0; r < c->n_streams; r++) {
		push_rx &q = *c->push[r];
		std::lock_guard<std::mutex> lk(q.m);
		if(q.head - q.tail >= (whole_group ? group_bytes(c, r) : 1u)) return true;
	}
	return false;
}

/* Ragged spans: receiver r brings n_dec[r] decimated samples (host buffer, or device buffer ordered after producer_stream).
 * Everything is checked before the device is touched; the span then runs the chain at its width, the largest count, with
 * the span's receiver table (built in the slot's pinned copy: the slot's previous chunk has been harvested) telling every
 * kernel lane its receiver's count, place in the buffer and position. */
static int ragged_submit(vdl2gpu_ctx *c, const void *iq, const uint32_t *n_dec, bool device, void *producer_stream, const char *what) {
	if(!c || !n_dec) return VDL2GPU_EINVAL;
	if(!c->ragged) {
		snprintf(g_last_error, sizeof(g_last_error), "%s: needs a context made by vdl2gpu_create_mixed_receivers with VDL2GPU_FLAG_RAGGED", what);
		return VDL2GPU_EINVAL;
	}
	uint32_t width = 0;
	for(uint32_t r = 0; r < c->n_streams; r++) {
		if(n_dec[r] > c->max_span) {
			snprintf(g_last_error, sizeof(g_last_error), "%s: receiver %u brings %u decimated samples, at most %u fit max_chunk_bytes", what, r, n_dec[r], c->max_span);
			return VDL2GPU_ETOOBIG;
		}
		width = std::max(width, n_dec[r]);
	}
	if(width == 0) return VDL2GPU_OK;
	if(!iq) return VDL2GPU_EINVAL;
	if(push_queued(c, false)) {          /* those bytes come first in their receivers' streams */
		snprintf(g_last_error, sizeof(g_last_error), "%s: receivers have pushed bytes not yet in a span (vdl2gpu_submit_pushed first)", what);
		return VDL2GPU_EINVAL;
	}
	CU(cudaSetDevice(c->device));
	chunk_slot *s;
	int rc = acquire_slot(c, &s);
	if(rc) return rc;
	if(!device) {
		rc = ensure_raw(c, *s);
		if(rc) return rc;
	}
	/* every buffer is at most max_span x its receiver's bytes per decimated sample <= max_chunk_bytes: the span fits the
	 * max_chunk_bytes x n_rx staging buffer */
	const uint64_t bytes = vdl2_rx_span_table(c->rx_in.data(), c->n_streams, n_dec, c->rx_pos.data(), c->rx_prev.data(), s->h_span);
	fill_restarts(c, *s);
	if(device) {
		CU(cudaEventRecord(c->ev_input_ready, (cudaStream_t)producer_stream));
		CU(cudaStreamWaitEvent(c->stream, c->ev_input_ready, 0));
		return run_chain(c, *s, iq, width);
	}
	memcpy(s->h_raw, iq, bytes);
	CU(cudaMemcpyAsync(s->d_raw, s->h_raw, bytes, cudaMemcpyHostToDevice, c->stream));
	return run_chain(c, *s, s->d_raw, width);
}

extern "C" int vdl2gpu_submit_ragged(vdl2gpu_ctx *c, const void *iq, const uint32_t *n_dec) {
	return ragged_submit(c, iq, n_dec, false, nullptr, "vdl2gpu_submit_ragged");
}

extern "C" int vdl2gpu_submit_ragged_device(vdl2gpu_ctx *c, const void *dev_iq, const uint32_t *n_dec, void *producer_stream) {
	return ragged_submit(c, dev_iq, n_dec, true, producer_stream, "vdl2gpu_submit_ragged_device");
}

/* ------------------------------------------------------------------------------------------------
 * pushed input (vdl2gpu_push, vdl2gpu_submit_pushed; see DESIGN.md, "Pushed input", for the ordering rules)
 * ---------------------------------------------------------------------------------------------- */
/* the rings of layout L's receivers, their pinned host mirror and empty queues, built into the empty P (on failure P holds
 * what it got, and frees it) */
static int alloc_rings(push_rings &P, const ctx_layout &L, uint32_t max_chunk_bytes) {
	const uint32_t n_rx = L.n_streams;
	P.rings.resize(n_rx);
	const uint64_t total = vdl2_push_ring_layout(L.rx_in.data(), n_rx, max_chunk_bytes, L.max_span, P.rings.data());
	CU(cudaMalloc(P.d_rings.put(), total));
	CU(cudaHostAlloc((void **)P.h_rings.put(), total, cudaHostAllocDefault));
	CU(cudaMalloc(P.d_ring_tab.put(), (size_t)n_rx * sizeof(vdl2_rx_ring)));
	CU(cudaMemcpy(P.d_ring_tab, P.rings.data(), (size_t)n_rx * sizeof(vdl2_rx_ring), cudaMemcpyHostToDevice));
	P.push.resize(n_rx);
	for(auto &q : P.push) q.reset(new push_rx());
	return VDL2GPU_OK;
}

/* len bytes at stream position pos of receiver r's ring: into the host mirror, then one copy per piece on stream st */
static int ring_write(const push_rings &P, cudaStream_t st, uint32_t r, uint64_t pos, const uint8_t *src, uint32_t len) {
	const vdl2_rx_ring &rg = P.rings[r];
	const vdl2_ring_segs sg = vdl2_ring_segments(rg.cap, pos, len);
	for(int k = 0; k < 2; k++) {
		if(!sg.len[k]) continue;
		uint8_t *h = P.h_rings + rg.base + sg.off[k];
		memcpy(h, src, sg.len[k]);
		CU(cudaMemcpyAsync(P.d_rings + rg.base + sg.off[k], h, sg.len[k], cudaMemcpyHostToDevice, st));
		src += sg.len[k];
	}
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_push(vdl2gpu_ctx *c, uint32_t r, const void *iq, uint32_t len) {
	struct timeval arrival;
	gettimeofday(&arrival, NULL);
	const char *why = nullptr;
	if(!c) why = "no context";
	else if(!c->ragged) why = "needs a context made by vdl2gpu_create_mixed_receivers with VDL2GPU_FLAG_RAGGED";
	else if(r >= c->n_streams) why = "no such receiver";
	else if(!iq && len) why = "no buffer";
	if(why) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_push: %s", why);
		return VDL2GPU_EINVAL;
	}
	if(len > c->cfg.max_chunk_bytes) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_push: %u bytes, at most max_chunk_bytes = %u", len, c->cfg.max_chunk_bytes);
		return VDL2GPU_ETOOBIG;
	}
	if(len == 0) return VDL2GPU_OK;
	CU(cudaSetDevice(c->device));
	if(!c->push_ready) {
		std::lock_guard<std::mutex> lk(c->push_alloc);
		if(!c->push_ready) {
			if(!c->s_copy) {
				CU(cudaStreamCreateWithFlags(c->s_copy.put(), cudaStreamNonBlocking));
				CU(cudaEventCreateWithFlags(c->ev_copied.put(), cudaEventDisableTiming));
				CU(cudaEventCreateWithFlags(c->ev_dropped.put(), cudaEventDisableTiming));
			}
			push_rings P;
			const int rc = alloc_rings(P, *c, c->cfg.max_chunk_bytes);
			if(rc) return rc;
			static_cast<push_rings &>(*c) = std::move(P);
			c->push_ready = true;
		}
	}
	push_rx &q = *c->push[r];
	const uint64_t cap = c->rings[r].cap;
	std::unique_lock<std::mutex> lk(q.m);
	/* back-pressure: wait until the bytes before `freed` cover enough of the ring.  Fences complete without the caller;
	 * with none left, only vdl2gpu_submit_pushed (taking the queue into spans, which adds fences) makes room. */
	while(vdl2_push_room(cap, q.head, q.freed) < len) {
		while(!q.fences.empty()) {
			const cudaError_t e = cudaEventQuery(q.fences.front().ev);
			if(e == cudaErrorNotReady) break;
			if(e != cudaSuccess) return fail_cuda(e, "cudaEventQuery", __LINE__);
			q.freed = q.fences.front().pos;
			q.fences.pop_front();
		}
		if(vdl2_push_room(cap, q.head, q.freed) >= len) break;
		if(!q.fences.empty()) {
			const cudaEvent_t ev = q.fences.front().ev;
			lk.unlock();
			const cudaError_t e = cudaEventSynchronize(ev);
			lk.lock();
			if(e != cudaSuccess) return fail_cuda(e, "cudaEventSynchronize", __LINE__);
		} else {
			q.room.wait(lk);
		}
	}
	const int rc = ring_write(*c, c->s_copy, r, q.head, static_cast<const uint8_t *>(iq), len);
	if(rc) return rc;
	/* published only now: the copies are issued, so an event submit_pushed records on the copy stream after reading head
	 * covers every byte before it */
	q.head += len;
	q.recs.push_back({ q.head, (double)arrival.tv_sec + 1e-6 * (double)arrival.tv_usec });
	return VDL2GPU_OK;
}

/* vdl2gpu_update_receivers: rings P for the new layout n beside the old ones in c, each kept receiver's queue moved to its
 * new index: its partial group (fewer bytes than a group, read from the host mirror of its old ring, written at the same
 * stream positions of its new ring) and its arrival and span records.  c is left as it was. */
static int carry_pushed(vdl2gpu_ctx *c, const ctx_layout &n, const int32_t *from, push_rings &P) {
	int rc = alloc_rings(P, n, c->cfg.max_chunk_bytes);
	for(uint32_t r = 0; r < n.n_streams && rc == VDL2GPU_OK; r++) {
		if(from[r] < 0) continue;
		push_rx &o = *c->push[from[r]], &q = *P.push[r];
		q.head = o.head; q.tail = q.freed = o.tail;
		q.recs = o.recs; q.anchors = o.anchors;
		std::vector<uint8_t> part;
		const vdl2_rx_ring &rg = c->rings[from[r]];
		const vdl2_ring_segs sg = vdl2_ring_segments(rg.cap, o.tail, o.head - o.tail);
		for(int k = 0; k < 2; k++) part.insert(part.end(), c->h_rings + rg.base + sg.off[k], c->h_rings + rg.base + sg.off[k] + sg.len[k]);
		rc = ring_write(P, c->s_copy, r, q.tail, part.data(), (uint32_t)part.size());
	}
	/* also on failure: P's buffers may go only once their copies are done */
	const cudaError_t e = cudaStreamSynchronize(c->s_copy);
	if(rc == VDL2GPU_OK && e != cudaSuccess) rc = fail_cuda(e, "cudaStreamSynchronize", __LINE__);
	return rc;
}

/* decimated samples before a receiver's position for which span and arrival records are kept: a burst is harvested at
 * most n_inflight + 1 spans after the one it completes in, and its sync lies at most one burst before that */
static uint64_t push_keep_dec(const vdl2gpu_ctx *c) {
	return (uint64_t)(c->cfg.n_inflight + 2u) * c->max_span + (uint64_t)(VDL2_MAX_BURST_BITS / 3u + 64u) * VDL2_SPS;
}

extern "C" int vdl2gpu_submit_pushed(vdl2gpu_ctx *c) {
	if(!c) return VDL2GPU_EINVAL;
	if(!c->ragged) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_submit_pushed: needs a context made by vdl2gpu_create_mixed_receivers with VDL2GPU_FLAG_RAGGED");
		return VDL2GPU_EINVAL;
	}
	if(!c->push_ready) return 0;
	CU(cudaSetDevice(c->device));
	const uint32_t n_rx = c->n_streams;
	std::vector<uint32_t> take(n_rx);
	std::vector<uint64_t> tail(n_rx), start(n_rx), limit(n_rx);
	const uint64_t keep = push_keep_dec(c);
	/* One snapshot of the heads at entry: every byte before them has its copy issued.  The call drains up to them and no
	 * further, so it returns however fast other threads keep pushing; bytes pushed meanwhile wait for the next call. */
	for(uint32_t r = 0; r < n_rx; r++) {
		push_rx &q = *c->push[r];
		std::lock_guard<std::mutex> lk(q.m);
		limit[r] = q.head;
	}
	int spans = 0;
	for(;;) {
		uint32_t width = 0;
		for(uint32_t r = 0; r < n_rx; r++) {
			push_rx &q = *c->push[r];
			std::lock_guard<std::mutex> lk(q.m);
			take[r] = vdl2_push_take(limit[r], q.tail, group_bytes(c, r), c->max_span);
			start[r] = tail[r] = q.tail;
			width = std::max(width, take[r]);
		}
		if(width == 0) break;
		chunk_slot *s;
		int rc = acquire_slot(c, &s);
		if(rc) return rc;
		/* ... and the front stream waits for those copies */
		CU(cudaEventRecord(c->ev_copied, c->s_copy));
		CU(cudaStreamWaitEvent(c->stream, c->ev_copied, 0));
		vdl2_push_span_table(c->rx_in.data(), c->rings.data(), n_rx, take.data(), tail.data(), c->rx_pos.data(), c->rx_prev.data(), s->h_span);
		fill_restarts(c, *s);
		s->pushed = true;
		rc = run_chain(c, *s, nullptr, width);
		if(rc) return rc;
		for(uint32_t r = 0; r < n_rx; r++) {
			if(!take[r]) continue;
			push_rx &q = *c->push[r];
			q.anchors.push_back({ s->h_span[r].dec_base, start[r], take[r] });
			const uint64_t pos = c->rx_pos[r];
			while(!q.anchors.empty() && q.anchors.front().dec_base + q.anchors.front().n + keep < pos) q.anchors.pop_front();
			std::lock_guard<std::mutex> lk(q.m);
			q.tail = tail[r];
			q.fences.push_back({ s->k0_done, tail[r] });
			while(!q.recs.empty() && q.recs.front().end <= q.anchors.front().byte_base) q.recs.pop_front();
			q.room.notify_all();
		}
		spans++;
	}
	return spans;
}

/* Restart receiver r at the start of the next span that runs (see include/vdl2gpu.h).  Only the host's record of the
 * receiver's tuning changes here; the kernels of that span apply the restart, each at its own stage of the pipeline. */
extern "C" int vdl2gpu_restart_receiver(vdl2gpu_ctx *c, uint32_t r, uint32_t centerfreq, const uint32_t *freqs) {
	if(!c) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_restart_receiver: no context");
		return VDL2GPU_EINVAL;
	}
	if(!c->ragged) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_restart_receiver: needs a context made by vdl2gpu_create_mixed_receivers with VDL2GPU_FLAG_RAGGED");
		return VDL2GPU_EINVAL;
	}
	if(r >= c->n_streams) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_restart_receiver: receiver %u of %u", r, c->n_streams);
		return VDL2GPU_EINVAL;
	}
	if(c->push_ready) {
		/* the old process is killed now: its pushed bytes not yet in a span go with it, a split sample included; the
		 * receiver's next push starts on a sample boundary.  The dropped bytes' ring places come back once their copies
		 * are done. */
		push_rx &q = *c->push[r];
		std::lock_guard<std::mutex> lk(q.m);
		if(q.head != q.tail) {
			CU(cudaSetDevice(c->device));
			CU(cudaEventRecord(c->ev_dropped, c->s_copy));
			q.head = q.tail = vdl2_push_realign(q.head, c->rx_in[r].fmt == VDL2GPU_FMT_S16_LE ? 4u : 2u);
			q.fences.push_back({ c->ev_dropped, q.head });
		}
		q.room.notify_all();
	}
	if(centerfreq) c->rx_centre[r] = centerfreq;
	if(freqs) std::copy(freqs, freqs + (c->rx_first[r + 1] - c->rx_first[r]), c->freqs.begin() + c->rx_first[r]);
	if(!c->rx_restart_pending[r]) { c->rx_restart_pending[r] = 1; c->n_restart_pending++; }
	return VDL2GPU_OK;
}

/* vdl2gpu_update_receivers once everything is checked: the new layout n (setup_layout) is filled from the old one in c.
 * Only n's buffers are written; c's are read. */
static int migrate_receivers(vdl2gpu_ctx *c, ctx_layout &n, const vdl2gpu_receiver_ex *rx, const int32_t *from) {
	const uint32_t n_rx = n.n_streams;
	CU(cudaStreamSynchronize(c->stream));
	CU(cudaStreamSynchronize(c->s_back));
	vdl2_queue_ctl ctl;
	CU(cudaMemcpy(&ctl, c->d_ctl, sizeof(ctl), cudaMemcpyDeviceToHost));
	if(ctl.n_ready != 0) {           /* K3 empties the ready list of every span it decodes */
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_update_receivers: %u bursts wait in the ready list of a drained context", ctl.n_ready);
		return VDL2GPU_EINVAL;
	}
	std::vector<uint32_t> old_slot_of_burst(c->n_chp);          /* K2_SLOT of every old slot: the pool slot its burst in progress holds */
	CU(cudaMemcpy(old_slot_of_burst.data(), c->d_k2 + (size_t)K2_SLOT * c->n_chp, c->n_chp * 4, cudaMemcpyDeviceToHost));
	std::vector<vdl2_rx_migrate> map(n.n_chp);
	std::vector<uint8_t> held(n.n_slots, 0);
	for(uint32_t i = 0; i < n.n_chp; i++) {
		vdl2_rx_migrate &m = map[i];
		memset(&m, 0, sizeof(m));
		m.slot_from = vdl2_rx_slot_from(i, n.lanes, n.full_warps, n.n_ch, n.rx_first.data(), n_rx, from, c->lanes, c->full_warps,
				c->rx_first.data());
		m.chan_from = i < n.n_ch ? vdl2_rx_chan_from(i, n.rx_first.data(), n_rx, from, c->rx_first.data()) : -1;
		uint32_t chan;
		if(!vdl2_slot_channel(i, n.lanes, n.full_warps, n.n_ch, chan)) continue;
		const uint32_t r = n.ch_rx[chan];
		if(m.slot_from >= 0) {
			m.hist_row = c->rx_prev[from[r]];
			const int32_t b = (int32_t)old_slot_of_burst[m.slot_from];
			if(b >= 0) held[b] = 1;                               /* (b < old n_slots <= n_slots: the index stays valid) */
		} else {
			m.dphi = vdl2_nco_dphi(rx[r].centerfreq, n.freqs[chan], (uint32_t)VDL2_SYMBOL_RATE * VDL2_SPS * rx[r].oversample);
			m.freq = n.freqs[chan];
		}
	}
	/* the free list: every pool slot no kept channel holds (those of removed receivers come back) */
	std::vector<int32_t> fl;
	fl.reserve(n.n_slots);
	for(uint32_t i = 0; i < n.n_slots; i++) if(!held[i]) fl.push_back((int32_t)i);
	ctl.free_top = (int32_t)fl.size();
	dev_mem<vdl2_rx_migrate> d_map;
	CU(cudaMalloc(d_map.put(), map.size() * sizeof(vdl2_rx_migrate)));
	CU(cudaMemcpy(d_map, map.data(), map.size() * sizeof(vdl2_rx_migrate), cudaMemcpyHostToDevice));
	/* the plane the next span takes its history from: the other one of its own (run_chain) */
	const int pb_prev = (int)((c->chunk_seq & 1u) ^ 1u);
	vdl2_migrate_params p;
	p.map = d_map;
	p.n_chp = n.n_chp; p.old_n_chp = c->n_chp;
	p.old_k1 = c->d_k1; p.old_k2 = c->d_k2; p.old_counters = c->d_counters; p.old_ring = c->d_ring; p.old_phase = c->d_phase2[pb_prev];
	p.k1 = n.d_k1; p.k2 = n.d_k2; p.counters = n.d_counters; p.ring = n.d_ring; p.phase = n.d_phase2[pb_prev];
	p.old_chlv = c->d_chlv; p.chlv = n.d_chlv;                  /* (channel levels: both NULL or both allocated) */
	KL(vdl2_launch_migrate(&p, c->stream));
	/* held slots keep their indices (and their words): K2 writes a burst's channel number into its slot only at hand-off */
	CU(cudaMemcpyAsync(n.d_pool, c->d_pool, (size_t)c->n_slots * sizeof(vdl2_burst_slot), cudaMemcpyDeviceToDevice, c->stream));
	CU(cudaMemcpyAsync(n.d_free, fl.data(), fl.size() * 4, cudaMemcpyHostToDevice, c->stream));
	CU(cudaMemcpyAsync(n.d_ctl, &ctl, sizeof(ctl), cudaMemcpyHostToDevice, c->stream));
	/* input levels: a kept receiver carries its accumulator to its new index, a new one starts at zero (setup_layout) */
	std::vector<vdl2_levels> old_lv, new_lv;
	if(c->d_levels) {
		old_lv.resize(c->n_streams);
		new_lv.assign(n_rx, vdl2_levels());
		CU(cudaMemcpyAsync(old_lv.data(), c->d_levels, old_lv.size() * sizeof(vdl2_levels), cudaMemcpyDeviceToHost, c->stream));
		CU(cudaStreamSynchronize(c->stream));
		for(uint32_t r = 0; r < n_rx; r++) if(from[r] >= 0) new_lv[r] = old_lv[from[r]];
		CU(cudaMemcpyAsync(n.d_levels, new_lv.data(), new_lv.size() * sizeof(vdl2_levels), cudaMemcpyHostToDevice, c->stream));
	}
	/* spectrum: likewise, with its waiting samples and its place on its segment grid */
	if(c->d_spec)
		for(uint32_t r = 0; r < n_rx; r++) {
			if(from[r] < 0) continue;
			CU(cudaMemcpyAsync(n.d_spec + r, c->d_spec + from[r], sizeof(vdl2_spec_acc), cudaMemcpyDeviceToDevice, c->stream));
			n.spec_pos[r] = c->spec_pos[from[r]];
		}
	CU(cudaStreamSynchronize(c->stream));
	/* per receiver: a kept one carries its position and a pending restart over; every history now starts at row 0 */
	for(uint32_t r = 0; r < n_rx; r++) {
		if(from[r] < 0) continue;
		n.rx_pos[r] = c->rx_pos[from[r]];
		n.rx_restart_pending[r] = c->rx_restart_pending[from[r]];
		n.n_restart_pending += n.rx_restart_pending[r];
	}
	return VDL2GPU_OK;
}

/* Replace the receiver list of a drained ragged context (see include/vdl2gpu.h).  Everything is checked first; then the
 * new layout is allocated beside the old one, the kept channels' state is moved into it, the context switches to it and
 * the old one is freed.  Any failure before the switch frees the new layout and leaves the context as it was. */
extern "C" int vdl2gpu_update_receivers(vdl2gpu_ctx *c, const vdl2gpu_receiver_ex *rx, const int32_t *from, uint32_t n_rx,
		const uint32_t *freqs) {
	const char *why = nullptr;
	char buf[192];
	uint64_t sum = 0;
	if(!c) why = "no context";
	else if(!c->ragged) why = "needs a context made by vdl2gpu_create_mixed_receivers with VDL2GPU_FLAG_RAGGED";
	else if(vdl2gpu_chunks_in_flight(c) != 0) why = "spans are in flight (vdl2gpu_flush first)";
	else if(push_queued(c, true)) why = "receivers have whole decimation groups pushed and not yet in a span (vdl2gpu_submit_pushed first)";
	else if((why = mixed_count_error(rx, n_rx))) {}
	else if(!from || !freqs) why = "from and freqs must not be NULL";
	else if((why = mixed_list_error(rx, n_rx, buf, sizeof(buf), &sum))) {}
	else {
		std::vector<uint8_t> seen(c->n_streams, 0);
		uint64_t first = 0;
		for(uint32_t r = 0; r < n_rx && !why; first += rx[r].n_channels, r++) {
			if(from[r] == -1) continue;
			const uint32_t o = (uint32_t)from[r];
			if(from[r] < -1 || o >= c->n_streams) { snprintf(buf, sizeof(buf), "entry %u continues receiver %d of %u", r, from[r], c->n_streams); why = buf; }
			else if(seen[o]) { snprintf(buf, sizeof(buf), "entry %u continues receiver %u, which an earlier entry continues", r, o); why = buf; }
			else if(rx[r].centerfreq != c->rx_centre[o] || rx[r].n_channels != c->rx_first[o + 1] - c->rx_first[o]
					|| rx[r].oversample != c->rx_in[o].oversample || rx[r].sample_fmt != c->rx_in[o].fmt
					|| !std::equal(freqs + first, freqs + first + rx[r].n_channels, c->freqs.begin() + c->rx_first[o])) {
				snprintf(buf, sizeof(buf), "entry %u does not repeat receiver %u's centre, channels, oversample, format and frequencies "
						"(retune with vdl2gpu_restart_receiver)", r, o);
				why = buf;
			}
			if(!why) seen[o] = 1;
		}
		if(!why && sum > 0xFFFFFFFFull) why = "more than 2^32 - 1 channels";
	}
	if(why) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_update_receivers: %s", why);
		return VDL2GPU_EINVAL;
	}
	CU(cudaSetDevice(c->device));
	vdl2gpu_config cfg = c->cfg;
	cfg.n_channels = (uint32_t)sum;
	cfg.freqs = freqs;
	cfg.n_streams = n_rx;
	std::vector<vdl2gpu_receiver> base(n_rx);
	for(uint32_t r = 0; r < n_rx; r++) { base[r].centerfreq = rx[r].centerfreq; base[r].n_channels = rx[r].n_channels; }
	ctx_layout n;
	push_rings p;
	int rc = setup_layout(n, cfg, base.data(), n_rx, rx, true, true, true, false, c->n_sms, c->n_slots, "vdl2gpu_update_receivers");
	if(rc == VDL2GPU_OK) rc = migrate_receivers(c, n, rx, from);
	if(rc == VDL2GPU_OK && c->push_ready) rc = carry_pushed(c, n, from, p);
	if(rc) return rc;
	/* the switch: the old layout and rings go with n and p, the graphs with the old chunk slots (the next spans capture
	 * anew, as after create) */
	std::swap(static_cast<ctx_layout &>(*c), n);
	if(c->push_ready) std::swap(static_cast<push_rings &>(*c), p);
	c->graph_nominal = 0;
	c->last_n_dec = 0;
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_get_receiver_positions(vdl2gpu_ctx *c, uint64_t *out, uint32_t n_rx) {
	if(!c || !out || !c->receivers || n_rx > c->n_streams) return VDL2GPU_EINVAL;
	for(uint32_t r = 0; r < n_rx; r++) out[r] = c->ragged ? c->rx_pos[r] : c->total_dec;
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_submit_span(vdl2gpu_ctx *c, const void *iq, uint32_t n_dec) {
	uint32_t len = 0;
	int rc = span_check(c, iq, n_dec, "vdl2gpu_submit_span", &len);
	if(rc < 0) return rc;
	if(rc == 0) return vdl2gpu_submit(c, iq, len);
	if(n_dec == 0) return VDL2GPU_OK;
	if(c->ragged) {
		const std::vector<uint32_t> n(c->n_streams, n_dec);
		return ragged_submit(c, iq, n.data(), false, nullptr, "vdl2gpu_submit_span");
	}
	CU(cudaSetDevice(c->device));
	chunk_slot *s;
	rc = acquire_slot(c, &s);
	if(rc) return rc;
	rc = ensure_raw(c, *s);
	if(rc) return rc;
	/* n_dec x span_bytes_per_dec <= max_chunk_bytes x n_rx, the size of the staging buffers */
	const size_t bytes = (size_t)n_dec * c->span_bytes_per_dec;
	memcpy(s->h_raw, iq, bytes);
	CU(cudaMemcpyAsync(s->d_raw, s->h_raw, bytes, cudaMemcpyHostToDevice, c->stream));
	return run_chain(c, *s, s->d_raw, n_dec);
}

extern "C" int vdl2gpu_submit_span_device(vdl2gpu_ctx *c, const void *dev_iq, uint32_t n_dec, void *producer_stream) {
	uint32_t len = 0;
	int rc = span_check(c, dev_iq, n_dec, "vdl2gpu_submit_span_device", &len);
	if(rc < 0) return rc;
	if(rc == 0) return vdl2gpu_submit_device(c, dev_iq, len, producer_stream);
	if(n_dec == 0) return VDL2GPU_OK;
	if(c->ragged) {
		const std::vector<uint32_t> n(c->n_streams, n_dec);
		return ragged_submit(c, dev_iq, n.data(), true, producer_stream, "vdl2gpu_submit_span_device");
	}
	CU(cudaSetDevice(c->device));
	chunk_slot *s;
	rc = acquire_slot(c, &s);
	if(rc) return rc;
	CU(cudaEventRecord(c->ev_input_ready, (cudaStream_t)producer_stream));
	CU(cudaStreamWaitEvent(c->stream, c->ev_input_ready, 0));
	return run_chain(c, *s, dev_iq, n_dec);
}

extern "C" int vdl2gpu_wait_input_consumed(vdl2gpu_ctx *c, void *stream) {
	if(!c) return VDL2GPU_EINVAL;
	CU(cudaStreamWaitEvent((cudaStream_t)stream, c->ev_input_consumed, 0));
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_stream_wait(vdl2gpu_ctx *c, void *stream) {
	if(!c) return VDL2GPU_EINVAL;
	CU(cudaSetDevice(c->device));
	CU(cudaEventRecord(c->ev_drain, c->s_back));        /* every chunk's chain ends on the back stream */
	CU(cudaStreamWaitEvent((cudaStream_t)stream, c->ev_drain, 0));
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_poll(vdl2gpu_ctx *c, vdl2gpu_frame_cb cb, void *user) {
	if(!c) return VDL2GPU_EINVAL;
	CU(cudaSetDevice(c->device));
	while(!c->inflight.empty()) {
		chunk_slot &s = c->chunks[c->inflight.front()];
		if(!s.busy) { c->inflight.pop_front(); continue; }
		cudaError_t q = cudaEventQuery(s.done);
		if(q == cudaErrorNotReady) break;
		if(q != cudaSuccess) return fail_cuda(q, "cudaEventQuery", __LINE__);
		harvest(c, s);
		c->inflight.pop_front();
	}
	return deliver(c, cb, user);
}

extern "C" int vdl2gpu_chunks_in_flight(vdl2gpu_ctx *c) {
	if(!c) return VDL2GPU_EINVAL;
	int n = 0;
	for(auto &s : c->chunks) n += s.busy ? 1 : 0;
	return n;
}

extern "C" int vdl2gpu_flush(vdl2gpu_ctx *c, vdl2gpu_frame_cb cb, void *user) {
	if(!c) return VDL2GPU_EINVAL;
	CU(cudaSetDevice(c->device));
	CU(cudaStreamSynchronize(c->stream));
	CU(cudaStreamSynchronize(c->s_back));
	while(!c->inflight.empty()) {
		chunk_slot &s = c->chunks[c->inflight.front()];
		if(s.busy) harvest(c, s);
		c->inflight.pop_front();
	}
	return deliver(c, cb, user);
}

static int read_counters(vdl2gpu_ctx *c, std::vector<uint32_t> &k3, std::vector<uint32_t> &sync, std::vector<uint32_t> &hdr) {
	CU(cudaSetDevice(c->device));
	CU(cudaStreamSynchronize(c->stream));
	CU(cudaStreamSynchronize(c->s_back));
	k3.resize((size_t)VDL2_NUM_COUNTERS * c->n_chp);
	sync.resize(c->n_chp); hdr.resize(c->n_chp);
	CU(cudaMemcpy(k3.data(), c->d_counters, k3.size() * 4, cudaMemcpyDeviceToHost));
	CU(cudaMemcpy(sync.data(), c->d_k2 + (size_t)K2_CNT_SYNC * c->n_chp, c->n_chp * 4, cudaMemcpyDeviceToHost));
	CU(cudaMemcpy(hdr.data(), c->d_k2 + (size_t)K2_CNT_HDR_GOOD * c->n_chp, c->n_chp * 4, cudaMemcpyDeviceToHost));
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_get_stats(vdl2gpu_ctx *c, vdl2gpu_stats *out) {
	if(!c || !out) return VDL2GPU_EINVAL;
	std::vector<uint32_t> k3, sync, hdr;
	int rc = read_counters(c, k3, sync, hdr);
	if(rc) return rc;
	uint64_t a = 0, b = 0;
	for(uint32_t ch = 0; ch < c->n_ch; ch++) { a += sync[slot_of(ch, c->lanes, c->full_warps)]; b += hdr[slot_of(ch, c->lanes, c->full_warps)]; }
	c->stats.demod_sync_good = a;
	c->stats.decoder_crc_good = b;
	*out = c->stats;
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_get_channel_counters(vdl2gpu_ctx *c, uint64_t *out, uint32_t n_channels) {
	if(!c || !out || n_channels > c->n_ch) return VDL2GPU_EINVAL;
	std::vector<uint32_t> k3, sync, hdr;
	int rc = read_counters(c, k3, sync, hdr);
	if(rc) return rc;
	for(uint32_t ch = 0; ch < n_channels; ch++) {
		uint64_t *o = out + (size_t)ch * VDL2_NUM_COUNTERS;
		for(int k = 0; k < VDL2_NUM_COUNTERS; k++) o[k] = k3[(size_t)k * c->n_chp + ch];
		o[VDL2_CNT_SYNC_GOOD] = sync[slot_of(ch, c->lanes, c->full_warps)];          /* K2's own counters live in its state planes, by slot */
		o[VDL2_CNT_HDR_CRC_GOOD] = hdr[slot_of(ch, c->lanes, c->full_warps)];
	}
	return VDL2GPU_OK;
}

/* Input levels (VDL2GPU_FLAG_INPUT_LEVELS): out[k] for the first n inputs, after everything submitted so far has run */
extern "C" int vdl2gpu_get_input_levels(vdl2gpu_ctx *c, vdl2gpu_input_levels *out, uint32_t n) {
	const char *why = nullptr;
	if(!c) why = "no context";
	else if(!out) why = "no output";
	else if(!c->d_levels) why = "the context was created without VDL2GPU_FLAG_INPUT_LEVELS";
	else if(n > c->n_streams) why = "more inputs asked for than the context has";
	if(why) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_get_input_levels: %s", why);
		return VDL2GPU_EINVAL;
	}
	if(n == 0) return VDL2GPU_OK;
	CU(cudaSetDevice(c->device));
	CU(cudaStreamSynchronize(c->stream));
	CU(cudaStreamSynchronize(c->s_back));
	std::vector<vdl2_levels> lv(n);
	CU(cudaMemcpy(lv.data(), c->d_levels, (size_t)n * sizeof(vdl2_levels), cudaMemcpyDeviceToHost));
	for(uint32_t k = 0; k < n; k++) {
		vdl2gpu_input_levels &o = out[k];
		o.samples = lv[k].samples;
		o.sum_i = (int64_t)lv[k].sum_i; o.sum_q = (int64_t)lv[k].sum_q;
		o.pow_lo = lv[k].pow_lo; o.pow_hi = lv[k].pow_hi;
		o.clipped = lv[k].clipped;
		o.peak = lv[k].peak;
		o.full_scale = vdl2_level_full_scale(c->mixed ? c->rx_in[k].fmt : c->cfg.sample_fmt);
	}
	return VDL2GPU_OK;
}

/* Spectrum (VDL2GPU_FLAG_SPECTRUM): out[k] for inputs [first, first + n), after everything submitted so far has run */
extern "C" int vdl2gpu_get_spectrum(vdl2gpu_ctx *c, uint32_t first, uint32_t n, vdl2gpu_spectrum *out) {
	const char *why = nullptr;
	if(!c) why = "no context";
	else if(!out) why = "no output";
	else if(!c->d_spec) why = "the context was created without VDL2GPU_FLAG_SPECTRUM";
	else if((uint64_t)first + n > c->n_streams) why = "inputs asked for past the context's last input";
	if(why) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_get_spectrum: %s", why);
		return VDL2GPU_EINVAL;
	}
	if(n == 0) return VDL2GPU_OK;
	CU(cudaSetDevice(c->device));
	CU(cudaStreamSynchronize(c->stream));
	CU(cudaStreamSynchronize(c->s_back));
	const vdl2_spec_acc *a = c->d_spec + first;
	CU(cudaMemcpy2D(out->pow_lo, sizeof(vdl2gpu_spectrum), a->lo, sizeof(vdl2_spec_acc), sizeof(a->lo), n, cudaMemcpyDeviceToHost));
	CU(cudaMemcpy2D(out->pow_hi, sizeof(vdl2gpu_spectrum), a->hi, sizeof(vdl2_spec_acc), sizeof(a->hi), n, cudaMemcpyDeviceToHost));
	CU(cudaMemcpy2D(out->peak, sizeof(vdl2gpu_spectrum), a->peak, sizeof(vdl2_spec_acc), sizeof(a->peak), n, cudaMemcpyDeviceToHost));
	for(uint32_t k = 0; k < n; k++) {
		const uint64_t pos = c->spec_pos[first + k];
		out[k].segments = pos >> VDL2_SPEC_LOG2N;
		out[k].pending = (uint32_t)(pos & (VDL2_SPEC_N - 1u));
		out[k].reserved = 0;
	}
	return VDL2GPU_OK;
}

/* Channel levels (VDL2GPU_FLAG_CHANNEL_LEVELS): out[k] for the first n channels, after everything submitted so far has run */
extern "C" int vdl2gpu_get_channel_levels(vdl2gpu_ctx *c, vdl2gpu_channel_levels *out, uint32_t n) {
	const char *why = nullptr;
	if(!c) why = "no context";
	else if(!out) why = "no output";
	else if(!c->d_chlv) why = "the context was created without VDL2GPU_FLAG_CHANNEL_LEVELS";
	else if(n > c->n_ch) why = "more channels asked for than the context has";
	if(why) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_get_channel_levels: %s", why);
		return VDL2GPU_EINVAL;
	}
	if(n == 0) return VDL2GPU_OK;
	CU(cudaSetDevice(c->device));
	CU(cudaStreamSynchronize(c->stream));
	CU(cudaStreamSynchronize(c->s_back));
	const size_t s = c->n_chp;
	std::vector<uint64_t> lv(VDL2_CHLV_ROWS * s);
	std::vector<uint32_t> peak(s), nf(2 * s);
	CU(cudaMemcpy(lv.data(), c->d_chlv, lv.size() * 8, cudaMemcpyDeviceToHost));
	CU(cudaMemcpy(peak.data(), c->d_chlv + VDL2_CHLV_ROWS * s, s * 4, cudaMemcpyDeviceToHost));
	CU(cudaMemcpy(nf.data(), c->d_k2 + (size_t)K2_MAG_LP * s, 2 * s * 4, cudaMemcpyDeviceToHost));     /* K2_MAG_LP, K2_MAG_NF */
	for(uint32_t k = 0; k < n; k++) {
		const size_t i = slot_of(k, c->lanes, c->full_warps);
		vdl2gpu_channel_levels &o = out[k];
		for(int b = 0; b < VDL2_CHLV_BINS; b++) o.hist[b] = lv[b * s + i];
		o.pow_lo = lv[VDL2_CHLV_POW_LO * s + i]; o.pow_hi = lv[VDL2_CHLV_POW_HI * s + i];
		memcpy(&o.peak_pow, &peak[i], 4);
		memcpy(&o.mag_lp, &nf[i], 4);
		memcpy(&o.mag_nf, &nf[s + i], 4);
		o.nf_pwr_dbfs = nf_pwr_dbfs(o.mag_nf);
	}
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_get_tables(vdl2gpu_ctx *c, float levels[256], float sin_lut[257], float cos_lut[257],
		float A[3], float B[3], float lr_X[16], float *lr_denom, float pr_phase[16]) {
	if(!c) return VDL2GPU_EINVAL;
	if(c->mixed) {
		snprintf(g_last_error, sizeof(g_last_error), "vdl2gpu_get_tables: a mixed-receivers context has no single sample rate (and filter)");
		return VDL2GPU_EINVAL;
	}
	if(levels) memcpy(levels, c->tab.t.levels, sizeof(c->tab.t.levels));
	if(sin_lut) memcpy(sin_lut, c->tab.sin_lut, sizeof(c->tab.sin_lut));
	if(cos_lut) memcpy(cos_lut, c->tab.cos_lut, sizeof(c->tab.cos_lut));
	if(A) memcpy(A, c->tab.t.A, 12);
	if(B) memcpy(B, c->tab.t.B, 12);
	if(lr_X) memcpy(lr_X, c->tab.t.lr_X, 64);
	if(lr_denom) *lr_denom = c->tab.t.lr_denom;
	if(pr_phase) memcpy(pr_phase, c->tab.t.pr_phase, 64);
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_read_dec(vdl2gpu_ctx *c, float *out, size_t cap_floats, uint32_t *n_dec) {
	if(!c || !out || !n_dec) return VDL2GPU_EINVAL;
	CU(cudaSetDevice(c->device));
	CU(cudaStreamSynchronize(c->stream));
	CU(cudaStreamSynchronize(c->s_back));
	*n_dec = c->last_n_dec;
	if((size_t)c->last_n_dec * c->n_ch * 2 > cap_floats) return VDL2GPU_ETOOBIG;
	if(c->last_n_dec == 0) return VDL2GPU_OK;
	/* slot == channel only without the balanced mapping, which can deal 32 channels (lanes == 32) to the first full_warps
	 * warps and 31 to the others */
	if(c->full_warps == 0xFFFFFFFFu) {
		CU(cudaMemcpy2D(out, (size_t)c->n_ch * sizeof(float2), c->d_dec3[(c->chunk_seq + 2) % 3u], (size_t)c->n_chp * sizeof(float2),
				(size_t)c->n_ch * sizeof(float2), c->last_n_dec, cudaMemcpyDeviceToHost));
	} else {
		std::vector<float2> tmp((size_t)c->last_n_dec * c->n_chp);
		CU(cudaMemcpy(tmp.data(), c->d_dec3[(c->chunk_seq + 2) % 3u], tmp.size() * sizeof(float2), cudaMemcpyDeviceToHost));
		for(uint32_t m = 0; m < c->last_n_dec; m++)
			for(uint32_t ch = 0; ch < c->n_ch; ch++) {
				const float2 v = tmp[(size_t)m * c->n_chp + slot_of(ch, c->lanes, c->full_warps)];
				out[((size_t)m * c->n_ch + ch) * 2] = v.x; out[((size_t)m * c->n_ch + ch) * 2 + 1] = v.y;
			}
	}
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_read_events(vdl2gpu_ctx *c, vdl2gpu_event *out, uint32_t cap) {
	if(!c || !out) return VDL2GPU_EINVAL;
	if(!(c->cfg.flags & VDL2GPU_FLAG_TRACE)) return 0;
	CU(cudaSetDevice(c->device));
	CU(cudaStreamSynchronize(c->stream));
	CU(cudaStreamSynchronize(c->s_back));
	vdl2_queue_ctl ctl;
	CU(cudaMemcpy(&ctl, c->d_ctl, sizeof(ctl), cudaMemcpyDeviceToHost));
	uint32_t total = std::min(ctl.n_events, c->event_cap);
	uint32_t n = total > c->events_read ? total - c->events_read : 0;
	if(n > cap) n = cap;
	if(n) CU(cudaMemcpy(out, (const vdl2gpu_event *)c->d_events + c->events_read, (size_t)n * sizeof(vdl2gpu_event), cudaMemcpyDeviceToHost));
	c->events_read += n;
	if(c->events_read == total) {
		/* drained: the buffer is not a ring, so start it over (nothing is running: both streams were synchronised above).
		 * Events the kernels could not store because it was full are counted and reported once the stored ones are out. */
		if(ctl.n_events > c->event_cap) c->events_dropped += ctl.n_events - c->event_cap;
		if(ctl.n_events) {
			const uint32_t zero = 0;
			CU(cudaMemcpy(reinterpret_cast<uint8_t *>(c->d_ctl.get()) + offsetof(vdl2_queue_ctl, n_events), &zero, sizeof(zero), cudaMemcpyHostToDevice));
			c->events_read = 0;
		}
	}
	if(n == 0 && c->events_dropped) {
		snprintf(g_last_error, sizeof(g_last_error), "trace buffer overflow: %llu events were not recorded (drain more often)", (unsigned long long)c->events_dropped);
		c->events_dropped = 0;
		return VDL2GPU_EOVERFLOW;
	}
	return (int)n;
}

extern "C" int vdl2gpu_enable_timing(vdl2gpu_ctx *c, int on) {
	if(!c) return VDL2GPU_EINVAL;
	c->timing = on != 0;
	if(on && !c->ev_t0) {
		CU(cudaSetDevice(c->device));
		CU(cudaEventCreate(c->ev_t0.put()));
		CU(cudaEventRecord(c->ev_t0, c->stream));
	}
	return VDL2GPU_OK;
}

/* diagnostic: the per-block scheduling records (VDL2GPU_BLOCK_TRACE=1 at create): 6 x uint64 per record
 * {kernel (1 K1, 2 K2), block, SM id, 0, start ns, end ns}; synchronises; returns the number of records copied */
extern "C" int vdl2gpu_debug_block_trace(vdl2gpu_ctx *c, uint64_t *out, uint32_t cap_records) {
	if(!c || !out) return VDL2GPU_EINVAL;
	if(!c->d_block_trace) return 0;
	CU(cudaSetDevice(c->device));
	CU(cudaDeviceSynchronize());
	uint32_t n = 0;
	CU(cudaMemcpy(&n, &c->d_block_trace->n, 4, cudaMemcpyDeviceToHost));
	n = std::min(std::min(n, c->block_trace_cap), cap_records);
	std::vector<vdl2_block_rec> r(n);
	if(n) CU(cudaMemcpy(r.data(), c->d_block_trace->rec, (size_t)n * sizeof(vdl2_block_rec), cudaMemcpyDeviceToHost));
	for(uint32_t k = 0; k < n; k++) {
		out[6 * k] = r[k].kernel; out[6 * k + 1] = r[k].block; out[6 * k + 2] = r[k].smid; out[6 * k + 3] = 0;
		out[6 * k + 4] = r[k].t_start; out[6 * k + 5] = r[k].t_end;
	}
	return (int)n;
}

extern "C" int vdl2gpu_get_timeline(vdl2gpu_ctx *c, float *out, uint32_t cap_rows) {
	if(!c || !out) return VDL2GPU_EINVAL;
	const uint32_t n = std::min<uint32_t>(cap_rows, (uint32_t)(c->timeline.size() / 8));
	memcpy(out, c->timeline.data(), (size_t)n * 8 * sizeof(float));
	return (int)n;
}

extern "C" int vdl2gpu_get_kernel_ms(vdl2gpu_ctx *c, double ms[5], uint64_t launches[5]) {
	if(!c || !ms) return VDL2GPU_EINVAL;
	for(int k = 0; k < 5; k++) { ms[k] = c->k_ms[k]; if(launches) launches[k] = c->k_launches[k]; }
	return VDL2GPU_OK;
}

/* ------------------------------------------------------------------------------------------------
 * raw launch stubs (device pointers in, device pointers out; no allocation, no synchronisation)
 * ---------------------------------------------------------------------------------------------- */
/* GF tables for the stand-alone RS stub, one copy per device, made on first use on that device */
static vdl2_tables *g_stub_tables[64] = { nullptr };
static std::mutex g_stub_lock;

static int stub_tables(vdl2_tables **out) {
	int dev = 0;
	CU(cudaGetDevice(&dev));
	if(dev < 0 || dev >= 64) return VDL2GPU_EINVAL;
	std::lock_guard<std::mutex> lk(g_stub_lock);
	if(!g_stub_tables[dev]) {
		host_tables *h = new host_tables();
		memset(h, 0, sizeof(*h));
		make_gf(h->t);
		vdl2_tables *d = nullptr;
		cudaError_t e = cudaMalloc(&d, sizeof(vdl2_tables));
		if(e == cudaSuccess) e = cudaMemcpy(d, &h->t, sizeof(vdl2_tables), cudaMemcpyHostToDevice);
		delete h;
		if(e != cudaSuccess) { cudaFree(d); return fail_cuda(e, "RS stub tables", __LINE__); }
		g_stub_tables[dev] = d;
	}
	*out = g_stub_tables[dev];
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_launch_convert(const void *raw, uint32_t n_pairs, uint32_t sample_fmt, const float *levels256,
		float *samples_out, void *stream) {
	if(!raw || !samples_out || sample_fmt > 1 || (sample_fmt == 0 && !levels256)) return VDL2GPU_EINVAL;
	KL(vdl2_launch_k0(raw, n_pairs, sample_fmt, levels256, samples_out, 1, 0, 0, nullptr, nullptr, (cudaStream_t)stream));
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_launch_fcs_crc16(const uint8_t *frames, const uint32_t *offsets, const uint32_t *lens,
		uint32_t n_frames, uint16_t *residues_out, void *stream) {
	if(n_frames && (!frames || !offsets || !lens || !residues_out)) return VDL2GPU_EINVAL;
	KL(vdl2_launch_k4(frames, offsets, lens, n_frames, residues_out, (cudaStream_t)stream));
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_launch_rs_verify(uint8_t *blocks, const int32_t *fec_octets, uint32_t n_blocks, int32_t *ret_out, void *stream) {
	if(n_blocks && (!blocks || !fec_octets || !ret_out)) return VDL2GPU_EINVAL;
	vdl2_tables *t = nullptr;
	int rc = stub_tables(&t);            /* first call on a device allocates; later calls only launch */
	if(rc) return rc;
	KL(vdl2_launch_rs(blocks, fec_octets, n_blocks, ret_out, t, (cudaStream_t)stream));
	return VDL2GPU_OK;
}

/* K2a on its own: phase_out[i] = (float)atan2((double)im, (double)re), mag_out[i] = hypotf(re, im) of n_elems
 * decimated samples (src/demod.c:232,238,256).  exact_libm = 0: the Ziv-guarded short evaluation the pipeline
 * uses (vdl2_fastmath.cuh); 1: vdl2_phase_of / vdl2_mag_of for every element (no fast path).  Both give the same floats. */
extern "C" int vdl2gpu_launch_phase_mag(const float *dec, uint32_t n_elems, float *phase_out, float *mag_out, int exact_libm, void *stream) {
	if(n_elems && (!dec || !phase_out || !mag_out)) return VDL2GPU_EINVAL;
	if(n_elems == 0) return VDL2GPU_OK;
	int dev = 0;
	CU(cudaGetDevice(&dev));
	KL(vdl2_kernels_init_device(dev));
	vdl2_k2_params p2;
	memset(&p2, 0, sizeof(p2));
	/* one row of n_elems "channels": K2a is element-wise, the row structure does not matter */
	p2.dec = reinterpret_cast<const float2 *>(dec); p2.n_dec = 1; p2.n_ch = n_elems; p2.n_chp = n_elems; p2.lanes = 32; p2.full_warps = 0xFFFFFFFFu;
	p2.phase = phase_out - (size_t)VDL2_SYNC_BUFLEN * n_elems;       /* the launcher skips the 160 history rows */
	p2.mag = mag_out; p2.k2a_mode = exact_libm ? 0u : 1u;
	KL(vdl2_launch_k2a(&p2, (cudaStream_t)stream));
	return VDL2GPU_OK;
}

/* ---- stage stubs: K1, K2 (+K2a), K3 one at a time, on device memory the caller owns ---- */
struct vdl2gpu_stage {
	vdl2gpu_config cfg;
	std::vector<uint32_t> freqs;
	host_tables tab;
	uint32_t n_ch = 0, n_chp = 0, max_dec = 0, n_slots = 0, event_cap = 0;
	uint32_t decim_cnt = 0;
	uint64_t total_dec = 0;
	uint32_t events_read = 0;
	int k1_variant = 2, k2_variant = 5, k2a_mode = 1;
	vdl2_tables *d_tab = nullptr;
	uint32_t *d_k1 = nullptr, *d_k2 = nullptr, *d_counters = nullptr, *d_ready = nullptr;
	float *d_ring = nullptr, *d_phase = nullptr, *d_mag = nullptr, *d_hist_tmp = nullptr;
	vdl2_burst_slot *d_pool = nullptr;
	int32_t *d_free = nullptr;
	vdl2_queue_ctl *d_ctl = nullptr;
	void *d_events = nullptr;
};

static size_t al256(size_t x) { return (x + 255u) & ~(size_t)255u; }

struct stage_layout {
	size_t tab, k1, k2, counters, ring, phase, mag, hist, pool, free_list, ready, ctl, events, total;
};

static stage_layout stage_layout_of(uint32_t n_ch, uint32_t max_dec, uint32_t event_cap) {
	const size_t n_chp = (n_ch + 31u) & ~31u, n_slots = std::max(256u, 3u * n_ch);
	stage_layout L;
	size_t o = 0;
	L.tab = o; o += al256(sizeof(vdl2_tables));
	L.k1 = o; o += al256((size_t)K1_NFIELDS * n_chp * 4);
	L.k2 = o; o += al256((size_t)K2_NFIELDS * n_chp * 4);
	L.counters = o; o += al256((size_t)VDL2_NUM_COUNTERS * n_chp * 4);
	L.ring = o; o += al256((size_t)VDL2_SYNC_BUFLEN * n_chp * 4);
	L.phase = o; o += al256((size_t)(max_dec + VDL2_SYNC_BUFLEN) * n_chp * 4);
	L.mag = o; o += al256((size_t)max_dec * n_chp * 4);
	L.hist = o; o += al256((size_t)VDL2_SYNC_BUFLEN * n_chp * 4);
	L.pool = o; o += al256(n_slots * sizeof(vdl2_burst_slot));
	L.free_list = o; o += al256(n_slots * 4);
	L.ready = o; o += al256(n_slots * 4);
	L.ctl = o; o += al256(sizeof(vdl2_queue_ctl));
	L.events = o; o += al256((size_t)event_cap * sizeof(vdl2gpu_event));
	L.total = o;
	return L;
}

static uint32_t stage_event_cap(uint32_t flags) { return (flags & VDL2GPU_FLAG_TRACE) ? (1u << 18) : 1u; }

extern "C" size_t vdl2gpu_stage_device_bytes(uint32_t n_channels, uint32_t max_dec, uint32_t flags) {
	return stage_layout_of(n_channels, max_dec, stage_event_cap(flags)).total;
}

extern "C" uint32_t vdl2gpu_stage_row_stride(uint32_t n_channels) { return (n_channels + 31u) & ~31u; }

/* initial per-channel state: vdl2_channel_init + demod_reset (src/demod.c:205-220,379-392), process_samples locals
 * (src/demod.c:289-298); shared by the batch context and the stage stubs */
static void initial_state(const vdl2gpu_config &cfg, const uint32_t *freqs, const uint32_t *centres, const uint32_t *rates, uint32_t n_ch,
		uint32_t n_chp, uint32_t lanes, uint32_t full_warps, std::vector<uint32_t> &k1, std::vector<uint32_t> &k2) {
	k1.assign((size_t)K1_NFIELDS * n_chp, 0u); k2.assign((size_t)K2_NFIELDS * n_chp, 0u);
	for(uint32_t chan = 0; chan < n_ch; chan++) {
		const uint32_t ch = slot_of(chan, lanes, full_warps);          /* index into the per-channel planes */
		const uint32_t centre = centres ? centres[chan] : cfg.centerfreq;     /* centres: per channel, multi-receiver context */
		const uint32_t rate = rates ? rates[chan] : cfg.sample_rate;          /* rates: per channel, mixed-rate receivers */
		/* the same fresh state a restart gives (vdl2_core.cuh; the ring of zeros is the cudaMemset of create) */
		vdl2_k1_fresh(k1.data(), n_chp, ch, vdl2_nco_dphi(centre, freqs[chan], rate));
		vdl2_chan v;
		vdl2_chan_init(v, freqs[chan]);
		vdl2_chan_store(v, k2.data(), n_chp, ch);
	}
}

extern "C" int vdl2gpu_stage_create(const vdl2gpu_config *cfg, uint32_t max_dec, void *device_mem, size_t device_bytes, vdl2gpu_stage **out) {
	if(!cfg || !out || !device_mem || !cfg->freqs || cfg->n_channels == 0 || cfg->oversample == 0 || max_dec == 0
			|| cfg->sample_rate != (uint32_t)VDL2_SYMBOL_RATE * VDL2_SPS * cfg->oversample) return VDL2GPU_EINVAL;
	if(cfg->flags & VDL2GPU_FLAG_RAGGED) return refuse_ragged("vdl2gpu_stage_create");
	const uint32_t ecap = stage_event_cap(cfg->flags);
	const stage_layout L = stage_layout_of(cfg->n_channels, max_dec, ecap);
	if(device_bytes < L.total || ((uintptr_t)device_mem & 255u)) return VDL2GPU_EINVAL;
	int dev = 0;
	CU(cudaGetDevice(&dev));
	KL(vdl2_kernels_init_device(dev));
	vdl2gpu_stage *st = new vdl2gpu_stage();
	st->cfg = *cfg;
	st->freqs.assign(cfg->freqs, cfg->freqs + cfg->n_channels);
	st->cfg.freqs = st->freqs.data();
	st->n_ch = cfg->n_channels; st->n_chp = (st->n_ch + 31u) & ~31u; st->max_dec = max_dec;
	st->n_slots = std::max(256u, 3u * st->n_ch); st->event_cap = ecap;
	const char *e;
	if((e = getenv("VDL2GPU_K1_VARIANT"))) st->k1_variant = atoi(e);
	if((e = getenv("VDL2GPU_K2_VARIANT"))) st->k2_variant = atoi(e);
	if((e = getenv("VDL2GPU_K2A"))) st->k2a_mode = atoi(e);
	make_tables(st->tab, cfg->sample_rate);
	uint8_t *b = static_cast<uint8_t *>(device_mem);
	st->d_tab = reinterpret_cast<vdl2_tables *>(b + L.tab); st->d_k1 = reinterpret_cast<uint32_t *>(b + L.k1);
	st->d_k2 = reinterpret_cast<uint32_t *>(b + L.k2); st->d_counters = reinterpret_cast<uint32_t *>(b + L.counters);
	st->d_ring = reinterpret_cast<float *>(b + L.ring); st->d_phase = reinterpret_cast<float *>(b + L.phase);
	st->d_mag = reinterpret_cast<float *>(b + L.mag); st->d_hist_tmp = reinterpret_cast<float *>(b + L.hist);
	st->d_pool = reinterpret_cast<vdl2_burst_slot *>(b + L.pool); st->d_free = reinterpret_cast<int32_t *>(b + L.free_list);
	st->d_ready = reinterpret_cast<uint32_t *>(b + L.ready); st->d_ctl = reinterpret_cast<vdl2_queue_ctl *>(b + L.ctl);
	st->d_events = b + L.events;
	std::vector<uint32_t> k1, k2;
	initial_state(st->cfg, st->freqs.data(), nullptr, nullptr, st->n_ch, st->n_chp, 32u, 0xFFFFFFFFu, k1, k2);
	std::vector<int32_t> fl(st->n_slots);
	for(uint32_t i = 0; i < st->n_slots; i++) fl[i] = (int32_t)i;
	vdl2_queue_ctl ctl;
	memset(&ctl, 0, sizeof(ctl));
	ctl.free_top = (int32_t)st->n_slots;
	cudaError_t ce = cudaMemset(device_mem, 0, L.total);
	if(ce == cudaSuccess) ce = cudaMemcpy(st->d_tab, &st->tab.t, sizeof(vdl2_tables), cudaMemcpyHostToDevice);
	if(ce == cudaSuccess) ce = cudaMemcpy(st->d_k1, k1.data(), k1.size() * 4, cudaMemcpyHostToDevice);
	if(ce == cudaSuccess) ce = cudaMemcpy(st->d_k2, k2.data(), k2.size() * 4, cudaMemcpyHostToDevice);
	if(ce == cudaSuccess) ce = cudaMemcpy(st->d_free, fl.data(), fl.size() * 4, cudaMemcpyHostToDevice);
	if(ce == cudaSuccess) ce = cudaMemcpy(st->d_ctl, &ctl, sizeof(ctl), cudaMemcpyHostToDevice);
	if(ce != cudaSuccess) { delete st; return fail_cuda(ce, "vdl2gpu_stage_create", __LINE__); }
	*out = st;
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_stage_destroy(vdl2gpu_stage *st) { delete st; return VDL2GPU_OK; }

extern "C" int vdl2gpu_stage_levels(vdl2gpu_stage *st, const float **levels256_dev) {
	if(!st || !levels256_dev) return VDL2GPU_EINVAL;
	*levels256_dev = st->d_tab->levels;
	return VDL2GPU_OK;
}

/* K1 == the per-sample loop of process_samples (src/demod.c:288-337) for every channel of the stage */
extern "C" int vdl2gpu_launch_mix_iir_decimate(vdl2gpu_stage *st, const float *samples, uint32_t n_pairs, float *dec_out,
		uint32_t *n_dec_out, void *stream) {
	if(!st || (n_pairs && (!samples || !dec_out))) return VDL2GPU_EINVAL;
	const uint32_t os = st->cfg.oversample;
	const uint32_t n_dec = (st->decim_cnt + n_pairs) / os;
	if(n_dec > st->max_dec) return VDL2GPU_ETOOBIG;
	vdl2_k1_params p1;
	memset(&p1, 0, sizeof(p1));
	p1.samples = reinterpret_cast<const float2 *>(samples); p1.n_pairs = n_pairs; p1.oversample = os; p1.cnt0 = st->decim_cnt;
	p1.n_ch = st->n_ch; p1.n_chp = st->n_chp; p1.lanes = 32; p1.full_warps = 0xFFFFFFFFu; p1.dec = reinterpret_cast<float2 *>(dec_out); p1.state = st->d_k1;
	p1.lut = reinterpret_cast<const float4 *>(st->d_tab->lut);
	p1.a0 = st->tab.t.A[0]; p1.a1 = st->tab.t.A[1]; p1.a2 = st->tab.t.A[2]; p1.b1 = st->tab.t.B[1]; p1.b2 = st->tab.t.B[2];
	p1.one = 1.0f; p1.neg_one = -1.0f; p1.two = 2.0f;
	KL(vdl2_launch_k1(&p1, (st->cfg.flags & VDL2GPU_FLAG_K1_SCALAR) ? 1 : 0, st->k1_variant, (cudaStream_t)stream));
	st->decim_cnt = (st->decim_cnt + n_pairs) % os;
	if(n_dec_out) *n_dec_out = n_dec;
	return VDL2GPU_OK;
}

/* K2a + K2 == demod() (src/demod.c:222-286) + the header part of decode_vdl2_burst (src/decode.c:198-258) over n_dec
 * decimated samples of every channel; completed bursts queue up for vdl2gpu_launch_burst_fec */
extern "C" int vdl2gpu_launch_sync_slice(vdl2gpu_stage *st, const float *dec, uint32_t n_dec, void *stream) {
	if(!st || (n_dec && !dec)) return VDL2GPU_EINVAL;
	if(n_dec > st->max_dec) return VDL2GPU_ETOOBIG;
	if(n_dec == 0) return VDL2GPU_OK;
	vdl2_k2_params p2;
	memset(&p2, 0, sizeof(p2));
	p2.dec = reinterpret_cast<const float2 *>(dec); p2.phase = st->d_phase; p2.mag = st->d_mag; p2.hist_tmp = st->d_hist_tmp;
	p2.n_dec = n_dec; p2.n_ch = st->n_ch; p2.n_chp = st->n_chp; p2.lanes = 32; p2.full_warps = 0xFFFFFFFFu; p2.dec_base = st->total_dec;
	p2.state = st->d_k2; p2.ring = st->d_ring; p2.tables = st->d_tab; p2.max_ppm = st->cfg.max_ppm; p2.s27 = st->tab.s27;
	p2.pool = st->d_pool; p2.free_list = st->d_free; p2.ready = st->d_ready; p2.ctl = st->d_ctl;
	p2.events = st->d_events; p2.event_cap = st->event_cap; p2.trace = (st->cfg.flags & VDL2GPU_FLAG_TRACE) ? 1u : 0u;
	p2.variant = (uint32_t)st->k2_variant; p2.k2a_mode = (uint32_t)st->k2a_mode;
	KL(vdl2_launch_k2a(&p2, (cudaStream_t)stream));
	KL(vdl2_launch_k2(&p2, (cudaStream_t)stream));
	KL(vdl2_launch_copy_hist(&p2, (cudaStream_t)stream));
	st->total_dec += n_dec;
	return VDL2GPU_OK;
}

/* K3 (+K4) == the data part of decode_vdl2_burst (src/decode.c:259-380) for every queued burst.  `region` receives a
 * vdl2_out_header followed by the burst records (device memory or mapped pinned host memory, 16-byte aligned);
 * vdl2gpu_parse_records turns a host copy of it into frames. */
extern "C" int vdl2gpu_launch_burst_fec(vdl2gpu_stage *st, uint8_t *region, uint32_t region_bytes, void *stream) {
	if(!st || !region || region_bytes < sizeof(vdl2_out_header) + 256u || ((uintptr_t)region & 15u)) return VDL2GPU_EINVAL;
	vdl2_k3_params p3;
	memset(&p3, 0, sizeof(p3));
	p3.pool = st->d_pool; p3.free_list = st->d_free; p3.ready = st->d_ready; p3.ctl = st->d_ctl; p3.tables = st->d_tab;
	p3.out = region; p3.out_cap = region_bytes - (uint32_t)sizeof(vdl2_out_header); p3.n_chp = st->n_chp; p3.counters = st->d_counters;
	KL(vdl2_launch_k3(&p3, K3_GRID, (cudaStream_t)stream));
	return VDL2GPU_OK;
}

/* Queue n bursts exactly as K2 hands them over (vdl2_burst_complete): pop n slots from the device free list (burst i takes
 * the i-th pop), write each slot's header and its first ceil(nbits / 32) words only - the slot's later words keep whatever
 * an earlier burst left there - then ready[0..n), n_ready and free_top.  Synchronous. */
static_assert(sizeof(vdl2gpu_burst) == 48, "vdl2gpu_burst is part of the ABI");
extern "C" int vdl2gpu_stage_queue_bursts(vdl2gpu_stage *st, const vdl2gpu_burst *bursts, uint32_t n) {
	if(!st || (n && !bursts)) return VDL2GPU_EINVAL;
	for(uint32_t i = 0; i < n; i++) {
		const vdl2gpu_burst &b = bursts[i];
		if(b.channel >= st->n_ch || b.nbits > VDL2_MAX_BURST_BITS || (b.nbits && !b.words)) return VDL2GPU_EINVAL;
	}
	CU(cudaDeviceSynchronize());
	vdl2_queue_ctl ctl;
	CU(cudaMemcpy(&ctl, st->d_ctl, sizeof(ctl), cudaMemcpyDeviceToHost));
	if(ctl.n_ready) return VDL2GPU_EINVAL;                   /* the previous queue has not been decoded yet */
	if(ctl.free_top < 0 || n > (uint32_t)ctl.free_top) return VDL2GPU_ETOOBIG;
	if(n == 0) return VDL2GPU_OK;
	std::vector<int32_t> popped(n);
	CU(cudaMemcpy(popped.data(), st->d_free + (ctl.free_top - (int32_t)n), (size_t)n * 4, cudaMemcpyDeviceToHost));
	std::vector<uint32_t> ready(n);
	std::vector<uint8_t> buf(sizeof(vdl2_burst_slot));
	for(uint32_t i = 0; i < n; i++) {
		const vdl2gpu_burst &b = bursts[i];
		const int32_t slot = popped[n - 1u - i];                /* the free list is a stack: the top entry goes first */
		vdl2_burst_slot *s = reinterpret_cast<vdl2_burst_slot *>(buf.data());
		s->channel = b.channel; s->burst_seq = i; s->datalen_bits = b.datalen_bits; s->syndrome = b.syndrome; s->nbits = b.nbits;
		s->frame_pwr = b.frame_pwr; s->mag_nf = b.mag_nf; s->ppm_error = b.ppm_error;
		s->sync_lo = (uint32_t)b.sync_dec_index; s->sync_hi = (uint32_t)(b.sync_dec_index >> 32); s->freq = b.freq; s->pad = 0;
		const size_t nw = (b.nbits + 31u) / 32u;
		if(nw) memcpy(s->words, b.words, nw * 4);
		CU(cudaMemcpy(&st->d_pool[slot], s, offsetof(vdl2_burst_slot, words) + nw * 4, cudaMemcpyHostToDevice));
		ready[i] = (uint32_t)slot;
	}
	CU(cudaMemcpy(st->d_ready, ready.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
	ctl.free_top -= (int32_t)n;
	ctl.n_ready = n;
	static_assert(offsetof(vdl2_queue_ctl, n_ready) == sizeof(int32_t), "free_top and n_ready are the first two fields");
	CU(cudaMemcpy(st->d_ctl, &ctl, 2 * sizeof(uint32_t), cudaMemcpyHostToDevice));
	return VDL2GPU_OK;
}

/* the stage's per-channel counters, 9 x uint64 per channel in the order of vdl2gpu_get_channel_counters.  Synchronises. */
extern "C" int vdl2gpu_stage_read_counters(vdl2gpu_stage *st, uint64_t *out) {
	if(!st || !out) return VDL2GPU_EINVAL;
	CU(cudaDeviceSynchronize());
	std::vector<uint32_t> k3((size_t)VDL2_NUM_COUNTERS * st->n_chp), sync(st->n_chp), hdr(st->n_chp);
	CU(cudaMemcpy(k3.data(), st->d_counters, k3.size() * 4, cudaMemcpyDeviceToHost));
	CU(cudaMemcpy(sync.data(), st->d_k2 + (size_t)K2_CNT_SYNC * st->n_chp, st->n_chp * 4, cudaMemcpyDeviceToHost));
	CU(cudaMemcpy(hdr.data(), st->d_k2 + (size_t)K2_CNT_HDR_GOOD * st->n_chp, st->n_chp * 4, cudaMemcpyDeviceToHost));
	for(uint32_t ch = 0; ch < st->n_ch; ch++) {              /* a stage maps channel c to slot c */
		uint64_t *o = out + (size_t)ch * VDL2_NUM_COUNTERS;
		for(int k = 0; k < VDL2_NUM_COUNTERS; k++) o[k] = k3[(size_t)k * st->n_chp + ch];
		o[VDL2_CNT_SYNC_GOOD] = sync[ch];
		o[VDL2_CNT_HDR_CRC_GOOD] = hdr[ch];
	}
	return VDL2GPU_OK;
}

extern "C" int vdl2gpu_stage_read_events(vdl2gpu_stage *st, vdl2gpu_event *out, uint32_t cap) {
	if(!st || !out) return VDL2GPU_EINVAL;
	if(!(st->cfg.flags & VDL2GPU_FLAG_TRACE)) return 0;
	CU(cudaDeviceSynchronize());
	vdl2_queue_ctl ctl;
	CU(cudaMemcpy(&ctl, st->d_ctl, sizeof(ctl), cudaMemcpyDeviceToHost));
	uint32_t total = std::min(ctl.n_events, st->event_cap);
	uint32_t n = total > st->events_read ? total - st->events_read : 0;
	if(n > cap) n = cap;
	if(n) CU(cudaMemcpy(out, (const vdl2gpu_event *)st->d_events + st->events_read, (size_t)n * sizeof(vdl2gpu_event), cudaMemcpyDeviceToHost));
	st->events_read += n;
	return (int)n;
}

extern "C" int vdl2gpu_parse_records(const uint8_t *region_host, uint32_t region_bytes, uint32_t decimated_rate,
		vdl2gpu_frame_cb cb, void *user) {
	if(!region_host || region_bytes < sizeof(vdl2_out_header)) return VDL2GPU_EINVAL;
	std::vector<pending_frame> pending;
	vdl2gpu_stats stats;
	memset(&stats, 0, sizeof(stats));
	struct timeval now;
	gettimeofday(&now, NULL);
	parse_region(region_host, region_bytes - (uint32_t)sizeof(vdl2_out_header), (double)decimated_rate, now, 0, 0, pending, stats);
	const uint8_t *base = region_host + sizeof(vdl2_out_header);
	for(auto &pf : pending) {
		pf.f.data = base + pf.offset;
		if(cb) cb(&pf.f, user);
	}
	if(stats.pool_overflows || stats.out_overflows) return VDL2GPU_EOVERFLOW;
	return (int)pending.size();
}
