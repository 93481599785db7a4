"""Python face of libvdl2gpu.so (ctypes over the C-ABI in include/vdl2gpu.h).

The names mirror the reference's interface for this path: a `Vdl2Channels` object is the set of
vdl2_channel_t's created by vdl2_channel_init (src/demod.c:379-392); `process_buf_uchar` /
`process_buf_short` (src/demod.c:339-365) feed it; frames come back with the metadata of
decode_frame / vdl2_msg_metadata (src/decode.c:173-194, src/output-common.h:31-43) instead of through
avlc_decoder_queue_push.  There is no CPU path: constructing the object without the built extension or
without an H100 raises.
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvdl2gpu.so")
FMT_U8, FMT_S16 = 0, 1
FLAG_TRACE, FLAG_KEEP_DEC, FLAG_K1_SCALAR, FLAG_NO_OVERLAP, FLAG_NO_GRAPH, FLAG_RAGGED = 1, 2, 4, 8, 16, 32
FLAG_INPUT_LEVELS = 64
FLAG_CHANNEL_LEVELS = 128
FLAG_SPECTRUM = 256
SPECTRUM_BINS = 1024
CHANNEL_LEVEL_BINS = 40
NUM_COUNTERS = 9
COUNTER_NAMES = ["sync_good", "hdr_crc_good", "bursts", "burst_err", "blocks_processed",
                 "blocks_fec_ok", "msg_good", "fcs_good", "fcs_bad"]


class Vdl2GpuError(RuntimeError):
    pass


class _Timeval(C.Structure):
    _fields_ = [("tv_sec", C.c_long), ("tv_usec", C.c_long)]


class _Config(C.Structure):
    _fields_ = [("sample_rate", C.c_uint32), ("oversample", C.c_uint32), ("sample_fmt", C.c_uint32),
                ("centerfreq", C.c_uint32), ("n_channels", C.c_uint32), ("freqs", C.POINTER(C.c_uint32)),
                ("max_ppm", C.c_float), ("max_chunk_bytes", C.c_uint32), ("device", C.c_int32),
                ("flags", C.c_uint32), ("n_inflight", C.c_uint32), ("n_streams", C.c_uint32), ("reserved", C.c_uint32 * 4)]


class _Receiver(C.Structure):
    _fields_ = [("centerfreq", C.c_uint32), ("n_channels", C.c_uint32)]


class _ReceiverEx(C.Structure):
    _fields_ = [("centerfreq", C.c_uint32), ("n_channels", C.c_uint32), ("oversample", C.c_uint32), ("sample_fmt", C.c_uint32)]


class _Frame(C.Structure):
    _fields_ = [("channel", C.c_uint32), ("freq", C.c_uint32), ("burst_seq", C.c_uint32), ("idx", C.c_int32),
                ("data", C.POINTER(C.c_uint8)), ("len", C.c_uint32), ("synd_weight", C.c_uint32),
                ("datalen_octets", C.c_uint32), ("num_fec_corrections", C.c_int32),
                ("frame_pwr_dbfs", C.c_float), ("nf_pwr_dbfs", C.c_float), ("ppm_error", C.c_float),
                ("frame_pwr", C.c_float), ("mag_nf", C.c_float), ("sync_dec_index", C.c_uint64),
                ("burst_timestamp", _Timeval), ("fcs_residue", C.c_uint16), ("fcs_ok", C.c_uint16)]


class _Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in
                ("chunks_submitted", "chunks_completed", "iq_samples", "dec_samples", "demod_sync_good",
                 "decoder_crc_good", "bursts", "burst_errors", "blocks_processed", "blocks_fec_ok", "msg_good",
                 "fcs_good", "fcs_bad", "pool_overflows", "out_overflows", "kernel_launches", "out_bytes", "graph_launches")] + [("reserved", C.c_uint64 * 2)]


class _InputLevels(C.Structure):
    _fields_ = [("samples", C.c_uint64), ("sum_i", C.c_int64), ("sum_q", C.c_int64), ("pow_lo", C.c_uint64),
                ("pow_hi", C.c_uint64), ("clipped", C.c_uint64), ("peak", C.c_uint32), ("full_scale", C.c_uint32)]


class _ChannelLevels(C.Structure):
    _fields_ = [("hist", C.c_uint64 * CHANNEL_LEVEL_BINS), ("pow_lo", C.c_uint64), ("pow_hi", C.c_uint64), ("peak_pow", C.c_float),
                ("mag_lp", C.c_float), ("mag_nf", C.c_float), ("nf_pwr_dbfs", C.c_float)]


class _Spectrum(C.Structure):
    _fields_ = [("segments", C.c_uint64), ("pending", C.c_uint32), ("reserved", C.c_uint32), ("pow_lo", C.c_uint64 * SPECTRUM_BINS),
                ("pow_hi", C.c_uint64 * SPECTRUM_BINS), ("peak", C.c_float * SPECTRUM_BINS)]


class _Event(C.Structure):
    _fields_ = [("channel", C.c_uint32), ("kind", C.c_uint32), ("dec_index", C.c_uint64),
                ("i", C.c_int32 * 8), ("f", C.c_float * 8)]


class _Burst(C.Structure):
    _fields_ = [("channel", C.c_uint32), ("datalen_bits", C.c_uint32), ("nbits", C.c_uint32), ("syndrome", C.c_uint32),
                ("frame_pwr", C.c_float), ("mag_nf", C.c_float), ("ppm_error", C.c_float), ("freq", C.c_uint32),
                ("sync_dec_index", C.c_uint64), ("words", C.POINTER(C.c_uint32))]


_FRAME_CB = C.CFUNCTYPE(None, C.POINTER(_Frame), C.c_void_p)
_LIB = None


def load_library():
    """Load libvdl2gpu.so; raises if it has not been built (python -m dumpvdl2_b200.build)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise Vdl2GpuError(f"{LIB_PATH} is missing: build it with `python -m dumpvdl2_b200.build` "
                           "(nvcc, sm_90a). There is no CPU fallback for the demodulator path.")
    L = C.CDLL(LIB_PATH)
    L.vdl2gpu_create.argtypes = [C.POINTER(_Config), C.POINTER(C.c_void_p)]
    L.vdl2gpu_create_receivers.argtypes = [C.POINTER(_Config), C.POINTER(_Receiver), C.c_uint32, C.POINTER(C.c_void_p)]
    L.vdl2gpu_create_mixed_receivers.argtypes = [C.POINTER(_Config), C.POINTER(_ReceiverEx), C.c_uint32, C.POINTER(C.c_void_p)]
    L.vdl2gpu_submit_span.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.vdl2gpu_submit_span_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    L.vdl2gpu_submit_ragged.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.vdl2gpu_submit_ragged_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.vdl2gpu_get_receiver_positions.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.vdl2gpu_restart_receiver.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    L.vdl2gpu_update_receivers.argtypes = [C.c_void_p, C.POINTER(_ReceiverEx), C.c_void_p, C.c_uint32, C.c_void_p]
    L.vdl2gpu_push.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    L.vdl2gpu_submit_pushed.argtypes = [C.c_void_p]
    L.vdl2gpu_destroy.argtypes = [C.c_void_p]
    L.vdl2gpu_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.vdl2gpu_submit_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    L.vdl2gpu_submit_planar_s16.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    L.vdl2gpu_serialize_raw_frame.argtypes = [C.POINTER(_Frame), C.c_char_p, C.c_void_p, C.c_size_t]
    L.vdl2gpu_wait_input_consumed.argtypes = [C.c_void_p, C.c_void_p]
    L.vdl2gpu_stream_wait.argtypes = [C.c_void_p, C.c_void_p]
    L.vdl2gpu_poll.argtypes = [C.c_void_p, _FRAME_CB, C.c_void_p]
    L.vdl2gpu_flush.argtypes = [C.c_void_p, _FRAME_CB, C.c_void_p]
    L.vdl2gpu_get_stats.argtypes = [C.c_void_p, C.POINTER(_Stats)]
    L.vdl2gpu_get_channel_counters.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.vdl2gpu_get_input_levels.argtypes = [C.c_void_p, C.POINTER(_InputLevels), C.c_uint32]
    L.vdl2gpu_get_channel_levels.argtypes = [C.c_void_p, C.POINTER(_ChannelLevels), C.c_uint32]
    L.vdl2gpu_get_spectrum.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(_Spectrum)]
    L.vdl2gpu_get_tables.argtypes = [C.c_void_p] + [C.c_void_p] * 8
    L.vdl2gpu_read_dec.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_uint32)]
    L.vdl2gpu_read_events.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.vdl2gpu_enable_timing.argtypes = [C.c_void_p, C.c_int]
    L.vdl2gpu_get_kernel_ms.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.vdl2gpu_get_timeline.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.vdl2gpu_debug_block_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.vdl2gpu_strerror.restype = C.c_char_p
    L.vdl2gpu_strerror.argtypes = [C.c_int]
    L.vdl2gpu_last_error.restype = C.c_char_p
    L.vdl2gpu_launch_convert.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.vdl2gpu_launch_fcs_crc16.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    L.vdl2gpu_launch_rs_verify.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    L.vdl2gpu_launch_phase_mag.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    L.vdl2gpu_chunks_in_flight.argtypes = [C.c_void_p]
    L.vdl2gpu_stage_device_bytes.restype = C.c_size_t
    L.vdl2gpu_stage_device_bytes.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
    L.vdl2gpu_stage_row_stride.restype = C.c_uint32
    L.vdl2gpu_stage_row_stride.argtypes = [C.c_uint32]
    L.vdl2gpu_stage_create.argtypes = [C.POINTER(_Config), C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]
    L.vdl2gpu_stage_destroy.argtypes = [C.c_void_p]
    L.vdl2gpu_stage_levels.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    L.vdl2gpu_launch_mix_iir_decimate.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32), C.c_void_p]
    L.vdl2gpu_launch_sync_slice.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    L.vdl2gpu_launch_burst_fec.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    L.vdl2gpu_parse_records.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, _FRAME_CB, C.c_void_p]
    L.vdl2gpu_stage_read_events.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.vdl2gpu_stage_queue_bursts.argtypes = [C.c_void_p, C.POINTER(_Burst), C.c_uint32]
    L.vdl2gpu_stage_read_counters.argtypes = [C.c_void_p, C.c_void_p]
    _LIB = L
    return L


def _check(L, rc, what):
    if rc < 0:
        raise Vdl2GpuError(f"{what}: {L.vdl2gpu_strerror(rc).decode()} ({L.vdl2gpu_last_error().decode()})")
    return rc


class Frame:
    """One AVLC frame + vdl2_msg_metadata fields (src/output-common.h:31-43)."""
    __slots__ = ("channel", "freq", "burst_seq", "idx", "data", "synd_weight", "datalen_octets",
                 "num_fec_corrections", "frame_pwr_dbfs", "nf_pwr_dbfs", "ppm_error", "frame_pwr", "mag_nf",
                 "sync_dec_index", "burst_timestamp", "fcs_ok")

    def key(self):
        return (self.channel, self.burst_seq, self.idx)

    def __repr__(self):
        return (f"Frame(ch={self.channel} burst={self.burst_seq} idx={self.idx} len={len(self.data)} "
                f"fcs_ok={self.fcs_ok} fec={self.num_fec_corrections} synd={self.synd_weight})")


def serialize_raw_frame(frame, station_id=None, timestamp=(0, 0)):
    """Frame -> one record of the reference's raw-frame archive format (see vdl2gpu_serialize_raw_frame)."""
    L = load_library()
    f = _Frame()
    buf = (C.c_uint8 * max(len(frame.data), 1)).from_buffer_copy(frame.data or b"\0")
    f.channel, f.freq, f.burst_seq, f.idx = frame.channel, frame.freq, frame.burst_seq, frame.idx
    f.data, f.len = C.cast(buf, C.POINTER(C.c_uint8)), len(frame.data)
    f.synd_weight, f.datalen_octets, f.num_fec_corrections = frame.synd_weight, frame.datalen_octets, frame.num_fec_corrections
    f.frame_pwr_dbfs, f.nf_pwr_dbfs, f.ppm_error = frame.frame_pwr_dbfs, frame.nf_pwr_dbfs, frame.ppm_error
    f.burst_timestamp.tv_sec, f.burst_timestamp.tv_usec = timestamp
    out = (C.c_uint8 * 70000)()
    n = _check(L, L.vdl2gpu_serialize_raw_frame(C.byref(f), station_id.encode() if station_id else None, out, 70000), "vdl2gpu_serialize_raw_frame")
    return bytes(out[:n])


def frame_from_c(f):
    """vdl2gpu_frame (ctypes) -> Frame"""
    o = Frame()
    o.channel, o.freq, o.burst_seq, o.idx = f.channel, f.freq, f.burst_seq, f.idx
    o.data = C.string_at(f.data, f.len) if f.len else b""
    o.synd_weight, o.datalen_octets, o.num_fec_corrections = f.synd_weight, f.datalen_octets, f.num_fec_corrections
    o.frame_pwr_dbfs, o.nf_pwr_dbfs, o.ppm_error = f.frame_pwr_dbfs, f.nf_pwr_dbfs, f.ppm_error
    o.frame_pwr, o.mag_nf = f.frame_pwr, f.mag_nf
    o.sync_dec_index = f.sync_dec_index
    o.burst_timestamp = f.burst_timestamp.tv_sec + 1e-6 * f.burst_timestamp.tv_usec
    o.fcs_ok = bool(f.fcs_ok)
    return o


def level_metrics(rec):
    """What an operator reads off one record of input_levels(): mean power in dBFS (10 log10 of the mean of c_I^2 + c_Q^2
    over full_scale^2; -inf for an all-zero input), the DC offsets of I and Q and the peak in full-scale units, and the
    fraction of samples with a component on a rail.  All None for an input that has measured nothing yet."""
    n, fs = int(rec["samples"]), int(rec["full_scale"])
    if n == 0:
        return dict(power_dbfs=None, dc_i=None, dc_q=None, clipped_fraction=None, peak=None)
    pw = int(rec["pow"]) / (n * fs * fs)
    return dict(power_dbfs=10.0 * np.log10(pw) if pw > 0 else float("-inf"), dc_i=int(rec["sum_i"]) / (n * fs),
                dc_q=int(rec["sum_q"]) / (n * fs), clipped_fraction=int(rec["clipped"]) / n, peak=int(rec["peak"]) / fs)


def channel_level_metrics(rec):
    """What an operator reads off one record of channel_levels(): samples (the sum of hist), mean in-band power in dBFS
    (10 log10 of pow / 2^48 / samples; -inf for digital silence), peak in dBFS (10 log10 of peak_pow), noise floor in dBFS
    (nf_pwr_dbfs) and bin_floor_dbfs, the lower edge of each histogram bin in dBFS (bin 0 has none: -inf).  Power and peak
    are None for a channel that has measured nothing yet."""
    n = int(np.asarray(rec["hist"], np.uint64).astype(object).sum())
    edges = np.concatenate([[-np.inf], 10.0 * np.log10(2.0) * np.arange(-36, 3, dtype=np.float64)])
    if n == 0:
        return dict(samples=0, power_dbfs=None, peak_dbfs=None, nf_dbfs=float(rec["nf_pwr_dbfs"]), bin_floor_dbfs=edges)
    pw = int(rec["pow"]) / float(1 << 48) / n
    pk = float(rec["peak_pow"])
    return dict(samples=n, power_dbfs=10.0 * np.log10(pw) if pw > 0 else float("-inf"),
                peak_dbfs=10.0 * np.log10(pk) if pk > 0 else float("-inf"), nf_dbfs=float(rec["nf_pwr_dbfs"]), bin_floor_dbfs=edges)


def spectrum_metrics(rec, centerfreq, sample_rate):
    """What an operator reads off one record of spectrum(), for an input tuned to centerfreq at sample_rate (Hz): freq_hz,
    the frequency of each bin; mean_dbfs, the mean power per bin, 10 log10(pow / 2^40 / segments / 512^2), so that a
    full-scale complex tone on a bin reads 0 dBFS (-inf for a bin that only saw silence); peak_dbfs, the peak hold on the
    same scale.  The powers are None for an input that has no complete segment yet."""
    n = SPECTRUM_BINS
    freq = float(centerfreq) + (np.arange(n, dtype=np.float64) - n // 2) * (float(sample_rate) / n)
    segs = int(rec["segments"])
    if segs == 0:
        return dict(freq_hz=freq, mean_dbfs=None, peak_dbfs=None)
    full = float(n // 2) ** 2                        # sum of the Hann window, squared
    mean = np.array([int(v) for v in rec["pow"]], dtype=np.float64) / float(1 << 40) / segs / full
    peak = np.asarray(rec["peak"], np.float64) / full
    with np.errstate(divide="ignore"):
        return dict(freq_hz=freq, mean_dbfs=10.0 * np.log10(mean), peak_dbfs=10.0 * np.log10(peak))


def make_config(sample_rate, oversample, sample_fmt, centerfreq, freqs, max_ppm=0.0, flags=0):
    """(vdl2gpu_config, the freqs array it points at) for the stage stubs"""
    fr = np.ascontiguousarray(freqs, dtype=np.uint32)
    cfg = _Config()
    cfg.sample_rate, cfg.oversample, cfg.sample_fmt, cfg.centerfreq = sample_rate, oversample, sample_fmt, centerfreq
    cfg.n_channels = int(fr.size)
    cfg.freqs = fr.ctypes.data_as(C.POINTER(C.c_uint32))
    cfg.max_ppm, cfg.flags, cfg.device = max_ppm, flags, -1
    return cfg, fr


def parse_records(region_bytes, decimated_rate):
    """host copy of a vdl2gpu_launch_burst_fec region -> [Frame]"""
    L = load_library()
    out = []
    cb = _FRAME_CB(lambda fp, _u: out.append(frame_from_c(fp.contents)))
    buf = np.frombuffer(region_bytes, np.uint8)
    _check(L, L.vdl2gpu_parse_records(buf.ctypes.data, buf.size, decimated_rate, cb, None), "vdl2gpu_parse_records")
    return out


class Vdl2Channels:
    """N VDL2 channels demodulated from one IQ stream on one H100."""

    def __init__(self, sample_rate, oversample, sample_fmt, centerfreq, freqs, max_ppm=0.0,
                 max_chunk_bytes=1 << 20, device=-1, flags=0, n_inflight=4, n_streams=1, levels=False, channel_levels=False,
                 spectrum=False):
        """n_streams > 1: independent-streams mode, channels [s*C, (s+1)*C) demodulate stream s; process_buf_* then take
        the S per-stream buffers back to back.  levels=True: measure every input's levels (input_levels());
        channel_levels=True: measure every channel's in-band levels (channel_levels()); spectrum=True: measure every
        input's power spectrum (spectrum())."""
        if levels:
            flags |= FLAG_INPUT_LEVELS
        if channel_levels:
            flags |= FLAG_CHANNEL_LEVELS
        if spectrum:
            flags |= FLAG_SPECTRUM
        self.L = load_library()
        self.n_streams = int(n_streams)
        self.freqs = np.ascontiguousarray(freqs, dtype=np.uint32)
        self.n_channels = int(self.freqs.size)
        self.sample_fmt = sample_fmt
        cfg = _Config()
        cfg.sample_rate, cfg.oversample, cfg.sample_fmt, cfg.centerfreq = sample_rate, oversample, sample_fmt, centerfreq
        cfg.n_channels = self.n_channels
        cfg.freqs = self.freqs.ctypes.data_as(C.POINTER(C.c_uint32))
        cfg.max_ppm, cfg.max_chunk_bytes, cfg.device, cfg.flags, cfg.n_inflight = max_ppm, max_chunk_bytes, device, flags, n_inflight
        cfg.n_streams = self.n_streams
        self.h = C.c_void_p()
        _check(self.L, self.L.vdl2gpu_create(C.byref(cfg), C.byref(self.h)), "vdl2gpu_create")
        self._frames = []
        self._cb = _FRAME_CB(self._on_frame)

    def close(self):
        if getattr(self, "h", None):
            self.L.vdl2gpu_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _on_frame(self, fp, _user):
        self._frames.append(frame_from_c(fp.contents))

    # ---- the reference's entry points for this path ----
    def process_buf_uchar(self, buf):
        """src/demod.c:339-347: interleaved cu8 I,Q bytes."""
        return self._submit(buf, FMT_U8)

    def process_buf_short(self, buf):
        """src/demod.c:356-365: interleaved little-endian cs16 I,Q."""
        return self._submit(buf, FMT_S16)

    def _submit(self, buf, fmt):
        if fmt != self.sample_fmt:
            raise Vdl2GpuError("sample format differs from the one the channels were created with")
        b = np.ascontiguousarray(buf).view(np.uint8).reshape(-1)
        if b.size % self.n_streams:
            raise Vdl2GpuError("buffer size is not a multiple of n_streams")
        _check(self.L, self.L.vdl2gpu_submit(self.h, b.ctypes.data, b.size // self.n_streams), "vdl2gpu_submit")

    def submit(self, buf):
        return self._submit(buf, self.sample_fmt)

    def submit_planar_s16(self, xi, xq):
        """SDRplay-style hand-off: separate int16 I and Q arrays (src/sdrplay.c:72-134)."""
        xi = np.ascontiguousarray(xi, dtype=np.int16); xq = np.ascontiguousarray(xq, dtype=np.int16)
        assert xi.size == xq.size
        _check(self.L, self.L.vdl2gpu_submit_planar_s16(self.h, xi.ctypes.data, xq.ctypes.data, xi.size), "vdl2gpu_submit_planar_s16")

    def submit_device(self, dev_ptr, nbytes, producer_stream=0):
        _check(self.L, self.L.vdl2gpu_submit_device(self.h, C.c_void_p(dev_ptr), nbytes, C.c_void_p(producer_stream)), "vdl2gpu_submit_device")

    def wait_input_consumed(self, stream=0):
        _check(self.L, self.L.vdl2gpu_wait_input_consumed(self.h, C.c_void_p(stream)), "vdl2gpu_wait_input_consumed")

    def stream_wait(self, stream=0):
        _check(self.L, self.L.vdl2gpu_stream_wait(self.h, C.c_void_p(stream)), "vdl2gpu_stream_wait")

    def process_chunked(self, buf, chunk_bytes):
        b = np.ascontiguousarray(buf).view(np.uint8).reshape(-1)
        for off in range(0, b.size, chunk_bytes):
            self._submit(b[off:off + chunk_bytes], self.sample_fmt)

    def poll(self):
        """Frames of the chunks finished so far (non-blocking)."""
        _check(self.L, self.L.vdl2gpu_poll(self.h, self._cb, None), "vdl2gpu_poll")
        out, self._frames = self._frames, []
        return out

    def flush(self):
        """Block until everything submitted is processed; returns the frames."""
        _check(self.L, self.L.vdl2gpu_flush(self.h, self._cb, None), "vdl2gpu_flush")
        out, self._frames = self._frames, []
        return out

    def poll_count(self):
        """Like poll() but only counts frames (no Python object per frame)."""
        return _check(self.L, self.L.vdl2gpu_poll(self.h, C.cast(None, _FRAME_CB), None), "vdl2gpu_poll")

    def flush_count(self):
        """Like flush() but only counts frames (no Python object per frame)."""
        return _check(self.L, self.L.vdl2gpu_flush(self.h, C.cast(None, _FRAME_CB), None), "vdl2gpu_flush")

    # ---- introspection ----
    def stats(self):
        s = _Stats()
        _check(self.L, self.L.vdl2gpu_get_stats(self.h, C.byref(s)), "vdl2gpu_get_stats")
        return {n: getattr(s, n) for n, _ in _Stats._fields_ if n != "reserved"}

    def channel_counters(self):
        a = np.zeros((self.n_channels, NUM_COUNTERS), np.uint64)
        _check(self.L, self.L.vdl2gpu_get_channel_counters(self.h, a.ctypes.data, self.n_channels), "vdl2gpu_get_channel_counters")
        return a

    def tables(self):
        t = dict(levels=np.zeros(256, np.float32), sin_lut=np.zeros(257, np.float32), cos_lut=np.zeros(257, np.float32),
                 A=np.zeros(3, np.float32), B=np.zeros(3, np.float32), lr_X=np.zeros(16, np.float32),
                 lr_denom=np.zeros(1, np.float32), pr_phase=np.zeros(16, np.float32))
        _check(self.L, self.L.vdl2gpu_get_tables(self.h, *[t[k].ctypes.data for k in
               ("levels", "sin_lut", "cos_lut", "A", "B", "lr_X", "lr_denom", "pr_phase")]), "vdl2gpu_get_tables")
        return t

    def read_dec(self, max_dec):
        out = np.zeros((max_dec, self.n_channels, 2), np.float32)
        n = C.c_uint32(0)
        _check(self.L, self.L.vdl2gpu_read_dec(self.h, out.ctypes.data, out.size, C.byref(n)), "vdl2gpu_read_dec")
        return out[:n.value]

    def read_events(self, cap=1 << 16):
        ev = (_Event * cap)()
        n = _check(self.L, self.L.vdl2gpu_read_events(self.h, C.cast(ev, C.c_void_p), cap), "vdl2gpu_read_events")
        return [dict(channel=ev[k].channel, kind=ev[k].kind, dec_index=ev[k].dec_index, i=list(ev[k].i),
                     f=np.array(list(ev[k].f), np.float32)) for k in range(n)]

    def enable_timing(self, on=True):
        _check(self.L, self.L.vdl2gpu_enable_timing(self.h, 1 if on else 0), "vdl2gpu_enable_timing")

    def timeline(self, cap=4096):
        """rows of [chunk, front start, K1 end, K2a start, K2a end, K2 start, K2|K3, K3 end] (ms) for the timed chunks"""
        a = np.zeros((cap, 8), np.float32)
        n = _check(self.L, self.L.vdl2gpu_get_timeline(self.h, a.ctypes.data, cap), "vdl2gpu_get_timeline")
        return a[:n]

    def block_trace(self, cap=1 << 16):
        """rows of [kernel, block, smid, 0, start_ns, end_ns] (needs VDL2GPU_BLOCK_TRACE=1 when the object was created)"""
        a = np.zeros((cap, 6), np.uint64)
        n = _check(self.L, self.L.vdl2gpu_debug_block_trace(self.h, a.ctypes.data, cap), "vdl2gpu_debug_block_trace")
        return a[:n]

    def input_levels(self):
        """one dict per input (the stream; the n_streams streams; the receivers, in order) of the exact integers the device
        measured over every sample submitted so far: samples, sum_i, sum_q, pow (the 128-bit sum of c_I^2 + c_Q^2 as a
        Python int), clipped, peak, full_scale (see vdl2gpu_get_input_levels; level_metrics() turns one into dBFS and
        full-scale units).  Needs levels=True at creation."""
        n = self.n_streams
        out = (_InputLevels * max(n, 1))()
        _check(self.L, self.L.vdl2gpu_get_input_levels(self.h, out, n), "vdl2gpu_get_input_levels")
        return [dict(samples=o.samples, sum_i=o.sum_i, sum_q=o.sum_q, pow=(o.pow_hi << 64) | o.pow_lo, clipped=o.clipped,
                     peak=o.peak, full_scale=o.full_scale) for o in out[:n]]

    def channel_levels(self):
        """one dict per channel of what the device measured over every decimated sample submitted so far: hist (uint64
        array of 40 bins by octave of the sample power p), pow (the 128-bit sum of p x 2^48, truncated per sample, as a
        Python int), peak_pow, mag_lp, mag_nf and nf_pwr_dbfs (see vdl2gpu_get_channel_levels; channel_level_metrics()
        turns one into dBFS).  Needs channel_levels=True at creation."""
        n = self.n_channels
        out = (_ChannelLevels * max(n, 1))()
        _check(self.L, self.L.vdl2gpu_get_channel_levels(self.h, out, n), "vdl2gpu_get_channel_levels")
        return [dict(hist=np.array(o.hist[:], np.uint64), pow=(o.pow_hi << 64) | o.pow_lo, peak_pow=np.float32(o.peak_pow),
                     mag_lp=np.float32(o.mag_lp), mag_nf=np.float32(o.mag_nf), nf_pwr_dbfs=np.float32(o.nf_pwr_dbfs)) for o in out[:n]]

    def spectrum(self, first=0, n=None):
        """one dict per input first .. first + n - 1 (default: to the last input; inputs as for input_levels()) of what the
        device measured over every complete 1024-sample segment so far: segments, pending (samples of the incomplete segment
        held), pow (object array of 1024 Python ints, the 128-bit sums of p x 2^40 per bin) and peak (float32 array of the
        largest p per bin).  Bin k is centre + (k - 512) fs / 1024 (see vdl2gpu_get_spectrum; spectrum_metrics() turns one
        into Hz and dBFS).  Needs spectrum=True at creation."""
        if n is None:
            n = max(self.n_streams - first, 0)
        out = (_Spectrum * max(n, 1))()
        _check(self.L, self.L.vdl2gpu_get_spectrum(self.h, first, n, out), "vdl2gpu_get_spectrum")
        recs = []
        for o in out[:n]:
            lo = np.ctypeslib.as_array(o.pow_lo).astype(object)
            hi = np.ctypeslib.as_array(o.pow_hi).astype(object)
            recs.append(dict(segments=o.segments, pending=o.pending, pow=(hi << 64) | lo,
                             peak=np.ctypeslib.as_array(o.peak).astype(np.float32).copy()))
        return recs

    def kernel_ms(self):
        ms = (C.c_double * 5)()
        n = (C.c_uint64 * 5)()
        _check(self.L, self.L.vdl2gpu_get_kernel_ms(self.h, ms, n), "vdl2gpu_get_kernel_ms")
        return dict(K0=(ms[0], n[0]), K1=(ms[1], n[1]), K2a=(ms[2], n[2]), K2=(ms[3], n[3]), K3=(ms[4], n[4]))


class Vdl2Receivers(Vdl2Channels):
    """R receivers on one H100, each with its own centre frequency and its own channels; every receiver decodes exactly
    as one reference process tuned to its centre would.  Channel numbers are global: receiver r owns channels
    channels_of(r).  The receivers advance in lock step: submit() takes one equal-length buffer per receiver."""

    def __init__(self, sample_rate, oversample, sample_fmt, receivers, max_ppm=0.0, max_chunk_bytes=1 << 20, device=-1,
                 flags=0, n_inflight=4, levels=False, channel_levels=False, spectrum=False):
        """receivers: list of (centerfreq, [channel freqs...]); levels=True: measure every receiver's input levels;
        channel_levels=True: every channel's in-band levels; spectrum=True: every receiver's power spectrum"""
        if levels:
            flags |= FLAG_INPUT_LEVELS
        if channel_levels:
            flags |= FLAG_CHANNEL_LEVELS
        if spectrum:
            flags |= FLAG_SPECTRUM
        self.L = load_library()
        self.receivers = [(int(cf), [int(f) for f in fr]) for cf, fr in receivers]
        self.n_receivers = self.n_streams = len(self.receivers)
        self.freqs = np.ascontiguousarray([f for _, fr in self.receivers for f in fr], dtype=np.uint32)
        self.n_channels = int(self.freqs.size)
        self._first = np.concatenate([[0], np.cumsum([len(fr) for _, fr in self.receivers], dtype=np.int64)]).astype(np.int64)
        self.sample_fmt = sample_fmt
        rx = (_Receiver * max(self.n_receivers, 1))()
        for r, (cf, fr) in enumerate(self.receivers):
            rx[r].centerfreq, rx[r].n_channels = cf, len(fr)
        cfg = _Config()
        cfg.sample_rate, cfg.oversample, cfg.sample_fmt = sample_rate, oversample, sample_fmt
        cfg.n_channels = self.n_channels
        cfg.freqs = self.freqs.ctypes.data_as(C.POINTER(C.c_uint32))
        cfg.max_ppm, cfg.max_chunk_bytes, cfg.device, cfg.flags, cfg.n_inflight = max_ppm, max_chunk_bytes, device, flags, n_inflight
        cfg.n_streams = self.n_receivers
        self.h = C.c_void_p()
        _check(self.L, self.L.vdl2gpu_create_receivers(C.byref(cfg), rx, self.n_receivers, C.byref(self.h)), "vdl2gpu_create_receivers")
        self._frames = []
        self._cb = _FRAME_CB(self._on_frame)

    def channels_of(self, r):
        """global channel numbers of receiver r"""
        return range(int(self._first[r]), int(self._first[r + 1]))

    def receiver_of(self, channel):
        if not 0 <= channel < self.n_channels:
            raise IndexError(f"channel {channel} out of range")
        return int(np.searchsorted(self._first, channel, side="right")) - 1

    def submit(self, bufs):
        """one buffer per receiver, all of the same length in bytes"""
        if len(bufs) != self.n_receivers:
            raise Vdl2GpuError(f"{len(bufs)} buffers for {self.n_receivers} receivers")
        parts = [np.ascontiguousarray(b).view(np.uint8).reshape(-1) for b in bufs]
        if any(p.size != parts[0].size for p in parts):
            raise Vdl2GpuError("the receivers' buffers differ in length")
        return self._submit(np.concatenate(parts), self.sample_fmt)

    def process_chunked(self, bufs, chunk_bytes):
        """each receiver's whole stream (equal lengths), submitted chunk_bytes per receiver at a time"""
        parts = [np.ascontiguousarray(b).view(np.uint8).reshape(-1) for b in bufs]
        for off in range(0, parts[0].size, chunk_bytes):
            self.submit([p[off:off + chunk_bytes] for p in parts])


class Vdl2MixedReceivers(Vdl2Receivers):
    """Receivers of different sample rates and sample formats on one H100 (e.g. RTL-SDR dongles, cu8 at 1.05 Msps, next to
    SDRplay devices, cs16 at 2.1 Msps); every receiver decodes exactly as one reference process at its own rate, tuned to
    its own centre, would.  The receivers advance in lock step in decimated samples (105000 per second for every rate):
    submit_span() takes one buffer per receiver, receiver r's holding n_dec x oversample_r complex samples in its own
    format.  Listing the receivers grouped by rate keeps every K1 warp on one rate (faster than interleaved rates).

    With ragged=True the receivers do not advance in lock step: submit_ragged() takes whatever whole decimation groups each
    receiver has (any count, 0 included, per receiver and per span), and every receiver still decodes exactly what one
    reference process decodes from the concatenation of its buffers.  push() queues any length of one receiver's bytes
    inside the library (one call per device callback, from that device's own thread) and submit_pushed() turns what is
    queued into spans.  restart_receiver() starts one receiver afresh (a
    reconnect, a swapped device, a retune) without disturbing the others, and update_receivers() / add_receivers() /
    remove_receivers() let receivers join and leave (after flush()) while the others carry on."""

    def __init__(self, receivers, max_ppm=0.0, max_chunk_bytes=1 << 20, device=-1, flags=0, n_inflight=4, ragged=False,
                 levels=False, channel_levels=False, spectrum=False):
        """receivers: list of (centerfreq, [channel freqs...], oversample (10, 13 or 20), fmt (FMT_U8 or FMT_S16));
        levels=True: measure every receiver's input levels (input_levels()); channel_levels=True: every channel's in-band
        levels (channel_levels()); spectrum=True: every receiver's power spectrum (spectrum())"""
        if ragged:
            flags |= FLAG_RAGGED
        if levels:
            flags |= FLAG_INPUT_LEVELS
        if channel_levels:
            flags |= FLAG_CHANNEL_LEVELS
        if spectrum:
            flags |= FLAG_SPECTRUM
        self.ragged = bool(flags & FLAG_RAGGED)
        self.L = load_library()
        rxs = self._normalise(receivers)
        self._describe(rxs)
        self.sample_fmt = None
        rx = self._c_receivers(rxs)
        cfg = _Config()                              # sample_rate, oversample, sample_fmt and centerfreq stay 0: per receiver
        cfg.n_channels = self.n_channels
        cfg.freqs = self.freqs.ctypes.data_as(C.POINTER(C.c_uint32))
        cfg.max_ppm, cfg.max_chunk_bytes, cfg.device, cfg.flags, cfg.n_inflight = max_ppm, max_chunk_bytes, device, flags, n_inflight
        cfg.n_streams = self.n_receivers
        self.h = C.c_void_p()
        _check(self.L, self.L.vdl2gpu_create_mixed_receivers(C.byref(cfg), rx, self.n_receivers, C.byref(self.h)),
               "vdl2gpu_create_mixed_receivers")
        self._frames = []
        self._cb = _FRAME_CB(self._on_frame)

    @staticmethod
    def _normalise(receivers):
        return [(int(cf), [int(f) for f in fr], int(os_), int(fmt)) for cf, fr, os_, fmt in receivers]

    def _describe(self, rxs):
        """the per-receiver attributes of the list rxs of (centre, [freqs], oversample, format)"""
        self.receivers = [(cf, fr) for cf, fr, _, _ in rxs]
        self.oversample = [os_ for _, _, os_, _ in rxs]
        self.formats = [fmt for _, _, _, fmt in rxs]
        self.bytes_per_dec = [os_ * (4 if fmt == FMT_S16 else 2) for _, _, os_, fmt in rxs]
        self.n_receivers = self.n_streams = len(rxs)
        self.freqs = np.ascontiguousarray([f for _, fr in self.receivers for f in fr], dtype=np.uint32)
        self.n_channels = int(self.freqs.size)
        self._first = np.concatenate([[0], np.cumsum([len(fr) for _, fr in self.receivers], dtype=np.int64)]).astype(np.int64)

    @staticmethod
    def _c_receivers(rxs):
        rx = (_ReceiverEx * max(len(rxs), 1))()
        for r, (cf, fr, os_, fmt) in enumerate(rxs):
            rx[r].centerfreq, rx[r].n_channels, rx[r].oversample, rx[r].sample_fmt = cf, len(fr), os_, fmt
        return rx

    def _submit(self, buf, fmt):
        raise Vdl2GpuError("a mixed-receivers context takes spans of decimated samples: use submit_span / submit_span_device")

    def submit(self, bufs):
        return self._submit(bufs, None)

    def submit_device(self, dev_ptr, nbytes, producer_stream=0):
        return self._submit(None, None)

    def submit_span(self, bufs):
        """one buffer per receiver; receiver r's holds n_dec x oversample_r complex samples in its own format"""
        if len(bufs) != self.n_receivers:
            raise Vdl2GpuError(f"{len(bufs)} buffers for {self.n_receivers} receivers")
        parts = [np.ascontiguousarray(b).view(np.uint8).reshape(-1) for b in bufs]
        n_dec = parts[0].size // self.bytes_per_dec[0]
        for r, p in enumerate(parts):
            if p.size != n_dec * self.bytes_per_dec[r]:
                raise Vdl2GpuError(f"receiver {r}: {p.size} bytes, not {n_dec} decimated samples x {self.bytes_per_dec[r]} bytes")
        buf = np.concatenate(parts)
        _check(self.L, self.L.vdl2gpu_submit_span(self.h, buf.ctypes.data, n_dec), "vdl2gpu_submit_span")

    def submit_span_device(self, dev_ptr, n_dec, producer_stream=0):
        """the receivers' buffers back to back in device memory (receiver 0 first), n_dec decimated samples each"""
        _check(self.L, self.L.vdl2gpu_submit_span_device(self.h, C.c_void_p(dev_ptr), n_dec, C.c_void_p(producer_stream)),
               "vdl2gpu_submit_span_device")

    def process_chunked(self, bufs, n_dec):
        """each receiver's whole stream (the same duration for all), submitted n_dec decimated samples at a time; the last
        span may be shorter"""
        parts = [np.ascontiguousarray(b).view(np.uint8).reshape(-1) for b in bufs]
        total = parts[0].size // self.bytes_per_dec[0]
        for d0 in range(0, total, n_dec):
            d1 = min(total, d0 + n_dec)
            self.submit_span([p[d0 * w:d1 * w] for p, w in zip(parts, self.bytes_per_dec)])

    # ---- ragged spans (ragged=True) ----
    def submit_ragged(self, bufs):
        """one uint8 buffer per receiver, each a whole number of decimation groups (oversample_r complex samples in the
        receiver's format; an empty buffer is allowed): receiver r brings len(bufs[r]) / bytes_per_dec[r] decimated samples"""
        if len(bufs) != self.n_receivers:
            raise ValueError(f"{len(bufs)} buffers for {self.n_receivers} receivers")
        parts = [np.ascontiguousarray(b).view(np.uint8).reshape(-1) for b in bufs]
        for r, p in enumerate(parts):
            if p.size % self.bytes_per_dec[r]:
                raise ValueError(f"receiver {r}: {p.size} bytes is not a whole number of decimation groups of {self.bytes_per_dec[r]} bytes")
        counts = np.array([p.size // w for p, w in zip(parts, self.bytes_per_dec)], np.uint32)
        buf = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
        _check(self.L, self.L.vdl2gpu_submit_ragged(self.h, buf.ctypes.data if buf.size else None, counts.ctypes.data), "vdl2gpu_submit_ragged")

    def submit_ragged_device(self, dev_ptr, counts, producer_stream=0):
        """the receivers' buffers back to back in device memory (receiver 0 first), counts[r] decimated samples of receiver r"""
        n = np.ascontiguousarray(counts, np.uint32)
        if n.size != self.n_receivers:
            raise ValueError(f"{n.size} counts for {self.n_receivers} receivers")
        _check(self.L, self.L.vdl2gpu_submit_ragged_device(self.h, C.c_void_p(dev_ptr), n.ctypes.data, C.c_void_p(producer_stream)),
               "vdl2gpu_submit_ragged_device")

    def push(self, r, buf):
        """queue receiver r's next bytes (any length up to max_chunk_bytes, in its own format; may split a decimation group
        or a sample); blocks while the receiver's ring lacks room.  The GIL is released during the call, so one Python
        thread per receiver pushes concurrently."""
        b = np.ascontiguousarray(buf).view(np.uint8).reshape(-1)
        if b.size > 0xFFFFFFFF:                      # the C length is 32 bits: refuse rather than push size mod 2^32
            raise Vdl2GpuError(f"vdl2gpu_push: {b.size} bytes, more than max_chunk_bytes")
        _check(self.L, self.L.vdl2gpu_push(self.h, int(r), b.ctypes.data if b.size else None, b.size), "vdl2gpu_push")

    def submit_pushed(self):
        """submit spans of the whole decimation groups queued when the call starts (bytes pushed during the call wait for the
        next one); returns the number of spans"""
        return _check(self.L, self.L.vdl2gpu_submit_pushed(self.h), "vdl2gpu_submit_pushed")

    def receiver_positions(self):
        """decimated samples accepted so far per receiver (uint64[n_receivers])"""
        out = np.zeros(self.n_receivers, np.uint64)
        _check(self.L, self.L.vdl2gpu_get_receiver_positions(self.h, out.ctypes.data, self.n_receivers), "vdl2gpu_get_receiver_positions")
        return out

    def restart_receiver(self, r, centerfreq=None, freqs=None):
        """restart receiver r at the start of the next span that runs, as a freshly started reference process tuned to
        centerfreq (None: its centre) and freqs (None: its channel frequencies; otherwise one per channel of the receiver);
        every other receiver keeps its state.  receivers / freqs follow the new tuning."""
        r = int(r)
        if not 0 <= r < self.n_receivers:
            raise ValueError(f"receiver {r} of {self.n_receivers}")
        cf_old, fr_old = self.receivers[r]
        fr = None
        if freqs is not None:
            fr = np.ascontiguousarray([int(f) for f in freqs], np.uint32)
            if fr.size != len(fr_old):
                raise ValueError(f"receiver {r} has {len(fr_old)} channels, {fr.size} frequencies given")
        cf = 0 if centerfreq is None else int(centerfreq)
        _check(self.L, self.L.vdl2gpu_restart_receiver(self.h, r, cf, fr.ctypes.data if fr is not None else None),
               "vdl2gpu_restart_receiver")
        new_fr = [int(f) for f in fr] if fr is not None else fr_old
        self.receivers[r] = (cf if cf else cf_old, new_fr)
        self.freqs[self._first[r]:self._first[r + 1]] = new_fr

    def process_ragged(self, bufs, counts_per_span):
        """each receiver's whole stream, cut into ragged spans: span k brings counts_per_span[k][r] decimated samples of
        receiver r (a count past the end of that receiver's stream brings what is left)"""
        parts = [np.ascontiguousarray(b).view(np.uint8).reshape(-1) for b in bufs]
        pos = [0] * len(parts)
        for counts in counts_per_span:
            span = []
            for r, (p, w) in enumerate(zip(parts, self.bytes_per_dec)):
                n = min(int(counts[r]), p.size // w - pos[r])
                span.append(p[pos[r] * w:(pos[r] + n) * w])
                pos[r] += n
            self.submit_ragged(span)

    # ---- receivers joining and leaving (ragged=True) ----
    def update_receivers(self, receivers, from_):
        """Replace the receiver list with `receivers` [(centerfreq, [freqs...], oversample, fmt), ...] on a drained context
        (flush() first).  from_[i] is the current index of the receiver entry i continues, which it must describe exactly
        as it is now (receivers[k], oversample[k], formats[k]), or -1 for a new receiver; receivers not named are removed.
        Kept receivers carry on undisturbed under their new indices and channel numbers; a new one starts as a freshly
        started reference process.  Read a receiver's counters before removing it."""
        rxs = self._normalise(receivers)
        src = [int(k) for k in from_]
        if len(src) != len(rxs):
            raise ValueError(f"{len(src)} entries in from_ for {len(rxs)} receivers")
        if not rxs:
            raise ValueError("no receivers")
        seen = set()
        for i, k in enumerate(src):
            if k == -1:
                continue
            if not 0 <= k < self.n_receivers:
                raise ValueError(f"entry {i} continues receiver {k} of {self.n_receivers}")
            if k in seen:
                raise ValueError(f"entry {i} continues receiver {k}, which an earlier entry continues")
            seen.add(k)
            cf, fr = self.receivers[k]
            if rxs[i] != (cf, list(fr), self.oversample[k], self.formats[k]):
                raise ValueError(f"entry {i} does not repeat receiver {k}'s description (retune with restart_receiver)")
        rx = self._c_receivers(rxs)
        fr = np.ascontiguousarray([f for _, fl, _, _ in rxs for f in fl], dtype=np.uint32)
        fa = np.ascontiguousarray(src, dtype=np.int32)
        _check(self.L, self.L.vdl2gpu_update_receivers(self.h, rx, fa.ctypes.data, len(rxs), fr.ctypes.data), "vdl2gpu_update_receivers")
        self._describe(rxs)

    def _current(self, k):
        cf, fr = self.receivers[k]
        return (cf, list(fr), self.oversample[k], self.formats[k])

    def add_receivers(self, receivers, at=None):
        """insert new receivers before index `at` (None: at the end); every receiver from `at` on moves up"""
        new = self._normalise(receivers)
        at = self.n_receivers if at is None else int(at)
        if not 0 <= at <= self.n_receivers:
            raise ValueError(f"position {at} of {self.n_receivers} receivers")
        old = list(range(self.n_receivers))
        self.update_receivers([self._current(k) for k in old[:at]] + new + [self._current(k) for k in old[at:]],
                              old[:at] + [-1] * len(new) + old[at:])

    def remove_receivers(self, indices):
        """remove the receivers at these indices; the others keep their order and move down"""
        gone = set()
        for k in indices:
            k = int(k)
            if not 0 <= k < self.n_receivers:
                raise ValueError(f"receiver {k} of {self.n_receivers}")
            gone.add(k)
        keep = [k for k in range(self.n_receivers) if k not in gone]
        self.update_receivers([self._current(k) for k in keep], keep)
