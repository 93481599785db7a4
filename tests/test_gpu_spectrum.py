"""-m gpu: spectrum (VDL2GPU_FLAG_SPECTRUM) measured by k_spectrum.  Every input's figures (segments, pending, both
128-bit halves of every bin's sum and the peak bits) must equal, bit for bit, the host build of the same vdl2_core.cuh
arithmetic (tests/spectrum_sim.py) over the floats K0 made of the samples that entered the pipeline: through host, planar
and device submits, n_streams and one-stream-per-channel contexts (balanced slot mapping included), lock-step, mixed and
ragged receivers, pushed input, restarts and receivers joining and leaving, graphs, trace and n_inflight.  Frames,
counters, events, stats and both levels must not change with the flag, and a tone and VDL2 bursts must show where they
are on the air."""
import threading
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth
from tests import spectrum_sim as ss

pytestmark = pytest.mark.gpu
EINVAL = -1
CENTRE = 136975000
N = ss.N


def _bpp(fmt):
    return 4 if fmt == vd.FMT_S16 else 2


def _gb(os_, fmt):
    return os_ * _bpp(fmt)


def _raw(rng, n_bytes, fmt):
    if fmt == vd.FMT_U8:
        return np.clip(np.round(131 + 45 * rng.standard_normal(n_bytes)), 0, 255).astype(np.uint8)
    v = np.clip(np.round(-200 + 11000 * rng.standard_normal(n_bytes // 2)), -32768, 32767).astype("<i2")
    return v.view(np.uint8)


def _floats(raw, fmt):
    """the floats K0 makes of a byte stream (a trailing partial sample is not a sample)"""
    b = np.ascontiguousarray(raw).view(np.uint8).reshape(-1)
    bpp = _bpp(fmt)
    b = b[:b.size // bpp * bpp]
    return ss.cu8_floats(b) if fmt == vd.FMT_U8 else ss.cs16_floats(b)


def _ref(pieces, fmt, restarts=None):
    """the host restatement over an input's pieces, each a chunk or span"""
    xs = [_floats(p, fmt) for p in pieces]
    x = np.concatenate(xs) if xs else np.zeros((0, 2), np.float32)
    return ss.stream(x, [a.shape[0] for a in xs], restarts)


def _check(g, refs, what="", batch=256):
    for first in range(0, len(refs), batch):
        got = g.spectrum(first, min(batch, len(refs) - first))
        for k, rec in enumerate(got):
            ss.check_equal(rec, refs[first + k], f"{what} input {first + k}")


@pytest.mark.parametrize("os_,fmt", [(10, vd.FMT_U8), (20, vd.FMT_S16)], ids=["cu8_os10", "cs16_os20"])
def test_fan_out_host_planar_and_device_submits(os_, fmt):
    import torch
    rng = np.random.default_rng(os_)
    g = vd.Vdl2Channels(105000 * os_, os_, fmt, CENTRE, [CENTRE - 50000, CENTRE, CENTRE + 75000], max_chunk_bytes=1 << 18, spectrum=True)
    rec = g.spectrum()[0]
    assert rec["segments"] == 0 and rec["pending"] == 0 and not any(rec["pow"])
    pieces = [_raw(rng, n, fmt) for n in (1 << 18, 40001, 1 << 18, 1234, 99999, 77777, 4097)]   # not multiples of 1024 samples
    for p in pieces:
        g.submit(p)
    if fmt == vd.FMT_S16:                                  # planar cs16
        for n in (60000, 3331):
            v = _raw(rng, 4 * n, fmt).view("<i2")
            g.submit_planar_s16(v[0::2].copy(), v[1::2].copy())
            pieces.append(v.view(np.uint8))
    st = torch.cuda.current_stream()
    keep = []
    for n in (1 << 17, 50004):
        p = _raw(rng, n, fmt)
        d = torch.from_numpy(p).cuda()
        keep.append(d)
        g.submit_device(d.data_ptr(), n, st.cuda_stream)
        pieces.append(p)
    g.flush()
    _check(g, [_ref(pieces, fmt)], "fan-out")
    g.close()


def test_n_streams_32_channels_each():
    rng = np.random.default_rng(2)
    S = 3
    g = vd.Vdl2Channels(1050000, 10, vd.FMT_U8, CENTRE, [CENTRE - 480000 + 10000 * k for k in range(S * 32)],
                        max_chunk_bytes=1 << 16, n_streams=S, spectrum=True)
    streams = [[] for _ in range(S)]
    for n in (1 << 16, 30001, 4096, 777):
        bufs = [_raw(rng, n, vd.FMT_U8) for _ in range(S)]
        g.submit(np.concatenate(bufs))
        for s in range(S):
            streams[s].append(bufs[s])
    g.flush()
    _check(g, [_ref(p, vd.FMT_U8) for p in streams], "n_streams")
    g.close()


@pytest.mark.parametrize("S", [40, 8704], ids=["plain", "balanced"])
def test_one_stream_per_channel(S):
    # 8704 one-channel streams fill more than half of an H100's sub-partitions: the balanced slot mapping puts them in the
    # columns of the time-major plane out of order
    rng = np.random.default_rng(S)
    g = vd.Vdl2Channels(1050000, 10, vd.FMT_U8, CENTRE, [CENTRE - 400000 + 50 * k for k in range(S)],
                        max_chunk_bytes=4096, n_streams=S, spectrum=True)
    streams = [[] for _ in range(S)]
    for n in (4096, 2047, 3000, 4096):
        bufs = rng.integers(0, 256, (S, n)).astype(np.uint8)
        g.submit(bufs.reshape(-1))
        for s in range(S):
            streams[s].append(bufs[s])
    g.flush()
    _check(g, [_ref(p, vd.FMT_U8) for p in streams], f"{S} streams")
    g.close()


def test_lock_step_receivers():
    rng = np.random.default_rng(7)
    os_, fmt = 13, vd.FMT_U8
    rx = [(CENTRE + 300000 * r, [CENTRE + 300000 * r - 200000 + 10000 * k for k in range(n)]) for r, n in enumerate((3, 1, 40, 2))]
    g = vd.Vdl2Receivers(105000 * os_, os_, fmt, rx, max_chunk_bytes=1 << 17, spectrum=True)
    pieces = [[] for _ in rx]
    for n in (1 << 17, 65536 + 4 * 13, 4 * 13 * 7):
        bufs = [_raw(rng, n, fmt) for _ in rx]
        g.submit(bufs)
        for r in range(len(rx)):
            pieces[r].append(bufs[r])
    g.flush()
    _check(g, [_ref(p, fmt) for p in pieces], "lock step")
    g.close()


KINDS = [(10, vd.FMT_U8), (13, vd.FMT_U8), (20, vd.FMT_S16)]
GROUPED = [KINDS[0]] * 2 + [KINDS[1]] * 2 + [KINDS[2]] * 2
INTERLEAVED = KINDS * 2


def _mixed(mix, flags=0, ragged=True, n_inflight=4, spectrum=True, **kw):
    rx = [(CENTRE + 200000 * r, [CENTRE + 200000 * r + 25000], os_, fmt) for r, (os_, fmt) in enumerate(mix)]
    return vd.Vdl2MixedReceivers(rx, max_chunk_bytes=3001 * 80, flags=flags, ragged=ragged, n_inflight=n_inflight, spectrum=spectrum, **kw)


@pytest.mark.parametrize("mix", [GROUPED, INTERLEAVED], ids=["grouped", "interleaved"])
def test_mixed_receivers_in_lock_step(mix):
    rng = np.random.default_rng(5)
    g = _mixed(mix, ragged=False)
    pieces = [[] for _ in mix]
    for n_dec in (3001, 1, 2999, 7, 3001, 13):
        bufs = [_raw(rng, n_dec * _gb(*m), m[1]) for m in mix]
        g.submit_span(bufs)
        for r in range(len(mix)):
            pieces[r].append(bufs[r])
    g.flush()
    _check(g, [_ref(p, m[1]) for p, m in zip(pieces, mix)], "mixed")
    g.close()


def _ragged_spans(rng, n_rx, n_spans=12):
    spans = []
    for k in range(n_spans):
        c = [int(x) for x in rng.integers(0, 3002, n_rx)]
        c[k % n_rx] = 0
        c[(k + 2) % n_rx] = 1                              # one-group counts
        if k % 2:
            c[(k + 1) % n_rx] = 3001
        if k == 0:
            c = [3001] * n_rx                              # the graphs are kept for the first span's width
        if k in (4, 5):
            c = [0] * n_rx
        spans.append(c)
    return spans


def _ragged_run(mix, streams, spans, flags=0, n_inflight=4, **kw):
    g = _mixed(mix, flags=flags, n_inflight=n_inflight, **kw)
    pos = [0] * len(mix)
    pieces = [[] for _ in mix]
    for c in spans:
        bufs = [s[p * _gb(*m):(p + n) * _gb(*m)] for s, p, n, m in zip(streams, pos, c, mix)]
        g.submit_ragged(bufs)
        for r, b in enumerate(bufs):
            pieces[r].append(b)
        pos = [p + n for p, n in zip(pos, c)]
    return g, pieces


@pytest.mark.parametrize("flags,n_inflight", [(0, 4), (vd.FLAG_NO_GRAPH, 4), (vd.FLAG_TRACE, 4), (0, 1), (vd.FLAG_TRACE, 1)],
                         ids=["graphs", "no_graph", "trace", "inflight1", "trace_inflight1"])
def test_ragged_spans_with_zero_and_one_group_counts(flags, n_inflight):
    rng = np.random.default_rng(9)
    mix = INTERLEAVED
    streams = [_raw(rng, 40000 * _gb(*m), m[1]) for m in mix]
    g, pieces = _ragged_run(mix, streams, _ragged_spans(rng, len(mix)), flags, n_inflight)
    g.flush()
    _check(g, [_ref(p, m[1]) for p, m in zip(pieces, mix)], f"ragged flags {flags} inflight {n_inflight}")
    g.close()


def test_the_same_stream_cut_two_ways_gives_equal_figures():
    rng = np.random.default_rng(10)
    mix = GROUPED
    streams = [_raw(rng, 30000 * _gb(*m), m[1]) for m in mix]
    g1, _ = _ragged_run(mix, streams, [[3000] * len(mix)] * 10)
    g2, _ = _ragged_run(mix, streams, [[1023] * len(mix)] * 29 + [[333] * len(mix)])
    g1.flush(); g2.flush()
    a, b = g1.spectrum(), g2.spectrum()
    for r in range(len(mix)):
        assert a[r]["segments"] == b[r]["segments"] and a[r]["pending"] == b[r]["pending"]
        assert np.array_equal(a[r]["pow"], b[r]["pow"]) and np.array_equal(a[r]["peak"].view(np.uint32), b[r]["peak"].view(np.uint32))
    g1.close(); g2.close()


def test_pushes_of_random_lengths_from_one_thread_per_receiver():
    rng = np.random.default_rng(21)
    mix = INTERLEAVED
    g = _mixed(mix)
    streams = [_raw(rng, 30000 * _gb(*m) + 3, m[1]) for m in mix]

    def feed(r):
        s, off, prng = streams[r], 0, np.random.default_rng(100 + r)
        while off < s.size:
            n = int(prng.integers(1, 20000))
            g.push(r, s[off:off + n])
            off += n
    th = [threading.Thread(target=feed, args=(r,)) for r in range(len(mix))]
    for t in th:
        t.start()
    while any(t.is_alive() for t in th):
        g.submit_pushed()
        g.poll()
    for t in th:
        t.join()
    g.submit_pushed()
    g.flush()
    pos = g.receiver_positions().tolist()
    _check(g, [_ref([s[:p * _gb(*m)]], m[1]) for s, p, m in zip(streams, pos, mix)], "pushed")
    g.close()


@pytest.mark.parametrize("retune", [False, True], ids=["restart", "retune"])
def test_restart_mid_segment_starts_a_new_grid(retune):
    rng = np.random.default_rng(31)
    mix = INTERLEAVED
    g = _mixed(mix)
    a = [_raw(rng, 2503 * _gb(*m), m[1]) for m in mix]      # 2503 groups: every receiver stops inside a segment
    g.submit_ragged(a)
    g.push(2, _raw(rng, 3 * _gb(*mix[2]) + 1, mix[2][1]))  # queued bytes that the restart drops
    g.restart_receiver(2, centerfreq=CENTRE + 1000000 if retune else None,
                       freqs=[CENTRE + 1000000 + 25000] if retune else None)
    b = [_raw(rng, 2999 * _gb(*m), m[1]) for m in mix]
    g.submit_ragged(b)
    g.flush()
    refs = [_ref([a[r], b[r]], m[1], restarts=[1] if r == 2 else None) for r, m in enumerate(mix)]
    _check(g, refs, "restart")
    g.close()


def test_update_receivers_keeps_moves_adds_and_removes():
    rng = np.random.default_rng(41)
    mix = INTERLEAVED[:4]
    g = _mixed(mix)
    first = [_raw(rng, 3001 * _gb(*m), m[1]) for m in mix]
    g.submit_ragged(first)
    g.flush()
    new = (10, vd.FMT_S16)
    g.update_receivers([g._current(2), g._current(0), (CENTRE + 3000000, [CENTRE + 3025000], *new)], [2, 0, -1])   # 1, 3 removed
    mix2 = [mix[2], mix[0], new]
    second = [_raw(rng, 2500 * _gb(*m), m[1]) for m in mix2]
    g.submit_ragged(second)
    g.flush()
    _check(g, [_ref([first[2], second[0]], mix2[0][1]), _ref([first[0], second[1]], mix2[1][1]), _ref([second[2]], new[1])], "update")
    g.close()


def test_flag_on_and_off_changes_nothing_else():
    rng = np.random.default_rng(51)
    iq, offs, _ = synth.traffic_stream(fs=1050000, duration_s=0.6, n_slots=8, bursts_per_s=20.0, fmt="u8", seed=7)
    mix = [(10, vd.FMT_U8)] * 2 + [(20, vd.FMT_S16)]
    iq16 = np.clip(np.round(rng.normal(0, 3000, 2 * 20 * 63000)), -32768, 32767).astype("<i2").view(np.uint8)
    streams = [iq, iq[::-1].copy(), iq16]
    spans = [[int(x) for x in rng.integers(0, 3001, len(mix))] for _ in range(24)]
    out = []
    for spec in (False, True):
        rx = [(CENTRE, [CENTRE + int(o) for o in offs], 10, vd.FMT_U8), (CENTRE, [CENTRE + int(o) for o in offs[:3]], 10, vd.FMT_U8),
              (CENTRE, [CENTRE + 25000], 20, vd.FMT_S16)]
        g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=3001 * 80, ragged=True, flags=vd.FLAG_TRACE, levels=True, channel_levels=True,
                                  spectrum=spec)
        g.process_ragged(streams, spans)
        frames = g.flush()
        st = g.stats()
        fields = [f for f in vd.Frame.__slots__ if f != "burst_timestamp"]      # (the arrival time differs between runs)
        out.append(dict(frames=[tuple(bytes(getattr(f, k)) if k == "data" else getattr(f, k) for k in fields) for f in frames],
                        cnt=g.channel_counters().tolist(), stats=st, lv=g.input_levels(),
                        ev=[(e["channel"], e["kind"], e["dec_index"], tuple(e["i"]), e["f"].tobytes()) for e in g.read_events()],
                        chl=[(c["hist"].tobytes(), c["pow"], c["peak_pow"].tobytes(), c["mag_lp"].tobytes(), c["mag_nf"].tobytes())
                             for c in g.channel_levels()]))
        g.close()
    assert out[0]["frames"] and out[0] == out[1]


def test_refusals():
    L = vd.load_library()
    from dumpvdl2_b200 import api
    out = (api._Spectrum * 2)()
    g = vd.Vdl2Channels(2100000, 20, vd.FMT_U8, CENTRE, [CENTRE], max_chunk_bytes=1 << 16)
    assert L.vdl2gpu_get_spectrum(g.h, 0, 1, out) == EINVAL
    assert "VDL2GPU_FLAG_SPECTRUM" in L.vdl2gpu_last_error().decode()
    g.close()
    g = vd.Vdl2Channels(2100000, 20, vd.FMT_U8, CENTRE, [CENTRE], max_chunk_bytes=1 << 16, spectrum=True)
    assert L.vdl2gpu_get_spectrum(g.h, 0, 2, out) == EINVAL
    assert L.vdl2gpu_get_spectrum(g.h, 1, 1, out) == EINVAL
    assert "past" in L.vdl2gpu_last_error().decode()
    assert L.vdl2gpu_get_spectrum(g.h, 0, 1, None) == EINVAL
    assert L.vdl2gpu_get_spectrum(g.h, 1, 0, out) == 0
    g.close()


def test_bursts_and_a_tone_show_where_they_are():
    fs, os_ = 1050000, 10
    offs = [-300000.0, -75000.0, 125000.0, 400000.0]
    rng = np.random.default_rng(3)
    bursts = []
    for o in offs:
        t = 0.01
        while t < 0.9:
            fr = synth.random_frames(rng)
            bursts.append(synth.BurstSpec(t, o, fr, power_dbfs=-12.0))
            t += synth.burst_duration_s(fr) + 0.01
    iq = synth.synth_stream(fs, 1.0, bursts, noise_power=1e-5, fmt="s16", seed=4)
    # a clean tone of amplitude a on bin 512 + 200 of a second input
    a = 0.25
    n = np.arange(1 << 20)
    tone = a * np.exp(2j * np.pi * 200 * n / N)
    t16 = np.empty(2 * n.size, np.float64)
    t16[0::2], t16[1::2] = tone.real, tone.imag
    t16 = np.round(t16 * 32768).astype("<i2")
    rx = [(CENTRE, [CENTRE + int(o) for o in offs], os_, vd.FMT_S16), (CENTRE, [CENTRE + 25000], os_, vd.FMT_S16)]
    g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=3001 * 80, ragged=True, spectrum=True)
    b0, b1 = iq.view(np.uint8), t16.view(np.uint8)
    g.process_ragged([b0, b1], [[3000, 3000]] * (b1.size // 40 // 3000 + 1))
    g.flush()
    recs = g.spectrum()
    m0 = vd.spectrum_metrics(recs[0], CENTRE, fs)
    rel = m0["freq_hz"] - CENTRE
    for k in np.argsort(m0["mean_dbfs"])[::-1][:3 * len(offs)]:       # the loudest bins lie on the channels
        assert min(abs(rel[k] - o) for o in offs) <= 12500, f"bin {k} at {rel[k]} Hz is not near a channel"
    floor = float(np.median(m0["mean_dbfs"]))
    for o in offs:                                                     # and every channel stands out of the floor
        near = np.abs(rel - o) <= 12500
        assert float(m0["mean_dbfs"][near].max()) > floor + 20.0, o
    m1 = vd.spectrum_metrics(recs[1], CENTRE, fs)
    assert abs(m1["mean_dbfs"][712] - 20 * np.log10(a)) < 0.1
    assert abs(m1["peak_dbfs"][712] - 20 * np.log10(a)) < 0.1
    assert int(np.argmax(m1["mean_dbfs"])) == 712
    g.close()
