"""-m gpu: input levels (VDL2GPU_FLAG_INPUT_LEVELS) measured by the levels form of every K0 kernel.  Every figure is an
integer and must equal, exactly, the numpy restatement over the samples that entered the pipeline (levels_of): through
host, planar and device submits, n_streams and one-stream-per-channel contexts, lock-step, mixed and ragged receivers,
pushed input, restarts and receivers joining and leaving, graphs on and off, trace on, on the rails, and on the
2048-receiver fleet, whose frames, metadata and counters must not change with the flag."""
import threading
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth
from oracle import pyoracle as po
from tests import cases, util
from tests.test_gpu_mixed_receivers import _bpp, _local, _ofmt
from tests.test_input_levels import add_levels, levels_of

pytestmark = pytest.mark.gpu
EINVAL = -1
CENTRE = 136975000
MIX = [(10, vd.FMT_U8), (20, vd.FMT_S16), (13, vd.FMT_U8), (20, vd.FMT_U8), (10, vd.FMT_S16)]   # every rate/format kind


def _sum(pieces, fmt):
    """the record of a stream cut into pieces, each measured on its own (a piece's partial last sample is dropped)"""
    out = levels_of(np.zeros(0, np.uint8), fmt)
    for p in pieces:
        out = add_levels(out, levels_of(p, fmt))
    return out


def _raw(rng, n_bytes, fmt):
    """noise with a DC offset, rails included"""
    if fmt == vd.FMT_U8:
        return np.clip(np.round(131 + 45 * rng.standard_normal(n_bytes)), 0, 255).astype(np.uint8)
    v = np.clip(np.round(-200 + 11000 * rng.standard_normal(n_bytes // 2)), -32768, 32767).astype("<i2")
    return v.view(np.uint8)


def _gb(os_, fmt):
    return os_ * (4 if fmt == vd.FMT_S16 else 2)


def _mixed(mix, flags=0, ragged=True, max_chunk_bytes=3001 * 80, n_inflight=4):
    rx = [(CENTRE + 200000 * r, [CENTRE + 200000 * r + 25000], os_, fmt) for r, (os_, fmt) in enumerate(mix)]
    return vd.Vdl2MixedReceivers(rx, max_chunk_bytes=max_chunk_bytes, flags=flags, ragged=ragged, n_inflight=n_inflight, levels=True)


@pytest.mark.parametrize("os_,fmt", [(20, vd.FMT_U8), (10, vd.FMT_S16)], ids=["cu8_os20", "cs16_os10"])
def test_fan_out_host_planar_and_device_submits(os_, fmt):
    import torch
    rng = np.random.default_rng(os_)
    freqs = [CENTRE - 50000, CENTRE, CENTRE + 75000]
    g = vd.Vdl2Channels(105000 * os_, os_, fmt, CENTRE, freqs, max_chunk_bytes=1 << 18, levels=True)
    assert len(g.input_levels()) == 1 and g.input_levels()[0]["samples"] == 0
    # uneven chunks, the last with an odd byte count (its partial sample is not a sample)
    sizes = [1 << 18, 40001, 1 << 18, 1234, 99999, 77777] + ([] if fmt == vd.FMT_U8 else [4097])
    pieces = [_raw(rng, n, fmt) for n in sizes]
    for p in pieces:
        g.submit(p)
    want = _sum(pieces, fmt)
    assert g.input_levels() == [want]
    if fmt == vd.FMT_S16:                                  # planar cs16 (the SDRplay hand-off)
        for n in (60000, 3331):
            v = _raw(rng, 4 * n, fmt).view("<i2")
            g.submit_planar_s16(v[0::2].copy(), v[1::2].copy())
            want = add_levels(want, levels_of(v, fmt))
    st = torch.cuda.current_stream()
    keep = []
    for n in (1 << 17, 50004):                            # device buffers, ordered after the producer's stream
        p = _raw(rng, n, fmt)
        d = torch.from_numpy(p).cuda()
        keep.append(d)
        g.submit_device(d.data_ptr(), n, st.cuda_stream)
        want = add_levels(want, levels_of(p, fmt))
    g.flush()
    got = g.input_levels()
    assert got == [want] and got[0]["clipped"] > 0 and got[0]["full_scale"] == (255 if fmt == vd.FMT_U8 else 32768)
    g.close()


def test_n_streams_and_one_stream_per_channel():
    rng = np.random.default_rng(2)
    for S, C_per in ((3, 32), (40, 1)):
        freqs = [CENTRE - 480000 + 10000 * k for k in range(S * C_per)]
        g = vd.Vdl2Channels(1050000, 10, vd.FMT_U8, CENTRE, freqs, max_chunk_bytes=1 << 16, n_streams=S, levels=True)
        streams = [[] for _ in range(S)]
        for n in (1 << 16, 30001, 4096, 777):              # per stream; odd: each stream drops its last byte
            bufs = [_raw(rng, n, vd.FMT_U8) for _ in range(S)]
            if S == 40 and n == 4096:
                bufs[7][:] = 0                             # one dead stream for a chunk
            g.submit(np.concatenate(bufs))
            for s in range(S):
                streams[s].append(bufs[s])
        g.flush()
        got = g.input_levels()
        assert got == [_sum(p, vd.FMT_U8) for p in streams], f"{S} streams x {C_per}"
        g.close()


@pytest.mark.parametrize("os_,fmt", [(20, vd.FMT_U8), (10, vd.FMT_S16), (13, vd.FMT_U8)], ids=["os20", "os10", "os13"])
def test_lock_step_receivers(os_, fmt):
    rng = np.random.default_rng(os_ + 100)
    rx = [(CENTRE + 300000 * r, [CENTRE + 300000 * r - 200000 + 10000 * k for k in range(n)]) for r, n in enumerate((3, 1, 40, 2))]
    g = vd.Vdl2Receivers(105000 * os_, os_, fmt, rx, max_chunk_bytes=1 << 17, levels=True)
    pieces = [[] for _ in rx]
    for n in (1 << 17, 65536 + 4 * 13, 4 * 13 * 7):
        bufs = [_raw(rng, n, fmt) for _ in rx]
        g.submit(bufs)
        for r in range(len(rx)):
            pieces[r].append(bufs[r])
    g.flush()
    assert g.input_levels() == [_sum(p, fmt) for p in pieces]
    g.close()


def test_mixed_fleet_of_all_kinds_through_host_and_device_spans():
    import torch
    rng = np.random.default_rng(5)
    g = _mixed(MIX, ragged=False)
    pieces = [[] for _ in MIX]
    st = torch.cuda.current_stream()
    keep = []
    for k, n_dec in enumerate((3001, 1, 2999, 7, 3001, 13)):   # odd spans: odd groups at oversample 13
        bufs = [_raw(rng, n_dec * _gb(os_, fmt), fmt) for os_, fmt in MIX]
        if k % 2 == 0:
            g.submit_span(bufs)
        else:
            d = torch.from_numpy(np.concatenate(bufs)).cuda()
            keep.append(d)
            g.submit_span_device(d.data_ptr(), n_dec, st.cuda_stream)
        for r in range(len(MIX)):
            pieces[r].append(bufs[r])
    g.flush()
    assert g.input_levels() == [_sum(p, fmt) for p, (_, fmt) in zip(pieces, MIX)]
    g.close()


def _ragged_run(mix, streams, spans, flags, n_inflight=4):
    g = _mixed(mix, flags=flags, n_inflight=n_inflight)
    pos = [0] * len(mix)
    for c in spans:
        g.submit_ragged([s[p * _gb(*m):(p + n) * _gb(*m)] for s, p, n, m in zip(streams, pos, c, mix)])
        pos = [p + n for p, n in zip(pos, c)]
    frames = g.flush()
    res = dict(levels=g.input_levels(), positions=g.receiver_positions().tolist(), frames=frames, cnt=g.channel_counters())
    g.close()
    return res, pos


@pytest.mark.parametrize("flags,n_inflight", [(0, 4), (vd.FLAG_NO_GRAPH, 4), (vd.FLAG_TRACE, 4), (0, 1)],
                         ids=["graphs", "no_graph", "trace", "inflight1"])
def test_ragged_spans_with_zero_counts(flags, n_inflight):
    rng = np.random.default_rng(9)
    streams = [_raw(rng, 40000 * _gb(*m), m[1]) for m in MIX]
    spans = []
    for k in range(12):
        c = [int(x) for x in rng.integers(0, 3002, len(MIX))]
        c[k % len(MIX)] = 0
        if k % 2:
            c[(k + 1) % len(MIX)] = 3001                   # spans of the first span's width replay its graphs
        if k == 0:
            c = [3001] * len(MIX)                          # the graphs are kept for the first span's width
        if k in (4, 5):
            c = [0] * len(MIX)                             # whole spans of zero
        spans.append(c)
    res, pos = _ragged_run(MIX, streams, spans, flags, n_inflight)
    assert res["positions"] == pos
    assert res["levels"] == [levels_of(s[:p * _gb(*m)], m[1]) for s, p, m in zip(streams, pos, MIX)]


def _feed(g, streams, piece=50000):
    """push every receiver's stream in pieces, round robin, taking the queues into spans after each round"""
    for off in range(0, max(s.size for s in streams), piece):
        for r, s in enumerate(streams):
            if off < s.size:
                g.push(r, s[off:off + piece])
        g.submit_pushed()


def test_pushes_from_one_thread_per_receiver_count_what_entered_spans():
    rng = np.random.default_rng(21)
    g = _mixed(MIX)
    streams = [_raw(rng, 30000 * _gb(*m) + 3, m[1]) for m in MIX]   # split samples and partial groups at the end

    def feed(r):
        s, off, prng = streams[r], 0, np.random.default_rng(100 + r)
        while off < s.size:
            n = int(prng.integers(1, 20000))
            g.push(r, s[off:off + n])
            off += n
    th = [threading.Thread(target=feed, args=(r,)) for r in range(len(MIX))]
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
    assert pos == [s.size // _gb(*m) for s, m in zip(streams, MIX)]
    # the bytes after the last whole group stay queued and are not counted
    assert g.input_levels() == [levels_of(s[:p * _gb(*m)], m[1]) for s, p, m in zip(streams, pos, MIX)]
    g.close()


def test_restart_drops_queued_bytes_and_keeps_counting():
    rng = np.random.default_rng(31)
    g = _mixed(MIX)
    a = [_raw(rng, 5000 * _gb(*m) + 5, m[1]) for m in MIX]
    _feed(g, a)
    extra = _raw(rng, 3 * _gb(*MIX[2]) + 1, MIX[2][1])     # whole groups of receiver 2 that the restart drops
    g.push(2, extra)
    g.restart_receiver(2)
    b = [_raw(rng, 7000 * _gb(*m) + 2, m[1]) for m in MIX]
    _feed(g, b)
    g.flush()
    got = g.input_levels()
    for r, m in enumerate(MIX):
        w = _gb(*m)
        if r == 2:
            want = add_levels(levels_of(a[r][:5000 * w], m[1]), levels_of(b[r][:7000 * w], m[1]))
        else:
            n = (a[r].size + b[r].size) // w
            want = levels_of(np.concatenate([a[r], b[r]])[:n * w], m[1])
        assert got[r] == want, f"receiver {r}"
    g.close()


def test_update_receivers_carries_kept_levels_and_starts_new_ones_at_zero():
    rng = np.random.default_rng(41)
    mix = MIX[:4]
    g = _mixed(mix)
    first = [_raw(rng, 3000 * _gb(*m), m[1]) for m in mix]
    g.submit_ragged(first)
    g.flush()
    before = g.input_levels()
    new = (10, vd.FMT_S16)
    keep = [2, 0]
    g.update_receivers([g._current(2), g._current(0), (CENTRE + 3000000, [CENTRE + 3025000], *new)], keep + [-1])
    assert g.input_levels() == [before[2], before[0], levels_of(np.zeros(0, np.uint8), vd.FMT_S16)]
    mix2 = [mix[2], mix[0], new]
    second = [_raw(rng, 2500 * _gb(*m), m[1]) for m in mix2]
    g.submit_ragged(second)
    g.flush()
    got = g.input_levels()
    assert got[0] == add_levels(before[2], levels_of(second[0], mix2[0][1]))
    assert got[1] == add_levels(before[0], levels_of(second[1], mix2[1][1]))
    assert got[2] == levels_of(second[2], new[1])
    g.close()


def test_rails_extremes_and_a_dead_receiver():
    mix = [(20, vd.FMT_U8), (10, vd.FMT_S16), (13, vd.FMT_S16), (10, vd.FMT_U8)]
    n = 3000
    rails = np.tile(np.array([0, 255], np.uint8), n * 20)                        # cu8 alternating 0 / 255
    low = np.full(2 * n * 10, -32768, "<i2").view(np.uint8)                      # cs16 all -32768
    dead = np.zeros(n * _gb(*mix[2]), np.uint8)                                  # cs16 all zero
    dead8 = np.full(n * _gb(*mix[3]), 127, np.uint8)                             # cu8 stuck at mid-scale
    g = _mixed(mix)
    g.submit_ragged([rails, low, dead, dead8])
    g.flush()
    got = g.input_levels()
    g.close()
    assert got == [levels_of(rails, mix[0][1]), levels_of(low, vd.FMT_S16), levels_of(dead, vd.FMT_S16), levels_of(dead8, vd.FMT_U8)]
    s = n * 20
    assert got[0]["clipped"] == s and got[0]["peak"] == 255 and got[0]["pow"] == s * 2 * 255 ** 2
    assert got[0]["sum_i"] == -255 * s and got[0]["sum_q"] == 255 * s
    s = n * 10
    assert got[1]["peak"] == 32768 and got[1]["pow"] == s << 31 and got[1]["clipped"] == s and got[1]["sum_i"] == -32768 * s
    assert got[2]["samples"] == n * 13 and got[2]["pow"] == 0 and got[2]["peak"] == 0 and got[2]["clipped"] == 0
    assert vd.level_metrics(got[2])["power_dbfs"] == float("-inf")
    assert got[3]["peak"] == 1 and got[3]["clipped"] == 0 and got[3]["sum_i"] == -n * 10


def test_refusals_on_a_live_context():
    L = vd.load_library()
    g = vd.Vdl2Channels(2100000, 20, vd.FMT_U8, CENTRE, [CENTRE], max_chunk_bytes=1 << 16)
    from dumpvdl2_b200 import api
    out = (api._InputLevels * 4)()
    assert L.vdl2gpu_get_input_levels(g.h, out, 1) == EINVAL
    assert "VDL2GPU_FLAG_INPUT_LEVELS" in L.vdl2gpu_last_error().decode()
    g.close()
    g = vd.Vdl2Channels(2100000, 20, vd.FMT_U8, CENTRE, [CENTRE], max_chunk_bytes=1 << 16, levels=True)
    assert L.vdl2gpu_get_input_levels(g.h, out, 2) == EINVAL
    assert "more inputs" in L.vdl2gpu_last_error().decode()
    assert L.vdl2gpu_get_input_levels(g.h, None, 1) == EINVAL
    assert L.vdl2gpu_get_input_levels(g.h, out, 0) == 0
    g.close()


def test_a_case_still_matches_the_oracle_with_levels_on():
    c = cases.case_cfg2(0.5)
    o = util.run_oracle(c, trace=True)
    for flags in (0, vd.FLAG_TRACE):
        g = vd.Vdl2Channels(c["fs"], c["oversample"], util.fmt_code(c), c["centerfreq"], c["freqs"], max_ppm=c.get("max_ppm", 0.0),
                            max_chunk_bytes=max(c["chunk"], 1 << 16), flags=flags, levels=True)
        b = util.case_bytes(c)
        g.process_chunked(b, c["chunk"])
        frames = g.flush()
        util.assert_frames_equal(frames, o.frames(), f"levels on, flags {flags}")
        assert np.array_equal(g.channel_counters(), o.counters())
        if flags & vd.FLAG_TRACE:
            util.assert_events_equal(g.read_events(), o.events(), "levels on, trace")
        fmt = vd.FMT_S16 if c["fmt"] == "s16" else vd.FMT_U8
        assert g.input_levels() == [_sum([b[k:k + c["chunk"]] for k in range(0, b.size, c["chunk"])], fmt)]
        g.close()


def test_2048_receivers_flag_on_and_off():
    """the 2048 receivers x 8 channels ragged fleet (1024 cu8 at oversample 10, then 1024 cs16 at oversample 20) fed by
    device spans with jittered counts: levels exact per receiver, and frames, metadata, counters and stats identical to
    the same run without the flag"""
    import torch
    R, n_spans, Wd = 2048, 5, 4000
    kinds = [(10, "u8"), (20, "s16")]
    bases, offs = [], None
    for os_, fmt in kinds:
        iq, offs, _ = synth.traffic_stream(105000 * os_, 0.3, 8, 12.0, 24.0, -20.0, 0x4C564C00, fmt)
        bases.append(np.ascontiguousarray(iq).view(np.uint8).reshape(-1))
    widths = [os_ * _bpp(fmt) for os_, fmt in kinds]
    L = min(b.size // w for b, w in zip(bases, widths))
    dev = [torch.from_numpy(b[:L * w].reshape(L, w)).cuda() for b, w in zip(bases, widths)]
    rng = np.random.default_rng(6)
    counts = rng.integers(0, Wd + 1, (n_spans, R))
    counts[rng.random((n_spans, R)) < 0.1] = 0
    counts[0, 0] = Wd
    kind_of = [0 if r < R // 2 else 1 for r in range(R)]
    shift = [(7919 * r) % L for r in range(R)]
    centres = [135000000 + 1000 * r for r in range(R)]
    rx = [(centres[r], [centres[r] + int(o) for o in offs], *[(10, vd.FMT_U8), (20, vd.FMT_S16)][kind_of[r]]) for r in range(R)]
    st = torch.cuda.current_stream()
    spans = []
    for s in range(n_spans):
        pieces = []
        for r in range(R):
            n = int(counts[s, r])
            if n:
                p0 = int(counts[:s, r].sum())
                idx = (torch.arange(p0, p0 + n, device="cuda") + shift[r]) % L
                pieces.append(dev[kind_of[r]][idx].reshape(-1))
        spans.append(torch.cat(pieces))
    runs = {}
    for levels in (False, True):
        g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=Wd * 80, ragged=True, levels=levels)
        for s in range(n_spans):
            g.submit_ragged_device(spans[s].data_ptr(), counts[s], st.cuda_stream)
        frames = g.flush()
        runs[levels] = dict(frames=frames, cnt=g.channel_counters(), stats=g.stats(), lv=g.input_levels() if levels else None)
        g.close()
    a, b = runs[False], runs[True]
    util.assert_frames_equal(b["frames"], a["frames"], "2048 receivers, levels on vs off")
    assert len(a["frames"]) > R // 8
    assert np.array_equal(a["cnt"], b["cnt"]) and a["stats"] == b["stats"]
    pos = counts.sum(axis=0)
    for r in range(R):
        k = kind_of[r]
        raw = np.roll(bases[k][:L * widths[k]], -shift[r] * widths[k])[:int(pos[r]) * widths[k]]
        assert b["lv"][r] == levels_of(raw, vd.FMT_U8 if kinds[k][1] == "u8" else vd.FMT_S16), f"receiver {r}"
    # spot-check receivers at block and warp boundaries against the oracle with the flag on
    got = {}
    for f in b["frames"]:
        got.setdefault(f.channel // 8, []).append(f)
    for r in (0, 1023, 1024, 2047):
        k = kind_of[r]
        os_, fmt = kinds[k]
        raw = np.roll(bases[k][:L * widths[k]], -shift[r] * widths[k])[:int(pos[r]) * widths[k]]
        o = po.Oracle(105000 * os_, os_, _ofmt(fmt), centres[r], rx[r][1])
        o.process(raw)
        util.assert_frames_equal(_local(got.get(r, []), 8 * r), o.frames(), f"receiver {r}")
