"""-m gpu: channel levels (VDL2GPU_FLAG_CHANNEL_LEVELS) measured by the levels form of K2a.  Every integer must equal, and
every float must be bit-identical to, the numpy restatement over the oracle's decimated samples (levels_of_dec) and the
oracle's noise-floor filters (tests/nf_oracle.py): fan-out, n_streams and one-stream-per-channel contexts, host, planar and
device submits with uneven and tiny chunks, lock-step, mixed and ragged receivers with zero and tiny counts, pushed input,
restarts with and without a retune, receivers joining and leaving, graphs on and off, trace, one chunk in flight, every
K2a time split, digital silence and the balanced slot mapping.  Frames, metadata, counters and events must not change
with the flag."""
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth
from oracle import pyoracle as po
from tests import cases, util
from tests.nf_oracle import Oracle
from tests.test_channel_levels import add_levels, levels_of_dec, zero_levels

pytestmark = pytest.mark.gpu
EINVAL = -1
CENTRE = 136975000
MIX = [(10, vd.FMT_U8), (20, vd.FMT_S16), (13, vd.FMT_U8), (20, vd.FMT_U8), (10, vd.FMT_S16)]   # every rate/format kind


def _bits(x):
    return int(np.float32(x).view(np.uint32))


def _ofmt(fmt):
    return po.FMT_S16 if fmt == vd.FMT_S16 else po.FMT_U8


def _gb(os_, fmt):
    return os_ * (4 if fmt == vd.FMT_S16 else 2)


def _oracle(os_, fmt, centre, freqs, raw):
    """(levels per channel, noise floor [n][2]) of one reference process over raw"""
    o = Oracle(105000 * os_, os_, _ofmt(fmt), centre, freqs, dec_tap=True)
    o.process(np.ascontiguousarray(raw).view(np.uint8).reshape(-1))
    d = o.dec_samples()
    lv = levels_of_dec(d) if d.shape[0] else zero_levels(len(freqs))
    nf = o.noise_floor()
    o.close()
    return lv, nf


def _assert_levels(got, want, nf, what):
    assert len(got) == len(want) == len(nf), what
    for k, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g["hist"], w["hist"]), f"{what}: channel {k} hist"
        assert g["pow"] == w["pow"], f"{what}: channel {k} pow {g['pow']} != {w['pow']}"
        assert _bits(g["peak_pow"]) == _bits(w["peak_pow"]), f"{what}: channel {k} peak"
        assert _bits(g["mag_lp"]) == _bits(nf[k][0]) and _bits(g["mag_nf"]) == _bits(nf[k][1]), f"{what}: channel {k} noise floor"
        assert g["nf_pwr_dbfs"] == pytest.approx(20 * np.log10(np.float64(g["mag_nf"]) + 0.001), rel=1e-5, abs=1e-5)


def _noise(rng, n_bytes, fmt, scale=1.0):
    if fmt == vd.FMT_U8:
        return np.clip(np.round(127.5 + 30 * scale * rng.standard_normal(n_bytes)), 0, 255).astype(np.uint8)
    return np.clip(np.round(7000 * scale * rng.standard_normal(n_bytes // 2)), -32768, 32767).astype("<i2").view(np.uint8)


def _stream(os_, fmt, offs, seconds, seed):
    rng = np.random.default_rng(seed)
    bursts = [synth.BurstSpec(0.02 + 0.07 * k, offs[k % len(offs)], synth.random_frames(rng), power_dbfs=-14.0)
              for k in range(int(seconds / 0.07))]
    iq = synth.synth_stream(105000 * os_, seconds, bursts, es_n0_db=24, fmt="u8" if fmt == vd.FMT_U8 else "s16", seed=seed)
    return np.ascontiguousarray(iq).view(np.uint8).reshape(-1)


@pytest.mark.parametrize("os_,fmt", [(20, vd.FMT_U8), (10, vd.FMT_S16)], ids=["cu8_os20", "cs16_os10"])
def test_fan_out_host_planar_and_device_submits(os_, fmt):
    import torch
    offs = [-62500.0, 25000.0, 0.0, 87500.0]
    freqs = [int(CENTRE + o) for o in offs]
    raw = _stream(os_, fmt, offs[:2], 0.45, os_)
    gb = _gb(os_, fmt)
    g = vd.Vdl2Channels(105000 * os_, os_, fmt, CENTRE, freqs, max_chunk_bytes=1 << 17, channel_levels=True)
    l0 = g.channel_levels()
    assert len(l0) == 4 and all(int(r["hist"].sum()) == 0 and r["pow"] == 0 for r in l0)
    assert all(_bits(r["mag_nf"]) == _bits(2.0) and r["mag_lp"] == 0 for r in l0)
    # uneven chunks: 0 to 3 decimated rows (with the decimation phase carried over), fewer than 160, then large ones
    sizes = [gb // 2, gb, 2 * gb, 3 * gb + 4, 100 * gb + 8, 159 * gb, 1 << 17, 40000, 1 << 17, 1 << 17, 12344]
    st = torch.cuda.current_stream()
    keep, off = [], 0
    for k, n in enumerate(sizes):
        p = raw[off:off + n]
        off += n
        if fmt == vd.FMT_S16 and k in (6, 9):             # planar cs16
            v = p.view("<i2")
            g.submit_planar_s16(v[0::2].copy(), v[1::2].copy())
        elif k in (7, 8):                                 # device buffers, ordered after the producer's stream
            d = torch.from_numpy(p.copy()).cuda()
            keep.append(d)
            g.submit_device(d.data_ptr(), n, st.cuda_stream)
        else:
            g.submit(p)
    g.flush()
    want, nf = _oracle(os_, fmt, CENTRE, freqs, raw[:off])
    got = g.channel_levels()
    _assert_levels(got, want, nf, f"fan-out os {os_}")
    assert int(got[0]["hist"].sum()) == off // gb
    assert any(_bits(r["mag_nf"]) != _bits(2.0) for r in got)
    g.close()


def test_n_streams_and_one_stream_per_channel():
    rng = np.random.default_rng(2)
    for S, C_per in ((3, 32), (40, 1)):
        freqs = [CENTRE - 480000 + 10000 * k for k in range(S * C_per)]
        g = vd.Vdl2Channels(1050000, 10, vd.FMT_U8, CENTRE, freqs, max_chunk_bytes=1 << 16, n_streams=S, channel_levels=True)
        streams = [[] for _ in range(S)]
        for n in (1 << 16, 30000, 4096, 60, 778):          # per stream
            bufs = [_noise(rng, n, vd.FMT_U8) for _ in range(S)]
            g.submit(np.concatenate(bufs))
            for s in range(S):
                streams[s].append(bufs[s])
        g.flush()
        got = g.channel_levels()
        for s in range(S):
            fr = freqs[s * C_per:(s + 1) * C_per]
            want, nf = _oracle(10, vd.FMT_U8, CENTRE, fr, np.concatenate(streams[s]))
            _assert_levels(got[s * C_per:(s + 1) * C_per], want, nf, f"{S} streams, stream {s}")
        g.close()


def test_lock_step_and_mixed_receivers():
    import torch
    rng = np.random.default_rng(3)
    os_, fmt = 13, vd.FMT_U8
    rx = [(CENTRE + 300000 * r, [CENTRE + 300000 * r - 200000 + 10000 * k for k in range(n)]) for r, n in enumerate((3, 1, 40, 2))]
    g = vd.Vdl2Receivers(105000 * os_, os_, fmt, rx, max_chunk_bytes=1 << 17, channel_levels=True)
    pieces = [[] for _ in rx]
    for n in (1 << 17, 65536 + 26, 26 * 7, 26):
        bufs = [_noise(rng, n, fmt) for _ in rx]
        g.submit(bufs)
        for r in range(len(rx)):
            pieces[r].append(bufs[r])
    g.flush()
    got = g.channel_levels()
    for r, (cf, fr) in enumerate(rx):
        want, nf = _oracle(os_, fmt, cf, fr, np.concatenate(pieces[r]))
        _assert_levels([got[c] for c in g.channels_of(r)], want, nf, f"lock-step receiver {r}")
    g.close()
    rxm = [(CENTRE + 200000 * r, [CENTRE + 200000 * r + 25000, CENTRE + 200000 * r - 50000], os_, fmt) for r, (os_, fmt) in enumerate(MIX)]
    g = vd.Vdl2MixedReceivers(rxm, max_chunk_bytes=3001 * 80, channel_levels=True)
    pieces = [[] for _ in MIX]
    st = torch.cuda.current_stream()
    keep = []
    for k, n_dec in enumerate((3001, 1, 2999, 3, 159, 2)):
        bufs = [_noise(rng, n_dec * _gb(*m), m[1]) for m in MIX]
        if k % 2 == 0:
            g.submit_span(bufs)
        else:
            d = torch.from_numpy(np.concatenate(bufs)).cuda()
            keep.append(d)
            g.submit_span_device(d.data_ptr(), n_dec, st.cuda_stream)
        for r in range(len(MIX)):
            pieces[r].append(bufs[r])
    g.flush()
    got = g.channel_levels()
    for r, (cf, fr, os_, fmt) in enumerate(rxm):
        want, nf = _oracle(os_, fmt, cf, fr, np.concatenate(pieces[r]))
        _assert_levels([got[c] for c in g.channels_of(r)], want, nf, f"mixed receiver {r}")
    g.close()


def _ragged_rx():
    offs = [25000.0, -50000.0]
    return [(CENTRE + 200000 * r, [int(CENTRE + 200000 * r + o) for o in offs], os_, fmt) for r, (os_, fmt) in enumerate(MIX)], offs


@pytest.mark.parametrize("flags,n_inflight", [(0, 4), (vd.FLAG_NO_GRAPH, 4), (vd.FLAG_TRACE, 4), (0, 1)],
                         ids=["graphs", "no_graph", "trace", "inflight1"])
def test_ragged_spans_with_zero_and_tiny_counts_flag_on_and_off(flags, n_inflight):
    rxs, offs = _ragged_rx()
    streams = [_stream(os_, fmt, offs, 0.4, 50 + r) for r, (_, _, os_, fmt) in enumerate(rxs)]
    rng = np.random.default_rng(9)
    spans = []
    for k in range(14):
        c = [int(x) for x in rng.integers(0, 3002, len(MIX))]
        c[k % len(MIX)] = 0
        c[(k + 2) % len(MIX)] = int(rng.integers(1, 4))   # counts 1 to 3
        if k % 2:
            c[(k + 1) % len(MIX)] = 3001                   # spans of the first span's width replay its graphs
        if k == 0:
            c = [3001] * len(MIX)
        if k == 5:
            c = [0] * len(MIX)
        spans.append(c)
    runs = {}
    for on in (False, True):
        g = vd.Vdl2MixedReceivers(rxs, max_chunk_bytes=3001 * 80, flags=flags, ragged=True, n_inflight=n_inflight, channel_levels=on)
        g.process_ragged(streams, spans)
        frames = g.flush()
        runs[on] = dict(frames=frames, cnt=g.channel_counters(), stats=g.stats(), pos=g.receiver_positions().tolist(),
                        ev=g.read_events() if flags & vd.FLAG_TRACE else None, lv=g.channel_levels() if on else None)
        g.close()
    a, b = runs[False], runs[True]
    util.assert_frames_equal(b["frames"], a["frames"], "ragged, channel levels on vs off")
    assert len(a["frames"]) > 0
    assert np.array_equal(a["cnt"], b["cnt"]) and a["stats"] == b["stats"] and a["pos"] == b["pos"]
    if flags & vd.FLAG_TRACE:
        assert len(a["ev"]) > 0 and len(a["ev"]) == len(b["ev"])
        for x, y in zip(a["ev"], b["ev"]):
            assert (x["channel"], x["kind"], x["dec_index"], x["i"]) == (y["channel"], y["kind"], y["dec_index"], y["i"])
            assert np.array_equal(x["f"].view(np.uint32), y["f"].view(np.uint32))
    for r, (cf, fr, os_, fmt) in enumerate(rxs):
        want, nf = _oracle(os_, fmt, cf, fr, streams[r][:b["pos"][r] * _gb(os_, fmt)])
        _assert_levels(b["lv"][2 * r:2 * r + 2], want, nf, f"ragged receiver {r}")


def test_push_restart_with_and_without_retune_and_update_receivers():
    rxs, offs = _ragged_rx()
    g = vd.Vdl2MixedReceivers(rxs, max_chunk_bytes=3001 * 80, ragged=True, channel_levels=True)
    a = [_stream(os_, fmt, offs, 0.15, 70 + r)[:4000 * _gb(os_, fmt)] for r, (_, _, os_, fmt) in enumerate(rxs)]
    for off in range(0, max(s.size for s in a), 50001):    # pushes of any length, then spans of what is queued
        for r, s in enumerate(a):
            if off < s.size:
                g.push(r, s[off:off + 50001])
        g.submit_pushed()
    g.flush()
    assert g.receiver_positions().tolist() == [4000] * len(rxs)
    retune = [f + 12500 for f in rxs[3][1]]
    g.restart_receiver(2)
    g.restart_receiver(3, freqs=retune)
    b = [_noise(np.random.default_rng(80 + r), 2500 * _gb(os_, fmt), fmt) for r, (_, _, os_, fmt) in enumerate(rxs)]
    g.process_ragged(b, [[1000, 3, 0, 1, 1000], [1500, 2497, 2500, 2499, 1500]])
    g.flush()
    got = g.channel_levels()
    expect = {}
    for r, (cf, fr, os_, fmt) in enumerate(rxs):
        if r in (2, 3):                                    # the old process's figures, then a new process's
            lv_a, _ = _oracle(os_, fmt, cf, fr, a[r])
            lv_b, nf = _oracle(os_, fmt, cf, retune if r == 3 else fr, b[r])
            want = [add_levels(x, y) for x, y in zip(lv_a, lv_b)]
        else:
            want, nf = _oracle(os_, fmt, cf, fr, np.concatenate([a[r], b[r]]))
        _assert_levels(got[2 * r:2 * r + 2], want, nf, f"restart, receiver {r}")
        expect[r] = [dict(x, mag_lp=y["mag_lp"], mag_nf=y["mag_nf"]) for x, y in zip(want, got[2 * r:2 * r + 2])]
    # receivers 3 and 0 kept (in that order), 1, 2 and 4 removed, one new receiver
    new = (CENTRE + 3000000, [CENTRE + 3025000, CENTRE + 2950000, CENTRE + 3000000], 10, vd.FMT_S16)
    g.update_receivers([g._current(3), g._current(0), new], [3, 0, -1])
    moved = g.channel_levels()
    assert len(moved) == 7
    for k, w in enumerate(expect[3] + expect[0]):
        assert np.array_equal(moved[k]["hist"], w["hist"]) and moved[k]["pow"] == w["pow"]
        assert _bits(moved[k]["peak_pow"]) == _bits(w["peak_pow"]) and _bits(moved[k]["mag_nf"]) == _bits(w["mag_nf"])
    assert all(int(r["hist"].sum()) == 0 and r["pow"] == 0 and r["peak_pow"] == 0 and _bits(r["mag_nf"]) == _bits(2.0) for r in moved[4:])
    c = [_noise(np.random.default_rng(90 + k), 2000 * _gb(*m), m[1]) for k, m in enumerate([(20, vd.FMT_U8), (10, vd.FMT_U8), (10, vd.FMT_S16)])]
    g.process_ragged(c, [[2000, 7, 1], [0, 1993, 1999]])
    g.flush()
    got = g.channel_levels()
    cf3, _, os3, fmt3 = rxs[3]
    lv_c, nf3 = _oracle(os3, fmt3, cf3, retune, np.concatenate([b[3], c[0]]))
    lv_a, _ = _oracle(os3, fmt3, cf3, rxs[3][1], a[3])
    _assert_levels(got[0:2], [add_levels(x, y) for x, y in zip(lv_a, lv_c)], nf3, "kept receiver 3")
    cf0, fr0, os0, fmt0 = rxs[0]
    want, nf = _oracle(os0, fmt0, cf0, fr0, np.concatenate([a[0], b[0], c[1]]))
    _assert_levels(got[2:4], want, nf, "kept receiver 0")
    want, nf = _oracle(10, vd.FMT_S16, new[0], new[1], c[2])
    _assert_levels(got[4:7], want, nf, "new receiver")
    g.close()


@pytest.mark.parametrize("env", [dict(VDL2GPU_K2A_SPLIT="1"), dict(VDL2GPU_K2A_SPLIT="256"), dict(VDL2GPU_STAGES="3")],
                         ids=["split1", "split256", "stages3"])
def test_time_splits_with_loud_clipped_input(env, monkeypatch):
    """a rail-to-rail cu8 input at oversample 10 in chunks of 52428 decimated samples: a loud channel's p ~ 2, q ~ 2^49, so
    with one time slice a thread's partial passes 2^64 (the register fold)"""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(4)
    n = 3 * (1 << 20)
    raw = np.where(rng.random(n) < 0.5, 0, 255).astype(np.uint8)
    raw[: n // 2] = 255                                    # first half: I = Q = +1 (DC: p near 2 for the channel at the centre)
    freqs = [CENTRE, CENTRE + 25000, CENTRE - 87500]
    g = vd.Vdl2Channels(1050000, 10, vd.FMT_U8, CENTRE, freqs, max_chunk_bytes=1 << 20, channel_levels=True)
    g.process_chunked(raw, 1 << 20)
    g.flush()
    got = g.channel_levels()
    want, nf = _oracle(10, vd.FMT_U8, CENTRE, freqs, raw)
    _assert_levels(got, want, nf, f"loud input, {env}")
    assert got[0]["pow"] > 1 << 64 and got[0]["peak_pow"] > 1.9 and int(got[0]["hist"][37:39].sum()) > 70000   # p near 2
    g.close()


def test_digital_silence():
    g = vd.Vdl2Channels(1050000, 10, vd.FMT_S16, CENTRE, [CENTRE, CENTRE + 50000], max_chunk_bytes=1 << 17, channel_levels=True)
    raw = np.zeros(5 * (1 << 17) + 40, np.uint8)
    g.process_chunked(raw, 1 << 17)
    g.flush()
    got = g.channel_levels()
    want, nf = _oracle(10, vd.FMT_S16, CENTRE, [CENTRE, CENTRE + 50000], raw)
    _assert_levels(got, want, nf, "digital silence")
    n = raw.size // 40
    for r in got:
        assert int(r["hist"][0]) == n and int(r["hist"][1:].sum()) == 0 and r["pow"] == 0 and _bits(r["peak_pow"]) == 0
        assert vd.channel_level_metrics(r)["power_dbfs"] == float("-inf")
    g.close()


def test_balanced_slot_mapping_against_the_contexts_own_decimated_samples():
    """9000 channels (between 16 and 32 per warp of a 132-SM H100: the balanced mapping deals 17 or 18 to each warp);
    the expected figures come from vdl2gpu_read_dec after each chunk"""
    import torch
    props = torch.cuda.get_device_properties(0)
    n_ch = 9000
    assert 16 * 4 * props.multi_processor_count < n_ch <= 32 * 4 * props.multi_processor_count
    freqs = [CENTRE - 450000 + 100 * k for k in range(n_ch)]
    g = vd.Vdl2Channels(1050000, 10, vd.FMT_U8, CENTRE, freqs, max_chunk_bytes=1 << 16, n_inflight=1, channel_levels=True)
    rng = np.random.default_rng(8)
    want = zero_levels(n_ch)
    for n in (1 << 16, 20000, 58, 1 << 16):
        g.submit(_noise(rng, n, vd.FMT_U8, scale=2.0))
        g.flush()
        d = g.read_dec(4000)
        want = [add_levels(x, y) for x, y in zip(want, levels_of_dec(d))] if d.shape[0] else want
    got = g.channel_levels()
    for k in range(n_ch):
        assert np.array_equal(got[k]["hist"], want[k]["hist"]) and got[k]["pow"] == want[k]["pow"], f"channel {k}"
        assert _bits(got[k]["peak_pow"]) == _bits(want[k]["peak_pow"]), f"channel {k}"
    g.close()


def test_a_case_matches_the_oracle_flag_on_and_off():
    c = cases.case_cfg2(0.5)
    b = util.case_bytes(c)
    o = Oracle(c["fs"], c["oversample"], util.fmt_code(c), c["centerfreq"], c["freqs"], max_ppm=c.get("max_ppm", 0.0), trace=True,
               dec_tap=True)
    o.process_chunked(b, c["chunk"])
    for flags in (0, vd.FLAG_TRACE):
        runs = {}
        for on in (False, True):
            g = vd.Vdl2Channels(c["fs"], c["oversample"], util.fmt_code(c), c["centerfreq"], c["freqs"], max_ppm=c.get("max_ppm", 0.0),
                                max_chunk_bytes=max(c["chunk"], 1 << 16), flags=flags, channel_levels=on)
            g.process_chunked(b, c["chunk"])
            runs[on] = dict(frames=g.flush(), cnt=g.channel_counters(), stats=g.stats(),
                            ev=g.read_events() if flags else None, lv=g.channel_levels() if on else None)
            g.close()
        util.assert_frames_equal(runs[True]["frames"], o.frames(), f"channel levels on, flags {flags}")
        util.assert_frames_equal(runs[True]["frames"], runs[False]["frames"], f"channel levels on vs off, flags {flags}")
        assert np.array_equal(runs[True]["cnt"], o.counters()) and np.array_equal(runs[True]["cnt"], runs[False]["cnt"])
        assert runs[True]["stats"] == runs[False]["stats"]
        if flags:
            util.assert_events_equal(runs[True]["ev"], o.events(), "channel levels on, trace")
            util.assert_events_equal(runs[True]["ev"], runs[False]["ev"], "channel levels on vs off, trace")
        _assert_levels(runs[True]["lv"], levels_of_dec(o.dec_samples()), o.noise_floor(), "cfg2")


def test_refusals_on_a_live_context():
    L = vd.load_library()
    from dumpvdl2_b200 import api
    out = (api._ChannelLevels * 4)()
    g = vd.Vdl2Channels(2100000, 20, vd.FMT_U8, CENTRE, [CENTRE, CENTRE + 25000], max_chunk_bytes=1 << 16, levels=True)
    assert L.vdl2gpu_get_channel_levels(g.h, out, 1) == EINVAL
    assert "VDL2GPU_FLAG_CHANNEL_LEVELS" in L.vdl2gpu_last_error().decode()
    g.close()
    g = vd.Vdl2Channels(2100000, 20, vd.FMT_U8, CENTRE, [CENTRE, CENTRE + 25000], max_chunk_bytes=1 << 16, channel_levels=True)
    assert L.vdl2gpu_get_channel_levels(g.h, out, 3) == EINVAL
    assert "more channels" in L.vdl2gpu_last_error().decode()
    assert L.vdl2gpu_get_channel_levels(g.h, None, 1) == EINVAL
    assert L.vdl2gpu_get_channel_levels(g.h, out, 0) == 0
    assert L.vdl2gpu_get_channel_levels(g.h, out, 2) == 0
    g.close()
