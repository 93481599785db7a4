"""-m gpu: ragged spans on a mixed-receivers context (Vdl2MixedReceivers(..., ragged=True), vdl2gpu_submit_ragged).  Every
receiver brings its own number of decimated samples to each span - absent for a while and then catching up, always a
fraction of the width, counts below 12 and 160, stopping early - and must still decode exactly what one reference process
at its own rate decodes from the concatenation of everything it brought: frames (all but burst_timestamp, sync_dec_index
included), counters, trace events and the defined rows of the last span's decimated samples.  The fleet is the one of
test_gpu_mixed_receivers.py: sizes {1, 3, 8, 13, 32, 33, 40, 5, 17}, all five rate/format kinds."""
import ctypes as C
import time
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth
from oracle import pyoracle as po
from tests import util
from tests.test_gpu_mixed_receivers import SIZES, _bpp, _local, _ofmt, _ragged, _vfmt

pytestmark = pytest.mark.gpu
EINVAL, ETOOBIG = -1, -5
W = 3001                                       # the largest count of a span (max_chunk_bytes = W x 80)


def _schedule(total, seed):
    """per-span counts [span][receiver] that consume `total` decimated samples of every receiver but receiver 4, which stops
    after a third of its stream; receiver 0 is absent for the first spans, receiver 1 for three spans in the middle of a
    burst, both then catching up at full width; receiver 2 always brings a fraction of the width; receiver 3 brings counts
    below 12 and below 160 in between; the others jitter"""
    rng = np.random.default_rng(seed)
    n_rx = len(SIZES)
    target = [total] * n_rx
    target[4] = total // 3
    pos = [0] * n_rx
    spans, k = [], 0
    while any(p < t for p, t in zip(pos, target)):
        c = [int(rng.integers(W // 3, W + 1)) for _ in range(n_rx)]
        if k == 0:
            c[5] = W                                # the first span is full width (the graphs are kept for that width)
        c[0] = 0 if k < 4 else W
        c[1] = 0 if 5 <= k < 8 else W               # a burst every ~50 ms per channel: three spans of silence cut into one
        c[2] = int(0.37 * W)
        c[3] = [0, 1, 7, 11, 12, 100, 159, 160, W][k % 9]
        c = [min(n, t - p) for n, t, p in zip(c, target, pos)]
        pos = [p + n for p, n in zip(pos, c)]
        spans.append(c)
        k += 1
    return spans, pos


def _oracle_whole(x, n, trace=False):
    w = x["os"] * _bpp(x["fmt"])
    o = po.Oracle(105000 * x["os"], x["os"], _ofmt(x["fmt"]), x["centre"], x["freqs"], trace=trace, dec_tap=True)
    o.process(x["buf"][:n * w])
    return o


def _run(rxs, spans, flags, pace=False):
    g = vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"])) for x in rxs], max_chunk_bytes=W * 80,
                              flags=flags | vd.FLAG_KEEP_DEC, ragged=True)
    parts = [x["buf"] for x in rxs]
    pos = [0] * len(rxs)
    for c in spans:
        t0 = time.monotonic()
        w = [x["os"] * _bpp(x["fmt"]) for x in rxs]
        g.submit_ragged([p[q * ww:(q + n) * ww] for p, q, n, ww in zip(parts, pos, c, w)])
        pos = [q + n for q, n in zip(pos, c)]
        if pace:
            # real-time pacing for the fastest receiver of the span: arrival times then advance at least as fast as any
            # receiver's own stream, the condition under which arrival-based timestamps are monotonic
            time.sleep(max(0.0, max(c) / 105000 - (time.monotonic() - t0)))
    frames = g.flush()
    dec = g.read_dec(W + 2)
    res = dict(frames=frames, dec=dec, cnt=g.channel_counters(), stats=g.stats(), positions=g.receiver_positions(),
               events=g.read_events(1 << 20) if flags & vd.FLAG_TRACE else None)
    g.close()
    return res


@pytest.fixture(scope="module")
def fleet():
    rxs, total = _ragged(0.3, 0x52414700)
    spans, pos = _schedule(total, 11)
    oracles = [_oracle_whole(x, n, trace=True) for x, n in zip(rxs, pos)]
    first = np.concatenate([[0], np.cumsum([len(x["freqs"]) for x in rxs])])
    return rxs, spans, pos, oracles, first


@pytest.mark.parametrize("flags,k1_variant", [(0, None), (vd.FLAG_NO_GRAPH, None), (vd.FLAG_TRACE, None), (0, "4")],
                         ids=["graphs", "no_graph", "trace", "k1_variant4"])
def test_ragged_spans_match_the_oracle_per_receiver(fleet, flags, k1_variant, monkeypatch):
    rxs, spans, pos, oracles, first = fleet
    if k1_variant:                                  # without the symmetric-tap form of the filter (read at create)
        monkeypatch.setenv("VDL2GPU_K1_VARIANT", k1_variant)
    res = _run(rxs, spans, flags, pace=(flags == 0))
    st = res["stats"]
    assert st["pool_overflows"] == 0 and st["out_overflows"] == 0
    assert (st["graph_launches"] > 0) == (flags == 0)
    assert st["iq_samples"] == sum(n * x["os"] for n, x in zip(pos, rxs))
    submitted = [c for c in spans if max(c) > 0]                     # a span of all-zero counts is a no-op
    assert len(submitted) < len(spans)
    assert st["dec_samples"] == sum(max(c) for c in spans) and st["chunks_submitted"] == len(submitted)
    assert res["positions"].tolist() == pos
    last = submitted[-1]
    assert res["dec"].shape[0] == max(last)
    n_frames = 0
    for r, o in enumerate(oracles):
        chans = range(int(first[r]), int(first[r + 1]))
        what = f"receiver {r} (os {rxs[r]['os']}, {rxs[r]['fmt']}, flags {flags})"
        mine = _local([f for f in res["frames"] if f.channel in chans], chans[0])
        util.assert_frames_equal(mine, o.frames(), what)
        assert np.array_equal(res["cnt"][chans[0]:chans[-1] + 1], o.counters()), f"{what}: counters"
        n = last[r]
        wd = o.dec_samples()
        assert wd.shape[0] == pos[r]
        assert np.array_equal(res["dec"][:n, chans[0]:chans[-1] + 1].view(np.uint32), wd[pos[r] - n:pos[r]].view(np.uint32)), \
            f"{what}: decimated samples of the last span"
        if flags & vd.FLAG_TRACE:
            ev = [dict(e, channel=e["channel"] - chans[0]) for e in res["events"] if e["channel"] in chans]
            util.assert_events_equal(ev, o.events(), what)
        if flags == 0:
            by_ch = {}
            for f in mine:
                by_ch.setdefault(f.channel, []).append(f.burst_timestamp)
            for ch, ts in by_ch.items():
                assert all(b >= a for a, b in zip(ts, ts[1:])), f"{what}: channel {ch}: timestamps go back: {ts}"
        n_frames += len(mine)
    assert n_frames > 40


def test_equal_counts_equal_the_lock_step_context():
    rxs, total = _ragged(0.25, 0x52414800)
    n_dec = 2048
    plain = vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"])) for x in rxs], max_chunk_bytes=n_dec * 80,
                                  flags=vd.FLAG_KEEP_DEC)
    plain.process_chunked([x["buf"] for x in rxs], n_dec)
    fa, ca, da, sa = plain.flush(), plain.channel_counters(), plain.read_dec(n_dec + 2), plain.stats()
    plain.close()
    rag = vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"])) for x in rxs], max_chunk_bytes=n_dec * 80,
                                flags=vd.FLAG_KEEP_DEC, ragged=True)
    n_spans = (total + n_dec - 1) // n_dec
    half = n_spans // 2
    # the first half through submit_span (the ragged call with equal counts), the rest through submit_ragged
    rag.process_chunked([x["buf"][:half * n_dec * x["os"] * _bpp(x["fmt"])] for x in rxs], n_dec)
    rag.process_ragged([x["buf"][half * n_dec * x["os"] * _bpp(x["fmt"]):] for x in rxs], [[n_dec] * len(rxs)] * (n_spans - half))
    fb, cb, db, sb = rag.flush(), rag.channel_counters(), rag.read_dec(n_dec + 2), rag.stats()
    assert rag.receiver_positions().tolist() == [total] * len(rxs)
    rag.close()
    assert len(fa) > 40
    util.assert_frames_equal(fb, fa, "ragged context, equal counts vs lock-step context")
    assert [(f.channel, f.burst_seq, f.idx, f.burst_timestamp > 0) for f in fb] == [(f.channel, f.burst_seq, f.idx, True) for f in fa]
    assert np.array_equal(ca, cb)
    assert da.shape == db.shape and np.array_equal(da.view(np.uint32), db.view(np.uint32))
    for k in ("iq_samples", "dec_samples", "chunks_submitted", "msg_good", "bursts"):
        assert sa[k] == sb[k], k


def test_2048_receivers_with_jittered_counts_through_device_spans():
    """16384 channels = 2048 receivers x 8 (1024 cu8 at oversample 10, then 1024 cs16 at oversample 20), every receiver
    bringing a seeded count of up to 4000 decimated samples per span, 10 % of them absent in any span; the spans are packed
    on the device and fed through submit_ragged_device; receivers at block and warp boundaries are checked against the
    oracle on what they brought"""
    import torch
    R, n_spans, Wd = 2048, 5, 4000
    kinds = [(10, "u8"), (20, "s16")]
    bases, offs = [], None
    for os_, fmt in kinds:
        iq, offs, _ = synth.traffic_stream(105000 * os_, 0.3, 8, 12.0, 24.0, -20.0, 0x52414900, fmt)
        bases.append(np.ascontiguousarray(iq).view(np.uint8).reshape(-1))
    widths = [os_ * _bpp(fmt) for os_, fmt in kinds]
    L = min(b.size // w for b, w in zip(bases, widths))
    dev = [torch.from_numpy(b[:L * w].reshape(L, w)).cuda() for b, w in zip(bases, widths)]
    rng = np.random.default_rng(5)
    counts = rng.integers(0, Wd + 1, (n_spans, R))
    counts[rng.random((n_spans, R)) < 0.1] = 0
    counts[0, 0] = Wd
    kind_of = [0 if r < R // 2 else 1 for r in range(R)]
    shift = [(7919 * r) % L for r in range(R)]
    centres = [135000000 + 1000 * r for r in range(R)]
    rx = [(centres[r], [centres[r] + int(o) for o in offs], *[(10, vd.FMT_U8), (20, vd.FMT_S16)][kind_of[r]]) for r in range(R)]
    g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=Wd * 80, ragged=True)
    st = torch.cuda.current_stream()
    pos = np.zeros(R, np.int64)
    keep = []
    for s in range(n_spans):
        pieces = []
        for r in range(R):
            n = int(counts[s, r])
            if n:
                idx = (torch.arange(pos[r], pos[r] + n, device="cuda") + shift[r]) % L
                pieces.append(dev[kind_of[r]][idx].reshape(-1))
        buf = torch.cat(pieces)
        keep.append(buf)
        g.submit_ragged_device(buf.data_ptr(), counts[s], st.cuda_stream)
        pos += counts[s]
    got = {}
    for f in g.flush():
        got.setdefault(g.receiver_of(f.channel), []).append(f)
    stats, cnt = g.stats(), g.channel_counters()
    assert g.receiver_positions().tolist() == pos.tolist()
    g.close()
    assert stats["pool_overflows"] == 0 and stats["out_overflows"] == 0
    assert stats["msg_good"] > R // 8
    checked = 0
    for r in (0, 1, 63, 64, 67, 79, 80, 1023, 1024, 1025, 2046, 2047):
        k = kind_of[r]
        os_, fmt = kinds[k]
        iq = np.roll(bases[k][:L * widths[k]], -shift[r] * widths[k])[:int(pos[r]) * widths[k]]
        o = po.Oracle(105000 * os_, os_, _ofmt(fmt), centres[r], rx[r][1])
        o.process(iq)
        mine = _local(got.get(r, []), 8 * r)
        util.assert_frames_equal(mine, o.frames(), f"receiver {r} (os {os_}, {fmt})")
        assert np.array_equal(cnt[8 * r:8 * r + 8], o.counters()), f"receiver {r}: counters"
        checked += len(mine)
    assert checked > 2


def test_live_ragged_context_errors():
    L = vd.load_library()
    rx = [(136975000, [136975000, 137000000], 10, vd.FMT_U8), (136500000, [136525000], 20, vd.FMT_S16)]
    g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=100 * 80, ragged=True)
    buf = np.zeros(101 * (20 + 80), np.uint8)
    n = lambda *a: np.array(a, np.uint32)                                   # noqa: E731
    assert L.vdl2gpu_submit(g.h, buf.ctypes.data, 2000) == EINVAL
    assert L.vdl2gpu_submit_device(g.h, C.c_void_p(1), 2000, None) == EINVAL
    assert L.vdl2gpu_submit_planar_s16(g.h, buf.ctypes.data, buf.ctypes.data, 100) == EINVAL
    assert L.vdl2gpu_submit_ragged(g.h, buf.ctypes.data, n(0, 101).ctypes.data) == ETOOBIG
    assert "receiver 1" in L.vdl2gpu_last_error().decode()
    assert L.vdl2gpu_submit_ragged_device(g.h, C.c_void_p(1), n(101, 0).ctypes.data, None) == ETOOBIG
    assert L.vdl2gpu_submit_span(g.h, buf.ctypes.data, 101) == ETOOBIG
    assert L.vdl2gpu_submit_ragged(g.h, None, n(0, 0).ctypes.data) == 0               # all zero: a no-op
    assert L.vdl2gpu_submit_ragged(g.h, None, n(1, 0).ctypes.data) == EINVAL
    assert L.vdl2gpu_submit_ragged(g.h, buf.ctypes.data, None) == EINVAL
    assert L.vdl2gpu_get_receiver_positions(g.h, None, 2) == EINVAL
    assert L.vdl2gpu_get_receiver_positions(g.h, buf.ctypes.data, 3) == EINVAL
    assert g.stats()["chunks_submitted"] == 0 and g.receiver_positions().tolist() == [0, 0]
    assert L.vdl2gpu_submit_ragged(g.h, buf.ctypes.data, n(100, 3).ctypes.data) == 0
    g.submit_ragged([np.zeros(0, np.uint8), np.zeros(80 * 7, np.uint8)])
    g.submit_span([np.zeros(20 * 2, np.uint8), np.zeros(80 * 2, np.uint8)])
    with pytest.raises(ValueError, match="receiver 1"):
        g.submit_ragged([np.zeros(20, np.uint8), np.zeros(81, np.uint8)])
    g.flush()
    assert g.receiver_positions().tolist() == [102, 12]
    st = g.stats()
    assert st["iq_samples"] == 102 * 10 + 12 * 20 and st["dec_samples"] == 100 + 7 + 2
    g.close()
    # the ragged calls on contexts without ragged spans
    plain = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=100 * 80)
    assert L.vdl2gpu_submit_ragged(plain.h, buf.ctypes.data, n(1, 1).ctypes.data) == EINVAL
    assert "VDL2GPU_FLAG_RAGGED" in L.vdl2gpu_last_error().decode()
    assert L.vdl2gpu_submit_ragged_device(plain.h, C.c_void_p(1), n(1, 1).ctypes.data, None) == EINVAL
    plain.submit_span([np.zeros(20 * 3, np.uint8), np.zeros(80 * 3, np.uint8)])
    assert plain.receiver_positions().tolist() == [3, 3]
    plain.close()
    f = vd.Vdl2Channels(2100000, 20, vd.FMT_U8, 136975000, [136975000], max_chunk_bytes=4096)
    assert L.vdl2gpu_submit_ragged(f.h, buf.ctypes.data, n(1).ctypes.data) == EINVAL
    assert L.vdl2gpu_get_receiver_positions(f.h, buf.ctypes.data, 1) == EINVAL
    f.close()
