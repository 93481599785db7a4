"""-m gpu: pushed input on a ragged mixed-receivers context (Vdl2MixedReceivers.push / submit_pushed, vdl2gpu_push /
vdl2gpu_submit_pushed).  Every receiver's bytes arrive cut anywhere - single bytes, odd lengths that split cs16 samples,
pieces shorter than a group, exactly max_chunk_bytes, across the end of its ring - and each receiver must decode exactly
what one reference process at its rate decodes from the concatenation of its bytes up to its last whole decimation group:
frames (all but burst_timestamp), counters, trace events and positions.  The fleet is the one of
test_gpu_mixed_receivers.py: sizes {1, 3, 8, 13, 32, 33, 40, 5, 17}, all five rate/format kinds (oversample 13 gives odd
groups)."""
import ctypes as C
import threading
import time
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth
from oracle import pyoracle as po
from tests import util
from tests.test_gpu_mixed_receivers import _bpp, _local, _ofmt, _ragged, _vfmt
from tests.test_gpu_restart_receivers import _expected, _segments

pytestmark = pytest.mark.gpu
EINVAL, ETOOBIG = -1, -5
W = 3001                                       # the largest span (max_chunk_bytes = W x 80)
MAX_CHUNK = W * 80


def _ctx(rxs, flags=0, max_chunk=MAX_CHUNK):
    return vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"])) for x in rxs], max_chunk_bytes=max_chunk,
                                 flags=flags, ragged=True)


def _push_all(g, r, data):
    """data in max_chunk_bytes pieces, each followed by submit_pushed (a single thread must drain between pushes that
    could fill the ring: a push waits for the caller only when it follows another push without a drain)"""
    for p in range(0, data.size, MAX_CHUNK):
        g.push(r, data[p:p + MAX_CHUNK])
        g.submit_pushed()


def _cuts(n_bytes, gb, bpp, rng, max_chunk):
    """lengths that add up to n_bytes: 1 byte, odd lengths (splitting cs16 samples), shorter than a group, exactly
    max_chunk, and random ones"""
    out, left = [], n_bytes
    kinds = [1, 3, max(1, gb - 1), bpp + 1, max_chunk, None, None, None]
    while left > 0:
        k = kinds[int(rng.integers(len(kinds)))]
        n = int(rng.integers(1, max_chunk + 1)) if k is None else k
        n = min(n, left)
        out.append(n)
        left -= n
    return out


def _oracle(x, n_bytes, trace):
    w = x["os"] * _bpp(x["fmt"])
    o = po.Oracle(105000 * x["os"], x["os"], _ofmt(x["fmt"]), x["centre"], x["freqs"], trace=trace)
    o.process(x["buf"][:n_bytes // w * w])
    return o


def _check(res, rxs, n_bytes, first, trace, what):
    """every receiver against the oracle on its bytes up to its last whole group"""
    n_frames = 0
    for r, x in enumerate(rxs):
        w = x["os"] * _bpp(x["fmt"])
        o = _oracle(x, n_bytes[r], trace)
        chans = range(int(first[r]), int(first[r + 1]))
        who = f"{what}: receiver {r} (os {x['os']}, {x['fmt']})"
        mine = _local([f for f in res["frames"] if f.channel in chans], chans[0])
        util.assert_frames_equal(mine, o.frames(), who)
        assert np.array_equal(res["cnt"][chans[0]:chans[-1] + 1], o.counters()), f"{who}: counters"
        assert int(res["positions"][r]) == n_bytes[r] // w, f"{who}: position"
        if trace:
            ev = [dict(e, channel=e["channel"] - chans[0]) for e in res["events"] if e["channel"] in chans]
            util.assert_events_equal(ev, o.events(), who)
        n_frames += len(mine)
    return n_frames


@pytest.fixture(scope="module")
def fleet():
    rxs, total = _ragged(0.3, 0x50555300)
    first = np.concatenate([[0], np.cumsum([len(x["freqs"]) for x in rxs])])
    return rxs, first


@pytest.mark.parametrize("flags", [0, vd.FLAG_NO_GRAPH, vd.FLAG_TRACE], ids=["graphs", "no_graph", "trace"])
def test_random_cuts_match_the_oracle_per_receiver(fleet, flags):
    rxs, first = fleet
    rng = np.random.default_rng(0x5055 + flags)
    g = _ctx(rxs, flags)
    # every receiver stops at its own point, most of them inside a group or a sample
    n_bytes = [x["buf"].size - int(rng.integers(0, 3 * x["os"] * _bpp(x["fmt"]))) for x in rxs]
    cuts = [_cuts(n, x["os"] * _bpp(x["fmt"]), _bpp(x["fmt"]), rng, MAX_CHUNK) for n, x in zip(n_bytes, rxs)]
    off, k, since = [0] * len(rxs), [0] * len(rxs), [0] * len(rxs)
    spans = 0
    while any(kk < len(c) for kk, c in zip(k, cuts)):
        r = int(rng.integers(len(rxs)))
        if k[r] == len(cuts[r]):
            continue
        n = cuts[r][k[r]]
        if since[r] + n > MAX_CHUNK or rng.random() < 0.05:       # drain at random points, and before a push could fill the ring
            spans += g.submit_pushed()
            since = [0] * len(rxs)
        g.push(r, rxs[r]["buf"][off[r]:off[r] + n])
        since[r] += n
        off[r] += n
        k[r] += 1
    spans += g.submit_pushed()
    assert g.submit_pushed() == 0
    assert off == n_bytes
    frames = g.flush()
    res = dict(frames=frames, cnt=g.channel_counters(), stats=g.stats(), positions=g.receiver_positions(),
               events=g.read_events(1 << 20) if flags & vd.FLAG_TRACE else None)
    g.close()
    st = res["stats"]
    assert st["pool_overflows"] == 0 and st["out_overflows"] == 0
    assert st["chunks_submitted"] == spans and st["graph_launches"] == 0
    assert st["iq_samples"] == sum(n // (x["os"] * _bpp(x["fmt"])) * x["os"] for n, x in zip(n_bytes, rxs))
    # every receiver's stream wrapped its ring (max_chunk_bytes + one span + a group) at least once
    assert all(n > MAX_CHUNK + (W + 1) * x["os"] * _bpp(x["fmt"]) for n, x in zip(n_bytes, rxs))
    assert _check(res, rxs, n_bytes, first, bool(flags & vd.FLAG_TRACE), f"flags {flags}") > 40


def test_pushed_and_ragged_spans_give_the_same_frames(fleet):
    """the same bytes through submit_ragged (whole groups) and through push / submit_pushed: equal frames, counters,
    positions and span statistics when the spans take the same counts"""
    rxs, first = fleet
    n_dec = 2000
    total = min(x["buf"].size // (x["os"] * _bpp(x["fmt"])) for x in rxs) // n_dec * n_dec
    a = _ctx(rxs)
    a.process_ragged([x["buf"] for x in rxs], [[n_dec] * len(rxs)] * (total // n_dec))
    fa, ca, sa = a.flush(), a.channel_counters(), a.stats()
    a.close()
    b = _ctx(rxs)
    for s in range(total // n_dec):
        for r, x in enumerate(rxs):
            w = x["os"] * _bpp(x["fmt"])
            b.push(r, x["buf"][s * n_dec * w:(s + 1) * n_dec * w])
        assert b.submit_pushed() == 1
    fb, cb, sb = b.flush(), b.channel_counters(), b.stats()
    assert b.receiver_positions().tolist() == [total] * len(rxs)
    b.close()
    util.assert_frames_equal(fb, fa, "pushed vs ragged spans")
    assert np.array_equal(ca, cb)
    for k in ("iq_samples", "dec_samples", "chunks_submitted", "msg_good", "bursts"):
        assert sa[k] == sb[k], k


def test_one_thread_per_receiver(fleet):
    """one Python thread per receiver pushing pieces with random sleeps, the main thread pumping submit_pushed and poll; a
    small ring (max_chunk_bytes 8000) makes the fast pushers block on back-pressure, and nothing is lost"""
    rxs, first = fleet
    max_chunk = 100 * 80
    g = _ctx(rxs, max_chunk=max_chunk)

    def pusher(r):
        rng = np.random.default_rng(100 + r)
        x = rxs[r]
        off = 0
        while off < x["buf"].size:
            n = min(int(rng.integers(1, max_chunk + 1)), x["buf"].size - off)
            g.push(r, x["buf"][off:off + n])
            off += n
            if r % 3 == 0 and rng.random() < 0.1:
                time.sleep(float(rng.random()) * 2e-3)

    th = [threading.Thread(target=pusher, args=(r,)) for r in range(len(rxs))]
    for t in th:
        t.start()
    frames = []
    while any(t.is_alive() for t in th):
        g.submit_pushed()
        frames += g.poll()
        time.sleep(1e-3)
    for t in th:
        t.join()
    g.submit_pushed()
    frames += g.flush()
    res = dict(frames=frames, cnt=g.channel_counters(), stats=g.stats(), positions=g.receiver_positions())
    g.close()
    assert res["stats"]["pool_overflows"] == 0 and res["stats"]["out_overflows"] == 0
    assert _check(res, rxs, [x["buf"].size for x in rxs], first, False, "threads") > 40


def test_submit_pushed_returns_while_a_thread_keeps_pushing(fleet):
    """a thread pushes 8 MB of one receiver's stream (40 channels, cs16 at oversample 20) as fast as back-pressure lets it
    while the main thread loops submit_pushed and poll.  Each submit_pushed drains only what was queued when it was
    entered - at most a ring's worth, i.e. at most 3 spans here - so poll delivers frames while the pusher still runs;
    the decoded result equals the oracle on the bytes pushed up to the last whole group"""
    rxs, first = fleet
    x = rxs[6]
    assert len(x["freqs"]) == 40 and x["os"] == 20 and x["fmt"] == "s16"
    g = _ctx([x])
    stream = np.concatenate([x["buf"]] * (8 * 2 ** 20 // x["buf"].size + 1))[:8 * 2 ** 20]

    def pusher():
        for p in range(0, stream.size, 65536):
            g.push(0, stream[p:p + 65536])

    th = threading.Thread(target=pusher)
    th.start()
    frames, per_call, while_running = [], [], 0
    while th.is_alive():
        per_call.append(g.submit_pushed())
        got = g.poll()
        frames += got
        if th.is_alive():
            while_running += len(got)
    th.join()
    g.submit_pushed()
    frames += g.flush()
    cnt, pos = g.channel_counters(), g.receiver_positions()
    g.close()
    # a ring holds max_chunk_bytes + one span + a group: whatever is queued at entry fits in 3 spans
    assert max(per_call) <= 3 and sum(per_call) >= 10, per_call
    assert while_running >= 20, (while_running, len(frames))
    assert int(pos[0]) == stream.size // 80
    o = _oracle(dict(x, buf=stream), stream.size, False)
    util.assert_frames_equal(frames, o.frames(), "receiver pushed while submit_pushed and poll run")
    assert np.array_equal(cnt, o.counters())


def test_timestamps_follow_the_pushes(fleet):
    """paced pushes of 10 ms of samples each: every frame's timestamp is the arrival of the push that carried the last
    sample of its sync group (recorded around the call), moved back by the samples after it, within 1 ms; and monotonic
    per channel"""
    rxs, first = fleet
    g = _ctx(rxs)
    n = 5
    rxs = rxs[:n]
    rec = [[] for _ in rxs]                              # per receiver: (end position, time before, time after)
    off = [0] * n
    last = 0.0
    while any(o < x["buf"].size for o, x in zip(off, rxs)):
        # each step starts at least 10 ms after the previous one: arrivals advance at least as fast as the streams
        time.sleep(max(0.0, last + 0.01 - time.time()))
        last = time.time()
        for r, x in enumerate(rxs):
            bpp = _bpp(x["fmt"])
            k = min(1050 * x["os"] * bpp + (3 if r % 2 else 0), x["buf"].size - off[r])     # 10 ms (odd: split samples)
            if k <= 0:
                continue
            t0 = time.time()
            g.push(r, x["buf"][off[r]:off[r] + k])
            t1 = time.time()
            off[r] += k
            rec[r].append((off[r], t0, t1))
        g.submit_pushed()
    g.submit_pushed()
    frames = g.flush()
    g.close()
    checked = 0
    for r, x in enumerate(rxs):
        bpp = _bpp(x["fmt"])
        gb = x["os"] * bpp
        chans = range(int(first[r]), int(first[r + 1]))
        ends = np.array([e for e, _, _ in rec[r]])
        by_ch = {}
        for f in frames:
            if f.channel not in chans:
                continue
            e = (f.sync_dec_index + 1) * gb
            i = int(np.searchsorted(ends, e))
            back = ((ends[i] - e) // bpp) / (105000 * x["os"])
            _, t0, t1 = rec[r][i]
            assert t0 - back - 1e-3 <= f.burst_timestamp <= t1 - back + 1e-3, (r, f, t0 - back, t1 - back)
            by_ch.setdefault(f.channel, []).append(f.burst_timestamp)
            checked += 1
        for ch, ts in by_ch.items():
            assert all(b >= a for a, b in zip(ts, ts[1:])), f"receiver {r} channel {ch}: timestamps go back: {ts}"
    assert checked > 10


def test_restart_drops_the_queue(fleet):
    """receiver 2 (oversample 13, cu8) and receiver 4 (cs16) restart with whole groups and a split sample still queued:
    each decodes its old stream up to its last span, then a fresh process on the bytes pushed after the restart; the
    other receivers are unchanged"""
    rxs, first = fleet
    g = _ctx(rxs, vd.FLAG_TRACE)
    cut = 20000                                          # decimated samples before the restart that went into spans
    queued = {2: 7 * 13 * 2 + 1, 4: 5 * 10 * 4 + 3}      # whole groups and a split sample, dropped by the restart
    for r, x in enumerate(rxs):
        _push_all(g, r, x["buf"][:cut * x["os"] * _bpp(x["fmt"])])
    for r, q in queued.items():
        w = rxs[r]["os"] * _bpp(rxs[r]["fmt"])
        g.push(r, rxs[r]["buf"][cut * w:cut * w + q])
        g.restart_receiver(r)
    assert g.submit_pushed() == 0                        # nothing whole is left queued: the restarts stay pending
    rest = {}
    for r, x in enumerate(rxs):
        w = x["os"] * _bpp(x["fmt"])
        # after the restart, a restarted receiver gets the bytes from cut + 1000 groups on (a gap in its stream)
        s = (cut + 1000) * w if r in queued else cut * w
        rest[r] = x["buf"][s:]
        _push_all(g, r, rest[r])
    frames = g.flush()
    cnt, events, positions = g.channel_counters(), g.read_events(1 << 20), g.receiver_positions()
    g.close()
    for r, x in enumerate(rxs):
        w = x["os"] * _bpp(x["fmt"])
        chans = range(int(first[r]), int(first[r + 1]))
        mine = _local([f for f in frames if f.channel in chans], chans[0])
        ev = [dict(e, channel=e["channel"] - chans[0]) for e in events if e["channel"] in chans]
        what = f"receiver {r}"
        if r in queued:
            buf = np.concatenate([x["buf"][:cut * w], rest[r][:rest[r].size // w * w]])
            oracles, bounds = _segments(x, buf, [cut], [(x["centre"], x["freqs"])] * 2)
            want, want_cnt, want_ev = _expected(oracles, bounds)
            assert int(positions[r]) == buf.size // w
        else:
            o = _oracle(x, x["buf"].size, True)
            want, want_cnt, want_ev = o.frames(), o.counters().astype(np.int64), o.events()
            assert int(positions[r]) == x["buf"].size // w
        util.assert_frames_equal(mine, want, what)
        assert np.array_equal(cnt[chans[0]:chans[-1] + 1].astype(np.int64), want_cnt), f"{what}: counters"
        util.assert_events_equal(ev, want_ev, what)


def test_update_carries_partial_groups(fleet):
    """update_receivers is refused with a whole group queued; after submit_pushed the kept receivers' partial groups
    (split samples included) carry over to their new indices, and a new receiver starts empty"""
    rxs, first = fleet
    sub = rxs[:4]
    g = _ctx(sub)
    half = [x["buf"].size // 2 + (x["os"] * _bpp(x["fmt"]) // 2) + 1 for x in sub]     # ends inside a group and a sample
    for r, x in enumerate(sub):
        _push_all(g, r, x["buf"][:half[r] - 200])
        g.push(r, x["buf"][half[r] - 200:half[r]])          # more than a group queued
    before = g.flush()                                      # drained: no span in flight, but whole groups wait
    with pytest.raises(vd.Vdl2GpuError, match="whole decimation groups"):
        g.update_receivers([g._current(k) for k in (1, 0, 3)], [1, 0, 3])
    g.submit_pushed()
    old_first = np.concatenate([[0], np.cumsum([len(x["freqs"]) for x in sub])])
    before += g.flush()
    mine = {r: _local([f for f in before if old_first[r] <= f.channel < old_first[r + 1]], old_first[r]) for r in range(4)}
    # receiver 2 leaves, the others move, receiver 4 of the fleet joins
    new = rxs[4]
    g.update_receivers([g._current(1), (new["centre"], new["freqs"], new["os"], _vfmt(new["fmt"])), g._current(0), g._current(3)],
                       [1, -1, 0, 3])
    order = [1, 4, 0, 3]
    mine[4] = []
    for i, r in enumerate(order):
        x = rxs[r]
        _push_all(g, i, x["buf"][half[r] if r != 4 else 0:])
    frames = g.flush()
    cnt, positions = g.channel_counters(), g.receiver_positions()
    fnew = np.concatenate([[0], np.cumsum([len(rxs[r]["freqs"]) for r in order])])
    g.close()
    for i, r in enumerate(order):
        x = rxs[r]
        w = x["os"] * _bpp(x["fmt"])
        o = _oracle(x, x["buf"].size, False)
        chans = range(int(fnew[i]), int(fnew[i + 1]))
        got = mine[r] + _local([f for f in frames if f.channel in chans], chans[0])
        assert int(positions[i]) == x["buf"].size // w
        util.assert_frames_equal(got, o.frames(), f"receiver {r} as {i}")
        assert np.array_equal(cnt[chans[0]:chans[-1] + 1], o.counters()), f"receiver {r} as {i}: counters"


def test_refusals_on_the_device(fleet):
    rxs, _ = fleet
    L = vd.load_library()
    g = _ctx(rxs[:2])
    buf = np.zeros(MAX_CHUNK + 1, np.uint8)
    assert L.vdl2gpu_push(g.h, 2, buf.ctypes.data, 4) == EINVAL
    assert L.vdl2gpu_push(g.h, 0, None, 4) == EINVAL
    assert L.vdl2gpu_push(g.h, 0, buf.ctypes.data, MAX_CHUNK + 1) == ETOOBIG
    assert L.vdl2gpu_push(g.h, 0, None, 0) == 0
    assert g.submit_pushed() == 0
    g.push(1, buf[:5])                                      # less than a group, a split sample
    empty = [np.zeros(0, np.uint8)] * 2
    one = [np.zeros(20, np.uint8), np.zeros(0, np.uint8)]
    with pytest.raises(vd.Vdl2GpuError, match="not yet in a span"):
        g.submit_ragged(one)
    assert L.vdl2gpu_submit_span(g.h, buf.ctypes.data, 1) == EINVAL
    import torch
    dev = torch.zeros(4096, dtype=torch.uint8, device="cuda")      # a real buffer: a regression fails the assertion, nothing else
    assert L.vdl2gpu_submit_ragged_device(g.h, C.c_void_p(dev.data_ptr()), np.array([1, 0], np.uint32).ctypes.data, None) == EINVAL
    g.submit_ragged(empty)                                  # all zero: still a no-op
    g.restart_receiver(1)                                   # drops the 5 bytes
    g.submit_ragged(one)                                    # nothing queued: the two ways of feeding alternate
    g.push(0, buf[:40])
    assert g.submit_pushed() == 1
    g.flush()
    assert g.receiver_positions().tolist() == [3, 0]
    g.close()
    for ctx in (vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"])) for x in rxs[:2]], max_chunk_bytes=MAX_CHUNK),
                vd.Vdl2Channels(2100000, 20, vd.FMT_U8, 136975000, [136975000], max_chunk_bytes=4096)):
        assert L.vdl2gpu_push(ctx.h, 0, buf.ctypes.data, 4) == EINVAL
        assert "VDL2GPU_FLAG_RAGGED" in L.vdl2gpu_last_error().decode()
        assert L.vdl2gpu_submit_pushed(ctx.h) == EINVAL
        ctx.close()


def test_2048_receivers_from_eight_threads():
    """2048 receivers x 8 channels (1024 cu8 at oversample 10, then 1024 cs16 at oversample 20) fed by eight pushing
    threads in 320000-byte buffers (the reference's RTL_BUFSIZE), the main thread pumping; sampled receivers equal the
    oracle on their bytes up to the last whole group"""
    R, buf_len, n_bufs = 2048, 320000, 5
    kinds = [(10, "u8"), (20, "s16")]
    bases, offs = [], None
    total = buf_len * n_bufs
    for os_, fmt in kinds:
        secs = (total + 64 * 1024 * os_ * _bpp(fmt)) / (105000 * os_ * _bpp(fmt)) + 0.01
        iq, offs, _ = synth.traffic_stream(105000 * os_, secs, 8, 12.0, 24.0, -20.0, 0x50555400, fmt)
        bases.append(np.ascontiguousarray(iq).view(np.uint8).reshape(-1))
    kind_of = [0 if r < R // 2 else 1 for r in range(R)]
    widths = [os_ * _bpp(fmt) for os_, fmt in kinds]
    shift = [((7919 * r) % (60 * 1024)) * widths[kind_of[r]] for r in range(R)]
    centres = [135000000 + 1000 * r for r in range(R)]
    rx = [(centres[r], [centres[r] + int(o) for o in offs], *[(10, vd.FMT_U8), (20, vd.FMT_S16)][kind_of[r]]) for r in range(R)]
    g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=buf_len, ragged=True)
    errors = []

    def pusher(t):
        try:
            for k in range(n_bufs):
                for r in range(t, R, 8):
                    s = shift[r] + k * buf_len
                    g.push(r, bases[kind_of[r]][s:s + buf_len])
        except Exception as e:                               # noqa: BLE001 (reported by the main thread)
            errors.append(e)

    th = [threading.Thread(target=pusher, args=(t,)) for t in range(8)]
    for t in th:
        t.start()
    got = {}
    while any(t.is_alive() for t in th):
        g.submit_pushed()
        for f in g.poll():
            got.setdefault(g.receiver_of(f.channel), []).append(f)
        time.sleep(1e-3)
    for t in th:
        t.join()
    assert not errors, errors
    g.submit_pushed()
    for f in g.flush():
        got.setdefault(g.receiver_of(f.channel), []).append(f)
    stats, cnt, pos = g.stats(), g.channel_counters(), g.receiver_positions()
    g.close()
    assert stats["pool_overflows"] == 0 and stats["out_overflows"] == 0
    assert pos.tolist() == [total // widths[kind_of[r]] for r in range(R)]
    assert stats["msg_good"] > R // 8
    for r in (0, 1, 63, 64, 511, 1023, 1024, 1025, 2047):
        k = kind_of[r]
        os_, fmt = kinds[k]
        o = po.Oracle(105000 * os_, os_, _ofmt(fmt), centres[r], rx[r][1])
        o.process(bases[k][shift[r]:shift[r] + int(pos[r]) * widths[k]])
        mine = _local(got.get(r, []), 8 * r)
        util.assert_frames_equal(mine, o.frames(), f"receiver {r} (os {os_}, {fmt})")
        assert np.array_equal(cnt[8 * r:8 * r + 8], o.counters()), f"receiver {r}: counters"
