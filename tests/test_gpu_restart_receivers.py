"""-m gpu: restarting one receiver of a ragged mixed-receivers context (Vdl2MixedReceivers.restart_receiver,
vdl2gpu_restart_receiver).  A restarted receiver must decode what the oracle decodes from everything it brought before the
restart, followed by what a freshly started oracle - tuned to the receiver's new centre and frequencies - decodes from
everything it brings after: frames (all but burst_timestamp; the fresh oracle's sync_dec_index shifted by the restart
position and its burst_seq by the first oracle's per-channel burst count), the frequency of every frame, counters (the
sum of both oracles'), trace events (concatenated, with the same index shift) and the last span's decimated samples.
Every receiver that is not restarted must be bit for bit what it is in the same run without any restart.  The fleet is
the nine-receiver, five-kind one of test_gpu_ragged_receivers.py."""
import copy
import time
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth
from oracle import pyoracle as po
from tests import util
from tests.test_gpu_mixed_receivers import KINDS, SIZES, _bpp, _local, _ofmt, _ragged, _vfmt

pytestmark = pytest.mark.gpu
EINVAL = -1
W = 3001


def _segments(x, buf, cuts, tunings, trace=True):
    """one oracle per segment of receiver x's stream `buf` (decimated-sample cuts; equal cuts give an empty segment), each
    tuned to tunings[k] = (centre, freqs); returns the oracles and the segment bounds"""
    w = x["os"] * _bpp(x["fmt"])
    total = buf.size // w
    bounds = [0] + list(cuts) + [total]
    out = []
    for k, (cf, fr) in enumerate(tunings):
        o = po.Oracle(105000 * x["os"], x["os"], _ofmt(x["fmt"]), cf, fr, trace=trace, dec_tap=True)
        o.process(buf[bounds[k] * w:bounds[k + 1] * w])
        out.append(o)
    return out, bounds


def _expected(oracles, bounds):
    """frames (burst_seq and sync_dec_index shifted), counters and events of the segmented oracles as one stream"""
    frames, events = [], []
    cnt = None
    for o, b in zip(oracles, bounds):
        oc = o.counters().astype(np.int64)
        for f in o.frames():
            if cnt is not None:
                f.burst_seq += int(cnt[f.channel, 2])
            f.sync_dec_index += b
            frames.append(f)
        events += [dict(e, dec_index=e["dec_index"] + b) for e in o.events()]
        cnt = oc if cnt is None else cnt + oc
    return frames, cnt, events


def _check_restarted(mine, cnt, dec, events, oracles, bounds, n_last, what):
    want, want_cnt, want_ev = _expected(oracles, bounds)
    util.assert_frames_equal(mine, want, what)
    by_key = {f.key(): f for f in want}
    for f in mine:
        assert f.freq == by_key[f.key()].freq, f"{what}: {f} on {f.freq} Hz, expected {by_key[f.key()].freq}"
    assert np.array_equal(cnt.astype(np.int64), want_cnt), f"{what}: counters"
    wd = oracles[-1].dec_samples()
    assert np.array_equal(dec[:n_last].view(np.uint32), wd[wd.shape[0] - n_last:].view(np.uint32)), f"{what}: last span's samples"
    if events is not None:
        util.assert_events_equal(events, want_ev, what)


def _run(rxs, bufs, spans, restarts, flags, pace=False, zero_after=()):
    """spans[k][r] decimated samples of receiver r in span k; restarts[k] = [(r, centre or None, freqs or None), ...] called
    before span k; for k in zero_after an all-zero span (a no-op) is submitted between the restarts and span k"""
    g = vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"])) for x in rxs], max_chunk_bytes=W * 80,
                              flags=flags | vd.FLAG_KEEP_DEC, ragged=True)
    w = [x["os"] * _bpp(x["fmt"]) for x in rxs]
    pos = [0] * len(rxs)
    for k, c in enumerate(spans):
        t0 = time.monotonic()
        for r, cf, fr in restarts.get(k, []):
            g.restart_receiver(r, cf, fr)
        if k in zero_after:
            g.submit_ragged([np.zeros(0, np.uint8)] * len(rxs))
        g.submit_ragged([b[q * ww:(q + n) * ww] for b, q, n, ww in zip(bufs, pos, c, w)])
        pos = [q + n for q, n in zip(pos, c)]
        if pace:
            time.sleep(max(0.0, max(c) / 105000 - (time.monotonic() - t0)))
    res = dict(frames=g.flush(), dec=g.read_dec(W + 2), cnt=g.channel_counters(), stats=g.stats(), positions=g.receiver_positions(),
               events=g.read_events(1 << 20) if flags & vd.FLAG_TRACE else None, receivers=list(g.receivers), freqs=g.freqs.copy())
    g.close()
    return res, pos


def _in_burst(events, lo, hi, after=40):
    for e in sorted(events, key=lambda e: e["dec_index"]):
        if e["kind"] == 2 and e["i"][3] == 0 and lo <= e["dec_index"] + after < hi:
            return int(e["dec_index"]) + after
    raise AssertionError("no burst to cut into")


@pytest.fixture(scope="module")
def fleet():
    rxs, total = _ragged(0.3, 0x52535400)
    n_spans = (total + W - 1) // W
    bufs = [x["buf"].copy() for x in rxs]
    first = np.concatenate([[0], np.cumsum([len(x["freqs"]) for x in rxs])])
    # receiver 2: reset in the middle of a burst; its counts put a span boundary 40 samples into the burst's data
    x = rxs[2]
    whole = po.Oracle(105000 * x["os"], x["os"], _ofmt(x["fmt"]), x["centre"], x["freqs"], trace=True)
    whole.process(x["buf"])
    cut2 = _in_burst(whole.events(), W + 1, total - 2 * W)
    k2 = (cut2 + W - 1) // W
    # receiver 5: retuned at span 5 to a new centre and new frequencies, and fed another stream from then on
    x = rxs[5]
    os_, fmt = KINDS[5 % len(KINDS)]
    iq, offs, _ = synth.traffic_stream(105000 * os_, 0.3, SIZES[5] + SIZES[5] % 2, 6.0, 24.0, -20.0, 0x52535500, fmt)
    other = np.ascontiguousarray(iq).view(np.uint8).reshape(-1)
    k5, w5 = 5, os_ * _bpp(fmt)
    cut5 = k5 * W
    centre5 = x["centre"] + 1000000
    freqs5 = [centre5 + int(o) for o in offs[:SIZES[5]]][::-1]
    bufs[5] = np.concatenate([x["buf"][:cut5 * w5], other[:(total - cut5) * w5]])
    # receiver 3: restarted in span 3, which it brings nothing to, and again in span 4; receiver 7 in span 6, where it
    # brings 100 samples
    k3, k7 = 3, 6
    spans = []
    for k in range(n_spans + 1):
        c = [W] * len(rxs)
        c[2] = W if k < k2 - 1 else cut2 - (k2 - 1) * W if k == k2 - 1 else W
        c[3] = 0 if k == k3 else W
        c[7] = 100 if k == k7 else W
        spans.append(c)
    # trim every receiver's counts to its stream
    pos = [0] * len(rxs)
    for c in spans:
        for r in range(len(rxs)):
            c[r] = max(0, min(c[r], total - pos[r]))
            pos[r] += c[r]
    cuts = {2: [cut2], 3: [k3 * W, k3 * W], 5: [cut5], 7: [k7 * W]}
    restarts = {k2: [(2, None, None)], k3: [(3, None, None)], k3 + 1: [(3, rxs[3]["centre"], None)], k7: [(7, None, rxs[7]["freqs"])],
                k5: [(5, centre5 + 1, freqs5[::-1]), (5, centre5, freqs5)]}           # twice before one span: the last tuning wins
    tunings = {r: [(rxs[r]["centre"], rxs[r]["freqs"])] * (len(cuts[r]) + 1) for r in (2, 3, 7)}
    tunings[5] = [(rxs[5]["centre"], rxs[5]["freqs"]), (centre5, freqs5)]
    oracles = {r: _segments(rxs[r], bufs[r][:pos[r] * rxs[r]["os"] * _bpp(rxs[r]["fmt"])], cuts[r], tunings[r]) for r in cuts}
    baseline, _ = _run(rxs, bufs, spans, {}, vd.FLAG_TRACE)
    return dict(rxs=rxs, bufs=bufs, spans=spans, restarts=restarts, oracles=oracles, first=first, pos=pos, baseline=baseline,
                k2=k2, tunings=tunings)


@pytest.mark.parametrize("flags", [0, vd.FLAG_NO_GRAPH, vd.FLAG_TRACE], ids=["graphs", "no_graph", "trace"])
def test_restarted_receivers_match_segmented_oracles(fleet, flags):
    F = fleet
    rxs, first = F["rxs"], F["first"]
    res, pos = _run(rxs, F["bufs"], F["spans"], F["restarts"], flags, pace=(flags == 0), zero_after=(F["k2"],))
    st = res["stats"]
    assert st["pool_overflows"] == 0 and st["out_overflows"] == 0
    assert (st["graph_launches"] > 0) == (flags == 0)
    assert res["positions"].tolist() == pos == F["pos"]                     # positions do not reset
    assert res["receivers"][5] == F["tunings"][5][1] and res["freqs"][first[5]:first[6]].tolist() == F["tunings"][5][1][1]
    last = [c for c in F["spans"] if max(c) > 0][-1]
    base = F["baseline"]
    n_frames = 0
    for r, x in enumerate(rxs):
        chans = range(int(first[r]), int(first[r + 1]))
        what = f"receiver {r} (os {x['os']}, {x['fmt']}, flags {flags})"
        mine = _local([f for f in res["frames"] if f.channel in chans], chans[0])
        cnt = res["cnt"][chans[0]:chans[-1] + 1]
        dec = res["dec"][:, chans[0]:chans[-1] + 1]
        ev = [dict(e, channel=e["channel"] - chans[0]) for e in res["events"] if e["channel"] in chans] if res["events"] is not None else None
        if r in F["oracles"]:
            oracles, bounds = F["oracles"][r]
            _check_restarted(mine, cnt, dec, ev, oracles, bounds, last[r], what)
        else:
            theirs = _local([copy.copy(f) for f in base["frames"] if f.channel in chans], chans[0])
            util.assert_frames_equal(mine, theirs, what + " against the run without restarts")
            assert np.array_equal(cnt, base["cnt"][chans[0]:chans[-1] + 1]), f"{what}: counters"
            n = last[r]
            assert np.array_equal(dec[:n].view(np.uint32), base["dec"][:n, chans[0]:chans[-1] + 1].view(np.uint32)), f"{what}: samples"
            if ev is not None:
                util.assert_events_equal(ev, [dict(e, channel=e["channel"] - chans[0]) for e in base["events"] if e["channel"] in chans], what)
        if flags == 0:
            by_ch = {}
            for f in mine:
                by_ch.setdefault(f.channel, []).append(f.burst_timestamp)
            for ch, ts in by_ch.items():
                assert all(b >= a for a, b in zip(ts, ts[1:])), f"{what}: channel {ch}: timestamps go back: {ts}"
        n_frames += len(mine)
    assert n_frames > 40
    # the burst receiver 2 was in at its restart produced nothing
    oracles, bounds = F["oracles"][2]
    ev0 = oracles[0].events()
    assert sum(e["kind"] == 2 and e["i"][3] == 0 for e in ev0) > sum(e["kind"] == 3 for e in ev0)


def test_abandoned_bursts_return_their_pool_slots():
    """two receivers x 32 channels (a pool of 256 slots) at heavy traffic, both restarted at every span of 1000 samples: far
    more bursts are abandoned mid-way than the pool has slots, and none of them may leak"""
    os_, fmt = 10, "u8"
    w = os_ * 2
    rxs, bufs = [], []
    for r in range(2):
        iq, offs, _ = synth.traffic_stream(105000 * os_, 1.2, 32, 40.0, 24.0, -20.0, 0x52535600 + r, fmt)
        centre = 136500000 + 2000000 * r
        rxs.append(dict(centre=centre, freqs=[centre + int(o) for o in offs], os=os_, fmt=fmt))
        bufs.append(np.ascontiguousarray(iq).view(np.uint8).reshape(-1))
    total = min(b.size for b in bufs) // w
    S = 1000
    cuts = list(range(S, total, S))
    g = vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], os_, vd.FMT_U8) for x in rxs], max_chunk_bytes=W * 80, ragged=True)
    for k, c0 in enumerate(range(0, total, S)):
        if k:
            g.restart_receiver(0)
            g.restart_receiver(1)
        n = min(S, total - c0)
        g.submit_ragged([b[c0 * w:(c0 + n) * w] for b in bufs])
    frames, cnt, st = g.flush(), g.channel_counters(), g.stats()
    g.close()
    assert st["pool_overflows"] == 0
    abandoned = 0
    for r, x in enumerate(rxs):
        oracles, bounds = _segments(x, bufs[r][:total * w], cuts, [(x["centre"], x["freqs"])] * (len(cuts) + 1))
        for o in oracles[:-1]:
            ev = o.events()
            abandoned += sum(e["kind"] == 2 and e["i"][3] == 0 for e in ev) - sum(e["kind"] == 3 for e in ev)
        want, want_cnt, _ = _expected(oracles, bounds)
        mine = _local([f for f in frames if f.channel in range(32 * r, 32 * r + 32)], 32 * r)
        util.assert_frames_equal(mine, want, f"receiver {r}")
        assert np.array_equal(cnt[32 * r:32 * r + 32].astype(np.int64), want_cnt)
    assert abandoned > 256, abandoned


def test_2048_receivers_with_a_tenth_restarting_in_one_span():
    """16384 channels = 2048 receivers x 8 (1024 cu8 at oversample 10, then 1024 cs16 at oversample 20) fed through
    submit_ragged_device in full spans; in the third span about 10 % of the receivers restart, a third of those retuned
    (their channels' frequencies reversed); receivers at block and warp boundaries are checked against segmented oracles"""
    import torch
    R, n_spans, Wd = 2048, 6, 4000
    kinds = [(10, "u8"), (20, "s16")]
    bases, offs = [], None
    for os_, fmt in kinds:
        iq, offs, _ = synth.traffic_stream(105000 * os_, 0.25, 8, 12.0, 24.0, -20.0, 0x52535700, fmt)
        bases.append(np.ascontiguousarray(iq).view(np.uint8).reshape(-1))
    widths = [os_ * _bpp(fmt) for os_, fmt in kinds]
    L = min(b.size // w for b, w in zip(bases, widths))
    dev = [torch.from_numpy(b[:L * w].reshape(L, w)).cuda() for b, w in zip(bases, widths)]
    kind_of = [0 if r < R // 2 else 1 for r in range(R)]
    shift = [(7919 * r) % L for r in range(R)]
    centres = [135000000 + 1000 * r for r in range(R)]
    rx = [(centres[r], [centres[r] + int(o) for o in offs], *[(10, vd.FMT_U8), (20, vd.FMT_S16)][kind_of[r]]) for r in range(R)]
    rng = np.random.default_rng(9)
    k_restart = 2
    restarted = set(int(r) for r in rng.choice(R, R // 10, replace=False)) | {0, 63, 64, 1023, 1024, 2047}
    retuned = set(r for r in restarted if r % 3 == 0)
    g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=Wd * 80, ragged=True)
    st = torch.cuda.current_stream()
    keep = []
    for s in range(n_spans):
        if s == k_restart:
            for r in sorted(restarted):
                g.restart_receiver(r, None, rx[r][1][::-1] if r in retuned else None)
        idx = [((torch.arange(s * Wd, (s + 1) * Wd, device="cuda") + shift[r]) % L) for r in range(R)]
        buf = torch.cat([dev[kind_of[r]][idx[r]].reshape(-1) for r in range(R)])
        keep.append(buf)
        g.submit_ragged_device(buf.data_ptr(), np.full(R, Wd, np.uint32), st.cuda_stream)
    got = {}
    for f in g.flush():
        got.setdefault(g.receiver_of(f.channel), []).append(f)
    stats, cnt = g.stats(), g.channel_counters()
    g.close()
    assert stats["pool_overflows"] == 0 and stats["out_overflows"] == 0
    checked = 0
    for r in sorted({0, 1, 31, 63, 64, 67, 79, 80, 1023, 1024, 1025, 2046, 2047} | set(sorted(retuned)[:3])):
        k = kind_of[r]
        os_, fmt = kinds[k]
        x = dict(os=os_, fmt=fmt)
        iq = np.roll(bases[k][:L * widths[k]], -shift[r] * widths[k])[:n_spans * Wd * widths[k]]
        fr = rx[r][1]
        if r in restarted:
            tun = [(centres[r], fr), (centres[r], fr[::-1] if r in retuned else fr)]
            oracles, bounds = _segments(x, iq, [k_restart * Wd], tun, trace=False)
        else:
            oracles, bounds = _segments(x, iq, [], [(centres[r], fr)], trace=False)
        want, want_cnt, _ = _expected(oracles, bounds)
        mine = _local(got.get(r, []), 8 * r)
        what = f"receiver {r} (os {os_}, {fmt}{', restarted' if r in restarted else ''}{', retuned' if r in retuned else ''})"
        util.assert_frames_equal(mine, want, what)
        by_key = {f.key(): f for f in want}
        assert all(f.freq == by_key[f.key()].freq for f in mine), f"{what}: frequencies"
        assert np.array_equal(cnt[8 * r:8 * r + 8].astype(np.int64), want_cnt), f"{what}: counters"
        checked += len(mine)
    assert checked > 2


def test_live_restart_refusals():
    L = vd.load_library()
    rx = [(136975000, [136975000, 137000000], 10, vd.FMT_U8), (136500000, [136525000], 20, vd.FMT_S16)]
    fr = np.array([136500000, 136525000], np.uint32)
    g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=100 * 80, ragged=True)
    assert L.vdl2gpu_restart_receiver(g.h, 2, 0, None) == EINVAL
    assert "receiver 2 of 2" in L.vdl2gpu_last_error().decode()
    assert L.vdl2gpu_restart_receiver(g.h, 0xFFFFFFFF, 0, None) == EINVAL
    with pytest.raises(ValueError, match="1 channels, 2 frequencies"):
        g.restart_receiver(1, freqs=[136525000, 136550000])
    g.restart_receiver(0, 136950000, [136950000, 136925000])
    assert g.receivers[0] == (136950000, [136950000, 136925000])
    assert g.stats()["chunks_submitted"] == 0                  # nothing ran
    g.close()
    plain = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=100 * 80)    # lock step
    assert L.vdl2gpu_restart_receiver(plain.h, 0, 0, None) == EINVAL
    assert "VDL2GPU_FLAG_RAGGED" in L.vdl2gpu_last_error().decode()
    plain.close()
    uni = vd.Vdl2Receivers(2100000, 20, vd.FMT_U8, [(136975000, [136975000]), (136500000, [136525000])], max_chunk_bytes=4096)
    assert L.vdl2gpu_restart_receiver(uni.h, 0, 0, None) == EINVAL
    assert "VDL2GPU_FLAG_RAGGED" in L.vdl2gpu_last_error().decode()
    uni.close()
    fan = vd.Vdl2Channels(2100000, 20, vd.FMT_U8, 136975000, [136975000], max_chunk_bytes=4096)
    assert L.vdl2gpu_restart_receiver(fan.h, 0, 0, fr.ctypes.data) == EINVAL
    assert "VDL2GPU_FLAG_RAGGED" in L.vdl2gpu_last_error().decode()
    fan.close()
