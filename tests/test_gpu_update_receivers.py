"""-m gpu: receivers joining and leaving a running ragged mixed-receivers context (Vdl2MixedReceivers.update_receivers,
add_receivers, remove_receivers; vdl2gpu_update_receivers).  The oracle runs per receiver over exactly the samples that
receiver brought while it was a member: a kept receiver must equal one oracle over its whole stream, a receiver that
joined one oracle started at its join, and a removed receiver's output up to its removal one oracle over that prefix -
frames (all but burst_timestamp), per-channel counters and the last span's decimated samples.  The fleet has the rates,
formats and warp- and block-straddling sizes of test_gpu_mixed_receivers.py."""
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth
from oracle import pyoracle as po
from tests import util
from tests.test_gpu_mixed_receivers import _bpp, _local, _ofmt, _ragged, _vfmt
from tests.test_gpu_restart_receivers import _expected, _in_burst, _segments

pytestmark = pytest.mark.gpu
EINVAL = -1
W = 3001


def _desc(x):
    return (x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"]))


def _w(x):
    return x["os"] * _bpp(x["fmt"])


class _Fleet:
    """a context whose members (station ids, in context order) change; per station: samples brought, frames (local channel
    numbers), counters when it left or at the end"""

    def __init__(self, stations, members, flags=0, max_chunk_bytes=W * 80):
        self.st, self.members = stations, list(members)
        self.g = vd.Vdl2MixedReceivers([_desc(stations[i]) for i in members], max_chunk_bytes=max_chunk_bytes,
                                       flags=flags | vd.FLAG_KEEP_DEC, ragged=True)
        self.pos = {i: 0 for i in members}
        self.frames = {i: [] for i in members}
        self.counters = {}
        self.last = {}
        self.marks = []                  # per update: frames per station delivered before it

    def span(self, counts):
        """counts[id] decimated samples of each member (missing: 0)"""
        bufs = []
        for i in self.members:
            x, n = self.st[i], int(counts.get(i, 0))
            bufs.append(x["buf"][self.pos[i] * _w(x):(self.pos[i] + n) * _w(x)])
            self.pos[i] += n
            self.last[i] = n
        self.g.submit_ragged(bufs)

    def _drain(self):
        for f in self.g.flush():
            r = self.g.receiver_of(f.channel)
            f.channel -= self.g.channels_of(r)[0]
            self.frames[self.members[r]].append(f)
        cnt = self.g.channel_counters()
        return {i: cnt[self.g.channels_of(r)[0]:self.g.channels_of(r)[-1] + 1].astype(np.int64) for r, i in enumerate(self.members)}

    def update(self, members):
        cnt = self._drain()
        self.marks.append({i: len(f) for i, f in self.frames.items()})
        for i in self.members:
            if i not in members:
                self.counters[i] = cnt[i]
        old = {i: r for r, i in enumerate(self.members)}
        self.g.update_receivers([_desc(self.st[i]) for i in members], [old.get(i, -1) for i in members])
        for i in members:
            if i not in old:
                self.pos[i], self.frames[i] = 0, []
        self.members = list(members)
        assert self.g.read_dec(W + 2).shape[0] == 0                  # no rows until a span runs
        assert self.g.receiver_positions().tolist() == [self.pos[i] for i in members]

    def finish(self):
        cnt = self._drain()
        self.counters.update(cnt)
        dec = self.g.read_dec(W + 2)
        self.dec = {i: dec[:, self.g.channels_of(r)[0]:self.g.channels_of(r)[-1] + 1] for r, i in enumerate(self.members)}
        self.stats = self.g.stats()
        self.g.close()


def _check_station(F, i, what):
    x = F.st[i]
    o = po.Oracle(105000 * x["os"], x["os"], _ofmt(x["fmt"]), x["centre"], x["freqs"], dec_tap=True)
    o.process(x["buf"][:F.pos[i] * _w(x)])
    util.assert_frames_equal(F.frames[i], o.frames(), what)
    assert np.array_equal(F.counters[i], o.counters().astype(np.int64)), f"{what}: counters"
    if i in F.members:
        n, wd = F.last[i], o.dec_samples()
        assert n > 0
        assert np.array_equal(F.dec[i][:n].view(np.uint32), wd[wd.shape[0] - n:].view(np.uint32)), f"{what}: last span's samples"
    return len(F.frames[i])


@pytest.fixture(scope="module")
def stations():
    a, _ = _ragged(0.4, 0x55504400)
    b, _ = _ragged(0.4, 0x55504500)
    st = a + [b[4], b[5], b[1], b[2]]                                # ids 9..12: 32, 33, 3 and 8 channels
    whole = {}
    for i in (4, 3):
        x = st[i]
        o = po.Oracle(105000 * x["os"], x["os"], _ofmt(x["fmt"]), x["centre"], x["freqs"], trace=True)
        o.process(x["buf"])
        whole[i] = o.events()
    cut4 = _in_burst(whole[4], W + 1, 2 * W)                         # station 4 is inside a burst at the first update
    cut3 = _in_burst(whole[3], 3 * W + 1, 4 * W)                     # station 3 at the second, which removes it
    return st, cut4, cut3


@pytest.mark.parametrize("flags", [0, vd.FLAG_NO_GRAPH], ids=["graphs", "no_graph"])
def test_fleet_grows_shrinks_and_reorders(stations, flags):
    st, cut4, cut3 = stations
    F = _Fleet(st, range(9), flags)
    F.span({i: W for i in range(9)})
    F.span({**{i: W for i in range(9)}, 4: cut4 - W, 7: 0})
    F.update([11, 0, 1, 9, 2, 3, 4, 5, 6, 7, 8, 10])                 # join at the front, in the middle and at the end
    F.span({i: W for i in F.members})
    F.span({**{i: W for i in F.members}, 3: cut3 - F.pos[3]})
    F.update([0, 1, 9, 2, 4, 5, 7, 8])                               # the first, the last, one mid-burst and another leave
    F.span({i: W for i in F.members})
    F.span({i: W - 100 * k for k, i in enumerate(F.members)})
    F.update([8, 2, 9, 0, 7, 1, 5, 4])                               # reorder
    F.span({i: W for i in F.members})
    F.span({i: W - 37 * k - 1 for k, i in enumerate(F.members)})
    F.finish()
    assert F.stats["pool_overflows"] == 0 and F.stats["out_overflows"] == 0
    assert (F.stats["graph_launches"] > 0) == (flags == 0)
    n = sum(_check_station(F, i, f"station {i} (os {st[i]['os']}, {st[i]['fmt']}, flags {flags})") for i in sorted(F.pos))
    assert n > 40
    # station 4's burst in progress at the first update was delivered after it, under its new channel numbers
    assert any(f.sync_dec_index < cut4 for f in F.frames[4][F.marks[0][4]:]), "the burst across the update"
    assert F.pos[3] == cut3


def test_removed_receivers_return_their_pool_slots():
    """two receivers x 32 channels (a pool of 256 slots) at heavy traffic: receiver 1 is removed after every span of 1000
    samples, with bursts in progress, and a new receiver takes its place with the next piece of the stream; far more bursts
    are dropped than the pool has slots, and none may leak"""
    os_, fmt = 10, "u8"
    w = os_ * 2
    xs = []
    for r in range(2):
        iq, offs, _ = synth.traffic_stream(105000 * os_, 1.2, 32, 40.0, 24.0, -20.0, 0x55504600 + r, fmt)
        centre = 136500000 + 2000000 * r
        xs.append(dict(centre=centre, freqs=[centre + int(o) for o in offs], os=os_, fmt=fmt,
                       buf=np.ascontiguousarray(iq).view(np.uint8).reshape(-1)))
    total = min(x["buf"].size for x in xs) // w
    S = 1000
    g = vd.Vdl2MixedReceivers([_desc(x) for x in xs], max_chunk_bytes=W * 80, ragged=True)
    keep, pieces = [], []
    for k, c0 in enumerate(range(0, total, S)):
        n = min(S, total - c0)
        g.submit_ragged([xs[0]["buf"][c0 * w:(c0 + n) * w], xs[1]["buf"][c0 * w:(c0 + n) * w]])
        fr = g.flush()
        keep += [f for f in fr if f.channel < 32]
        pieces.append(_local([f for f in fr if f.channel >= 32], 32))
        if c0 + n < total:
            g.remove_receivers([1])
            g.add_receivers([_desc(xs[1])])
    cnt, stats = g.channel_counters(), g.stats()
    g.close()
    assert stats["pool_overflows"] == 0
    want = po.Oracle(105000 * os_, os_, _ofmt(fmt), xs[0]["centre"], xs[0]["freqs"])
    want.process(xs[0]["buf"][:total * w])
    util.assert_frames_equal(keep, want.frames(), "the receiver that stays")
    assert np.array_equal(cnt[:32].astype(np.int64), want.counters().astype(np.int64))
    dropped = 0
    for k, c0 in enumerate(range(0, total, S)):
        o = po.Oracle(105000 * os_, os_, _ofmt(fmt), xs[1]["centre"], xs[1]["freqs"], trace=True)
        o.process(xs[1]["buf"][c0 * w:min(total, c0 + S) * w])
        util.assert_frames_equal(pieces[k], o.frames(), f"piece {k} of the receiver that comes and goes")
        ev = o.events()
        dropped += sum(e["kind"] == 2 and e["i"][3] == 0 for e in ev) - sum(e["kind"] == 3 for e in ev)
    assert dropped > 256, dropped


def test_pending_restart_survives_an_index_shift(stations):
    """receiver 4 is retuned, then two receivers join in front of it before any span runs: the restart applies with the
    next span at its new index 6"""
    st, _, _ = stations
    F = _Fleet(st, range(9))
    F.span({i: W for i in range(9)})
    x = st[4]
    retuned = x["freqs"][::-1]
    F.g.restart_receiver(4, None, retuned)
    F.st = list(st)
    F.st[4] = dict(x, freqs=retuned)                                 # its description after the restart
    F.update([0, 9, 1, 10, 2, 3, 4, 5, 6, 7, 8])
    assert F.g.receivers[6] == (x["centre"], retuned)
    F.span({i: W for i in F.members})
    F.span({i: W - 11 for i in F.members})
    F.finish()
    oracles, bounds = _segments(x, x["buf"][:F.pos[4] * _w(x)], [W], [(x["centre"], x["freqs"]), (x["centre"], retuned)], trace=False)
    want, want_cnt, _ = _expected(oracles, bounds)
    util.assert_frames_equal(F.frames[4], want, "the restarted receiver")
    assert np.array_equal(F.counters[4], want_cnt)
    for i in (0, 1, 3, 8, 9, 10):
        _check_station(F, i, f"station {i}")


def test_2048_receivers_cross_the_balanced_mapping():
    """16384 channels = 2048 receivers x 8 (1024 cu8 at oversample 10, then 1024 cs16 at oversample 20; balanced slot
    mapping), fed through submit_ragged_device: 72 receivers join in the middle (16960 channels, past the balanced mapping),
    then 100 leave, the first and the last among them (balanced again); sampled receivers against the oracle"""
    import torch
    R, Wd = 2048, 4000
    kinds = [(10, "u8"), (20, "s16")]
    bases, offs = [], None
    for os_, fmt in kinds:
        iq, offs, _ = synth.traffic_stream(105000 * os_, 0.25, 8, 12.0, 24.0, -20.0, 0x55504700, fmt)
        bases.append(np.ascontiguousarray(iq).view(np.uint8).reshape(-1))
    widths = [os_ * _bpp(fmt) for os_, fmt in kinds]
    L = min(b.size // w for b, w in zip(bases, widths))
    dev = [torch.from_numpy(b[:L * w].reshape(L, w)).cuda() for b, w in zip(bases, widths)]
    n_st = R + 72
    kind_of = [0 if i < R // 2 else 1 for i in range(R)] + [i % 2 for i in range(72)]
    shift = [(7919 * i) % L for i in range(n_st)]
    desc = []
    for i in range(n_st):
        centre = 135000000 + 1000 * i
        desc.append((centre, [centre + int(o) for o in offs], *[(10, vd.FMT_U8), (20, vd.FMT_S16)][kind_of[i]]))
    members = list(range(R))
    g = vd.Vdl2MixedReceivers([desc[i] for i in members], max_chunk_bytes=Wd * 80, ragged=True)
    st = torch.cuda.current_stream()
    pos = {i: 0 for i in members}
    frames = {i: [] for i in range(n_st)}
    counters = {}
    keep = []

    def drain():
        for f in g.flush():
            r = g.receiver_of(f.channel)
            frames[members[r]].append(_local([f], 8 * r)[0])
        cnt = g.channel_counters()
        return {i: cnt[8 * r:8 * r + 8].astype(np.int64) for r, i in enumerate(members)}

    def span():
        parts = []
        for i in members:
            idx = (torch.arange(pos[i], pos[i] + Wd, device="cuda") + shift[i]) % L
            parts.append(dev[kind_of[i]][idx].reshape(-1))
            pos[i] += Wd
        buf = torch.cat(parts)
        keep.append(buf)
        g.submit_ragged_device(buf.data_ptr(), np.full(len(members), Wd, np.uint32), st.cuda_stream)

    span(); span()
    drain()
    members = members[:1024] + list(range(R, n_st)) + members[1024:]
    g.update_receivers([desc[i] for i in members], [i if i < R else -1 for i in members])
    for i in range(R, n_st):
        pos[i] = 0
    assert g.n_channels == 8 * (R + 72)
    span(); span()
    cnt = drain()
    gone = {members[0], members[-1]} | set(members[1:1024:21] + members[1024:1096:3] + members[1100:2120:40])
    for i in gone:
        counters[i] = cnt[i]
    keep_idx = {i: r for r, i in enumerate(members)}
    members = [i for i in members if i not in gone]
    g.remove_receivers(sorted(keep_idx[i] for i in gone))
    assert [g.receivers[r][0] for r in range(len(members))] == [desc[i][0] for i in members]
    span(); span()
    counters.update(drain())
    stats = g.stats()
    g.close()
    assert stats["pool_overflows"] == 0 and stats["out_overflows"] == 0
    checked = 0
    sample = sorted({0, 1, 63, 64, 1023, 1024, 1025, 2046, 2047, R, R + 1, R + 40, R + 71} | set(sorted(gone)[:4]))
    for i in sample:
        os_, fmt = kinds[kind_of[i]]
        iq = np.roll(bases[kind_of[i]][:L * widths[kind_of[i]]], -shift[i] * widths[kind_of[i]])[:pos[i] * widths[kind_of[i]]]
        o = po.Oracle(105000 * os_, os_, _ofmt(fmt), desc[i][0], desc[i][1])
        o.process(iq)
        what = f"station {i} (os {os_}, {fmt}{', joined' if i >= R else ''}{', left' if i in gone else ''})"
        util.assert_frames_equal(frames[i], o.frames(), what)
        assert np.array_equal(counters[i], o.counters().astype(np.int64)), f"{what}: counters"
        checked += len(frames[i])
    assert checked > 2


def _call(g, rx, src, fr, n=None):
    L = g.L
    a = (vd.api._ReceiverEx * max(len(rx), 1))()
    for r, (cf, f, os_, fmt) in enumerate(rx):
        a[r].centerfreq, a[r].n_channels, a[r].oversample, a[r].sample_fmt = cf, len(f), os_, fmt
    s = np.ascontiguousarray(src, np.int32)
    f = np.ascontiguousarray(fr, np.uint32)
    return L.vdl2gpu_update_receivers(g.h, a, s.ctypes.data, len(rx) if n is None else n, f.ctypes.data)


def test_refusals_leave_the_context_decoding(stations):
    st, _, _ = stations
    L = vd.load_library()
    runs = []
    for refuse in (False, True):
        F = _Fleet(st, range(4))
        me = [_desc(st[i]) for i in range(4)]
        fr = [f for d in me for f in d[1]]
        for k in range(4):
            F.span({i: W - 7 * i for i in range(4)})
            if refuse and k == 1:
                assert _call(F.g, me, [0, 1, 2, 3], fr) == EINVAL                       # a span in flight
                assert "in flight" in L.vdl2gpu_last_error().decode()
            if refuse and k == 2:
                frames = F.g.flush()
                for f in frames:
                    r = F.g.receiver_of(f.channel)
                    f.channel -= F.g.channels_of(r)[0]
                    F.frames[r].append(f)
                for src, msg in (([0, 1, 2, 4], "receiver 4 of 4"), ([0, 1, 2, -2], "receiver -2 of 4"),
                                 ([0, 1, 1, 3], "which an earlier entry continues"), ([0, 1, 3, 2], "does not repeat receiver 3")):
                    assert _call(F.g, me, src, fr) == EINVAL, src
                    assert msg in L.vdl2gpu_last_error().decode()
                bad = list(fr)
                bad[0] += 1
                assert _call(F.g, me, [0, 1, 2, 3], bad) == EINVAL
                assert _call(F.g, [], [], []) == EINVAL and "no receivers" in L.vdl2gpu_last_error().decode()
                many = [(136500000, [136500000], 10, vd.FMT_U8)] * 65536
                assert _call(F.g, many, [-1] * 65536, [136500000] * 65536) == EINVAL
                assert "65535" in L.vdl2gpu_last_error().decode()
                assert _call(F.g, [(136500000, [136500000], 11, vd.FMT_U8)], [-1], [136500000]) == EINVAL
                assert "oversample 11" in L.vdl2gpu_last_error().decode()
                assert F.g.n_receivers == 4 and F.g.receiver_positions().tolist() == [F.pos[i] for i in range(4)]
        F.finish()
        runs.append(F)
    a, b = runs
    for i in range(4):
        util.assert_frames_equal(b.frames[i], [f for f in a.frames[i]], f"receiver {i} with refusals")
        assert np.array_equal(a.counters[i], b.counters[i])
        assert np.array_equal(a.dec[i].view(np.uint32), b.dec[i].view(np.uint32))
    rx = [(136975000, [136975000, 137000000], 10, vd.FMT_U8), (136500000, [136525000], 20, vd.FMT_S16)]
    fr = [136975000, 137000000, 136525000]
    for g in (vd.Vdl2MixedReceivers(rx, max_chunk_bytes=100 * 80),
              vd.Vdl2Receivers(2100000, 20, vd.FMT_U8, [(136975000, [136975000]), (136500000, [136525000])], max_chunk_bytes=4096),
              vd.Vdl2Channels(2100000, 20, vd.FMT_U8, 136975000, [136975000], max_chunk_bytes=4096)):
        assert _call(g, rx, [-1, -1], fr) == EINVAL
        assert "VDL2GPU_FLAG_RAGGED" in L.vdl2gpu_last_error().decode()
        g.close()
