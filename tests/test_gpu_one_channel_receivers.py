"""-m gpu: fleets of one-channel receivers, the most common deployment (a ground receiver listening on 136.975 MHz alone).
One channel per receiver puts up to 128 receivers in one K1 block (G = 128), where the receiver K1 kernels take shapes no
fleet of multi-channel receivers reaches: one-group tiles in k1_mix_iir_decimate_groups (T = 20 / 26 / 30 samples at
oversample 20 / 13 / 10), two-group tiles above the 110 KB shared-memory budget in the mixed and ragged kernels
(VDL2_RX_MIXED_SMEM_MAX), staged rows beyond 32 in shared memory and warp 0 issuing four bulk copies per lane.  The CPU
companion, test_one_channel_receivers.py, checks that every fleet here reaches those shapes.

Receiver r's stream is the base traffic stream of its (rate, format) kind started 7919 r units later (samples in a
single-rate context, decimation groups in a mixed one), circularly; it is tuned to its own centre.  The oracle runs once
per receiver over exactly the samples the receiver brought, and every receiver's decimated samples are compared with the
oracle's bit for bit after every chunk or span (FLAG_KEEP_DEC, read_dec), then its frames with all metadata, its counters
and, with FLAG_TRACE, its trace events."""
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth
from oracle import pyoracle as po
from tests import util
from tests.test_gpu_mixed_receivers import KINDS, _bpp, _ofmt, _ragged, _vfmt
from tests.test_gpu_restart_receivers import _expected

pytestmark = pytest.mark.gpu
SHIFT = 7919
N_FLEET = 300                                  # blocks of G = 128, 128 and 44 receivers
ON_CENTRE = (1, 130, 299)                      # channel exactly on the receiver's centre: no mixing
TILE = {20: 20, 13: 26, 10: 30}                # K1 tile of the receiver-group kernel at G = 128 (samples)
W = 3001                                       # widest span of the mixed fleets (max_chunk_bytes = W x 80)
RESTARTED = (0, 31, 32, 70, 127, 128, 200, 255, 256, 299)
IDLE_AT_RESTART = (32, 256)                    # restarted, and bring nothing to the restart span
ALONE = 71                                     # the only receiver of block 0 with samples in one ragged span
BALANCED = 16384                               # 31 or 32 channels per warp over the 528 warps of an H100
# first and last; the block boundary 127/128; warp 15/16 (the last 32-channel warp, also blocks 3/4); warp 16/17 (the first
# 31-channel warps); blocks 4/5; mid-machine
BALANCED_SAMPLE = (0, 1, 127, 128, 511, 512, 542, 543, 635, 636, 8191, 8192, 16382, 16383)


# ---- fleets ----
def one_channel_fleet(kinds_of, seconds, seed, per_group, n_slots=8, on_centre=ON_CENTRE, centre0=135000000, spacing=1000,
                      bursts_per_s=12.0):
    """receiver r: kind kinds_of[r] = (oversample, format), one channel, centre centre0 + spacing r, channel on slot
    offset r mod n_slots of its kind's base stream (on the centre for r in on_centre), stream shifted by 7919 r units.
    A unit is one decimation group (os x bytes per sample) if per_group, else one sample."""
    bases, offs = {}, None
    for os_, fmt in sorted(set(kinds_of)):
        iq, offs, _ = synth.traffic_stream(105000 * os_, seconds, n_slots, bursts_per_s, 24.0, -20.0, seed, fmt)
        b = np.ascontiguousarray(iq).view(np.uint8).reshape(-1)
        w = _bpp(fmt) * (os_ if per_group else 1)
        bases[(os_, fmt)] = b[:b.size // w * w].reshape(-1, w)
    rx = []
    for r, (os_, fmt) in enumerate(kinds_of):
        centre = centre0 + spacing * r
        rx.append(dict(os=os_, fmt=fmt, centre=centre, freqs=[centre if r in on_centre else centre + int(offs[r % n_slots])],
                       shift=(SHIFT * r) % bases[(os_, fmt)].shape[0]))
    return dict(bases=bases, rx=rx, dev={})


def host_units(F, r, a, b):
    """receiver r's units [a, b) as bytes"""
    x = F["rx"][r]
    base = F["bases"][(x["os"], x["fmt"])]
    return base[(np.arange(a, b) + x["shift"]) % base.shape[0]].reshape(-1)


def _dev_base(F, kind, device):
    import torch
    if (kind, device) not in F["dev"]:
        F["dev"][(kind, device)] = torch.from_numpy(F["bases"][kind]).to(device)
    return F["dev"][(kind, device)]


def pack_lockstep(F, a, n, device="cuda"):
    """units [a, a + n) of every receiver of a single-kind fleet, receivers back to back: uint8 [R, n, unit]"""
    import torch
    kind = (F["rx"][0]["os"], F["rx"][0]["fmt"])
    base = _dev_base(F, kind, device)
    L = base.shape[0]
    shift = torch.tensor([x["shift"] for x in F["rx"]], dtype=torch.int64, device=device)
    ar = torch.arange(a, a + n, dtype=torch.int64, device=device)
    out = torch.empty(len(F["rx"]), n, base.shape[1], dtype=torch.uint8, device=device)
    for r0 in range(0, len(F["rx"]), 512):
        out[r0:r0 + 512] = base[(ar[None, :] + shift[r0:r0 + 512, None]) % L]
    return out


def pack_span(F, counts, pos, device="cuda"):
    """counts[r] units of receiver r from pos[r] on, receivers back to back (uint8, flat)"""
    import torch
    pieces = []
    for r, n in enumerate(counts):
        if n:
            x = F["rx"][r]
            base = _dev_base(F, (x["os"], x["fmt"]), device)
            idx = (torch.arange(int(pos[r]), int(pos[r]) + int(n), dtype=torch.int64, device=device) + x["shift"]) % base.shape[0]
            pieces.append(base[idx].reshape(-1))
    return torch.cat(pieces) if pieces else torch.zeros(0, dtype=torch.uint8, device=device)


def oracle(F, r, pieces, trace=False, cuts=()):
    """receiver r's oracles over its units, fed piece by piece (pieces: unit counts); a new oracle at every cut (a unit
    index: a restart there).  Returns (oracles, bounds) as test_gpu_restart_receivers._segments does."""
    x = F["rx"][r]
    total = int(sum(pieces))
    bounds = [0] + list(cuts) + [total]
    out = []
    for k in range(len(bounds) - 1):
        o = po.Oracle(105000 * x["os"], x["os"], _ofmt(x["fmt"]), x["centre"], x["freqs"], trace=trace, dec_tap=True)
        p0 = 0
        for n in pieces:                              # the same cuts the device sees, clipped to the segment
            a, b = max(p0, bounds[k]), min(p0 + n, bounds[k + 1])
            if b > a:
                o.process(host_units(F, r, a, b))
            p0 += n
        out.append(o)
    return out, bounds


def oracle_dec(oracles):
    """the decimated samples of a receiver's segmented oracles as one stream"""
    return np.concatenate([o.dec_samples() for o in oracles])


# ---- schedules ----
def chunk_schedule(os_, n_full=3):
    """samples per chunk of a single-rate fleet: an odd count (the decimation phase and the bulk copies' `mis` shift change
    on every odd chunk), one that stays inside the head of the current decimation group (no tile, no tail), one longer than
    a group but shorter than a tile (a tile of one group at oversample 20: shorter than a group there), one that ends
    mid-group, full odd chunks and a short tail"""
    c = [65537]
    c.append(max(1, (os_ - sum(c) % os_) % os_ - 1))
    c.append(TILE[os_] - 1)
    c.append(65535 - os_ // 2)
    c += [65537] * n_full
    c.append(333)
    return c


def mixed_spans():
    """decimated samples per span of the lock-step mixed fleet: 1, 2 and 3 (fewer than and straddling the two-group tile),
    7 and 3001 (odd: the last tile of an oversample-13 row ends on a hand-copied sample), long spans and a short one"""
    return [1, 2, 3, 7, W, 2, 1, 2048, W, W, 1999]


def ragged_spans(R, seed):
    """per-span counts [span][receiver] of the ragged fleet; the restart span is RESTART_SPAN"""
    rng = np.random.default_rng(seed)
    cycle = [0, 1, 2, 3, 5, 7, W, 12]
    spans = [[W] * R]                                                               # full width
    spans.append([cycle[r % len(cycle)] if r % 9 else int(rng.integers(0, W + 1)) for r in range(R)])
    one = [int(rng.integers(1, W + 1)) for _ in range(R)]                           # block 0: one receiver brings samples
    one[:128] = [0] * 128
    one[ALONE] = 3
    spans.append(one)
    spans.append([0 if r % 7 == 0 else 2 * int(rng.integers(0, W // 2)) + 1 for r in range(R)])      # odd counts
    restart = [int(rng.integers(0, W + 1)) for _ in range(R)]
    for r in IDLE_AT_RESTART:
        restart[r] = 0
    spans.append(restart)
    spans.append([1 + k % 3 for k in range(R)])                                    # 1, 2, 3 for every receiver
    spans.append([W] * R)
    spans.append([0 if rng.random() < 0.2 else int(rng.integers(0, W + 1)) for _ in range(R)])
    for s in spans[1:4]:                                                            # absent for whole spans
        for r in range(4, R, 11):
            s[r] = 0
    return spans


RESTART_SPAN = 4


def balanced_counts(R, n_spans, width, seed):
    """jittered counts up to `width`, 10 % absent in any span; receiver 0 at full width in the first span"""
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, width + 1, (n_spans, R))
    counts[rng.random((n_spans, R)) < 0.1] = 0
    counts[0, 0] = width
    return counts


# ---- checks ----
def _rows_equal(got, want):
    return np.array_equal(np.ascontiguousarray(got).view(np.uint32), np.ascontiguousarray(want).view(np.uint32))


def check_frames(frames, first, rxs, want, what, receivers=None):
    """frames of receivers (all: None) against want[r] = (frames, counters, events or None) per receiver; channels local"""
    by_rx = {}
    starts = np.asarray(first)
    for f in frames:
        r = int(np.searchsorted(starts, f.channel, side="right")) - 1
        by_rx.setdefault(r, []).append(f)
    n = 0
    for r in (range(len(rxs)) if receivers is None else receivers):
        mine = by_rx.get(r, [])
        for f in mine:
            f.channel -= int(first[r])
        wf = want[r][0]
        util.assert_frames_equal(mine, wf, f"{what}: receiver {r}")
        assert all(f.freq == rxs[r]["freqs"][f.channel] for f in mine), f"{what}: receiver {r}: frequencies"
        n += len(mine)
    return n


# ---- 1. k1_mix_iir_decimate_groups at G = 128 ----
@pytest.mark.parametrize("os_,fmt", [(20, "u8"), (13, "u8"), (10, "s16")], ids=["os20-cu8", "os13-cu8", "os10-cs16"])
def test_groups_kernel_with_128_receivers_per_block(os_, fmt, monkeypatch):
    import torch
    F = one_channel_fleet([(os_, fmt)] * N_FLEET, 0.3, 0x4F430000 + os_, per_group=False)
    rxs, bpp = F["rx"], _bpp(fmt)
    chunks = chunk_schedule(os_)
    res = [oracle(F, r, chunks) for r in range(N_FLEET)]
    want = [_expected(*x) for x in res]
    wdec = np.stack([oracle_dec(o)[:, 0] for o, _ in res], axis=1)                 # [decimated sample][receiver][2]
    wcnt = np.concatenate([w[1] for w in want]).astype(np.uint64)
    first = list(range(N_FLEET + 1))
    legs = []
    for name, flags, k1_variant in (("graphs", 0, None), ("no_graph", vd.FLAG_NO_GRAPH, None), ("k1_variant4", 0, "4")):
        if k1_variant:                              # without the symmetric-tap form of the filter (read at create)
            monkeypatch.setenv("VDL2GPU_K1_VARIANT", k1_variant)
        g = vd.Vdl2Receivers(105000 * os_, os_, _vfmt(fmt), [(x["centre"], x["freqs"]) for x in rxs],
                             max_chunk_bytes=max(chunks) * bpp, flags=flags | vd.FLAG_KEEP_DEC)
        st = torch.cuda.current_stream()
        decs, s0 = [], 0
        for k, n in enumerate(chunks):
            buf = pack_lockstep(F, s0, n)
            g.submit_device(buf.data_ptr(), n * bpp, st.cuda_stream)
            dec = g.read_dec(n // os_ + 2)
            d0, d1 = s0 // os_, (s0 + n) // os_
            assert dec.shape == (d1 - d0, N_FLEET, 2), f"{name}: chunk {k}"
            if not _rows_equal(dec, wdec[d0:d1]):
                bad = [r for r in range(N_FLEET) if not _rows_equal(dec[:, r], wdec[d0:d1, r])]
                raise AssertionError(f"os {os_} {fmt} {name}: chunk {k} ({n} samples): decimated samples differ for receivers {bad}")
            decs.append(dec)
            s0 += n
            del buf
        frames = g.flush()
        stats, cnt = g.stats(), g.channel_counters()
        g.close()
        assert stats["pool_overflows"] == 0 and stats["out_overflows"] == 0
        assert (stats["graph_launches"] > 0) == (not flags & vd.FLAG_NO_GRAPH)
        assert np.array_equal(cnt, wcnt), f"{name}: counters"
        tuples = sorted(util.frame_tuple(f) for f in frames)
        assert check_frames(frames, first, rxs, want, f"os {os_} {fmt} {name}") > 100
        legs.append((tuples, cnt, decs))
    for tuples, cnt, decs in legs[1:]:              # the three legs agree with each other
        assert tuples == legs[0][0] and np.array_equal(cnt, legs[0][1])
        assert all(_rows_equal(a, b) for a, b in zip(decs, legs[0][2]))


# ---- 2. k1_mix_iir_decimate_mixed with two-group tiles above the budget ----
@pytest.fixture(scope="module")
def mixed_fleet():
    F = one_channel_fleet([KINDS[r % len(KINDS)] for r in range(N_FLEET)], 0.3, 0x4F4D0000, per_group=True)
    return F


@pytest.mark.parametrize("order", ["interleaved", "grouped"])
def test_mixed_kernel_over_the_shared_memory_budget(mixed_fleet, order):
    """every warp runs all three rate arms (interleaved), or every warp but those at a rate boundary runs one (grouped)"""
    import torch
    F = dict(mixed_fleet)
    if order == "grouped":
        F["rx"] = sorted(F["rx"], key=lambda x: (x["os"], x["fmt"]))
    rxs = F["rx"]
    spans = mixed_spans()
    res = [oracle(F, r, spans) for r in range(N_FLEET)]
    want = [_expected(*x) for x in res]
    wdec = np.stack([oracle_dec(o)[:, 0] for o, _ in res], axis=1)
    g = vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"])) for x in rxs], max_chunk_bytes=W * 80,
                              flags=vd.FLAG_KEEP_DEC)
    st = torch.cuda.current_stream()
    d0 = 0
    for k, n in enumerate(spans):
        buf = pack_span(F, [n] * N_FLEET, [d0] * N_FLEET)
        assert buf.numel() == n * sum(x["os"] * _bpp(x["fmt"]) for x in rxs)
        g.submit_span_device(buf.data_ptr(), n, st.cuda_stream)
        dec = g.read_dec(W + 2)
        assert dec.shape == (n, N_FLEET, 2)
        if not _rows_equal(dec, wdec[d0:d0 + n]):
            bad = [r for r in range(N_FLEET) if not _rows_equal(dec[:, r], wdec[d0:d0 + n, r])]
            raise AssertionError(f"{order}: span {k} (n_dec {n}): decimated samples differ for receivers {bad}")
        d0 += n
        del buf
    frames = g.flush()
    stats, cnt = g.stats(), g.channel_counters()
    g.close()
    assert stats["pool_overflows"] == 0 and stats["out_overflows"] == 0
    assert stats["iq_samples"] == sum(spans) * sum(x["os"] for x in rxs)
    assert np.array_equal(cnt, np.concatenate([w[1] for w in want]).astype(np.uint64)), f"{order}: counters"
    assert check_frames(frames, list(range(N_FLEET + 1)), rxs, want, order) > 100


# ---- 3. k1_mix_iir_decimate_ragged, same fleet, with restarts ----
@pytest.fixture(scope="module")
def ragged_fleet(mixed_fleet):
    F = mixed_fleet
    spans = ragged_spans(N_FLEET, 0x4F52)
    per_rx = [[s[r] for s in spans] for r in range(N_FLEET)]
    cut = {r: sum(per_rx[r][:RESTART_SPAN]) for r in RESTARTED}
    res = [oracle(F, r, per_rx[r], trace=True, cuts=[cut[r]] if r in cut else []) for r in range(N_FLEET)]
    return F, spans, res


@pytest.mark.parametrize("flags", [0, vd.FLAG_TRACE | vd.FLAG_NO_GRAPH], ids=["graphs", "trace_no_graph"])
def test_ragged_kernel_over_the_shared_memory_budget(ragged_fleet, flags):
    import torch
    F, spans, res = ragged_fleet
    rxs = F["rx"]
    want = [_expected(*x) for x in res]
    wdec = [oracle_dec(o) for o, _ in res]
    g = vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"])) for x in rxs], max_chunk_bytes=W * 80,
                              flags=flags | vd.FLAG_KEEP_DEC, ragged=True)
    st = torch.cuda.current_stream()
    pos = np.zeros(N_FLEET, np.int64)
    for k, c in enumerate(spans):
        if k == RESTART_SPAN:
            for r in RESTARTED:
                g.restart_receiver(r)
        buf = pack_span(F, c, pos)
        g.submit_ragged_device(buf.data_ptr(), c, st.cuda_stream)
        dec = g.read_dec(W + 2)
        assert dec.shape[0] == max(c), f"span {k}"
        bad = [r for r in range(N_FLEET) if not _rows_equal(dec[:c[r], r], wdec[r][pos[r]:pos[r] + c[r], 0])]
        assert not bad, f"flags {flags}: span {k}: decimated samples differ for receivers {bad}"
        pos += c
        del buf
    frames = g.flush()
    stats, cnt = g.stats(), g.channel_counters()
    events = g.read_events(1 << 20) if flags & vd.FLAG_TRACE else None
    assert g.receiver_positions().tolist() == pos.tolist()
    g.close()
    assert stats["pool_overflows"] == 0 and stats["out_overflows"] == 0
    assert stats["dec_samples"] == sum(max(c) for c in spans)
    for r in range(N_FLEET):
        assert np.array_equal(cnt[r:r + 1].astype(np.int64), want[r][1].astype(np.int64)), f"flags {flags}: receiver {r}: counters"
    assert check_frames(frames, list(range(N_FLEET + 1)), rxs, want, f"ragged, flags {flags}") > 100
    if events is not None:
        by_rx = {}
        for e in events:
            by_rx.setdefault(e["channel"], []).append(dict(e, channel=0))
        for r in range(N_FLEET):
            util.assert_events_equal(by_rx.get(r, []), want[r][2], f"receiver {r}: events")


# ---- 4. the balanced mapping: 16384 one-channel receivers ----
def _check_sampled(F, pieces_of, decs, frames, cnt, what):
    """receivers of BALANCED_SAMPLE against their oracles (pieces_of(r): the units receiver r brought, span by span):
    decimated samples of every span (decs[k] = (dec, n, d0): rows dec[:n[r], r] are its samples d0[r] on), frames and
    counters; then frames and counters of eight more receivers spread over those that decoded something (their decimated
    samples are not kept).  Returns the frames checked."""
    rxs = F["rx"]
    by_rx = {}
    for f in frames:
        by_rx.setdefault(f.channel, []).append(f)
    busy = sorted(set(by_rx) - set(BALANCED_SAMPLE))
    checked = 0
    for r in BALANCED_SAMPLE + tuple(busy[::max(1, len(busy) // 8)][:8]):
        (o,), _ = oracle(F, r, pieces_of(r))
        if r in BALANCED_SAMPLE:
            wd = o.dec_samples()
            d = 0
            for k, (dec, n, d0) in enumerate(decs):
                n_r, d_r = n[r], d0[r]
                assert _rows_equal(dec[:n_r, r], wd[d_r:d_r + n_r, 0]), \
                    f"{what}: receiver {r} (os {rxs[r]['os']}): span {k}: decimated samples"
                d += n_r
            assert d == wd.shape[0]
        mine = by_rx.get(r, [])
        for f in mine:
            f.channel = 0
        util.assert_frames_equal(mine, o.frames(), f"{what}: receiver {r}")
        assert all(f.freq == rxs[r]["freqs"][0] for f in mine)
        assert np.array_equal(cnt[r:r + 1], o.counters()), f"{what}: receiver {r}: counters"
        checked += len(mine)
    return checked


def test_16384_one_channel_receivers_on_the_balanced_mapping():
    import torch
    os_, R = 20, BALANCED
    F = one_channel_fleet([(os_, "u8")] * R, 0.3, 0x4F420000, per_group=False, on_centre=(0,), bursts_per_s=30.0)
    chunks = [32769, 32767, 32768, 32768]
    g = vd.Vdl2Receivers(105000 * os_, os_, vd.FMT_U8, [(x["centre"], x["freqs"]) for x in F["rx"]],
                         max_chunk_bytes=2 * max(chunks), flags=vd.FLAG_KEEP_DEC)
    st = torch.cuda.current_stream()
    decs, s0 = [], 0
    for n in chunks:
        buf = pack_lockstep(F, s0, n)
        g.submit_device(buf.data_ptr(), 2 * n, st.cuda_stream)
        dec = g.read_dec(n // os_ + 2)
        d0, d1 = s0 // os_, (s0 + n) // os_
        assert dec.shape == (d1 - d0, R, 2)
        decs.append((dec[:, list(BALANCED_SAMPLE)], {r: d1 - d0 for r in BALANCED_SAMPLE}, {r: d0 for r in BALANCED_SAMPLE}))
        s0 += n
        del buf, dec
    frames = g.flush()
    stats, cnt = g.stats(), g.channel_counters()
    g.close()
    assert stats["pool_overflows"] == 0 and stats["out_overflows"] == 0 and stats["msg_good"] > R // 8
    # decs hold the sampled columns only: index them by position in BALANCED_SAMPLE
    col = {r: k for k, r in enumerate(BALANCED_SAMPLE)}
    decs = [(_Cols(d, col), n, d0) for d, n, d0 in decs]
    assert _check_sampled(F, lambda r: chunks, decs, frames, cnt, "16384 x 1, os 20") >= 8


class _Cols:
    """dec[:n, r] of a column subset, by receiver number"""

    def __init__(self, a, col):
        self.a, self.col = a, col

    def __getitem__(self, key):
        rows, r = key
        return self.a[rows, self.col[r]]


def test_16384_alternating_rate_receivers_with_ragged_spans_on_the_balanced_mapping():
    import torch
    R, n_spans, width = BALANCED, 4, 2000
    kinds = [(10, "u8"), (20, "s16")]
    F = one_channel_fleet([kinds[r % 2] for r in range(R)], 0.3, 0x4F470000, per_group=True, on_centre=(0,), bursts_per_s=30.0)
    counts = balanced_counts(R, n_spans, width, 0x4F47)
    g = vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"])) for x in F["rx"]], max_chunk_bytes=width * 80,
                              flags=vd.FLAG_KEEP_DEC, ragged=True)
    st = torch.cuda.current_stream()
    pos = np.zeros(R, np.int64)
    decs = []
    col = {r: k for k, r in enumerate(BALANCED_SAMPLE)}
    for s in range(n_spans):
        buf = pack_span(F, counts[s], pos)
        g.submit_ragged_device(buf.data_ptr(), counts[s], st.cuda_stream)
        dec = g.read_dec(width + 2)
        assert dec.shape == (counts[s].max(), R, 2)
        decs.append((_Cols(dec[:, list(BALANCED_SAMPLE)], col), counts[s], pos.copy()))
        pos += counts[s]
        del buf, dec
    frames = g.flush()
    stats, cnt = g.stats(), g.channel_counters()
    assert g.receiver_positions().tolist() == pos.tolist()
    g.close()
    assert stats["pool_overflows"] == 0 and stats["out_overflows"] == 0 and stats["msg_good"] > R // 32
    assert _check_sampled(F, lambda r: [int(c) for c in counts[:, r]], decs, frames, cnt, "16384 x 1 ragged, os 10 cu8 / os 20 cs16") >= 8


# ---- 5. one-channel receivers joining a ragged fleet of multi-channel receivers ----
def test_one_channel_receivers_join_a_ragged_fleet():
    """the nine receivers of test_gpu_mixed_receivers.py (1 to 40 channels, a multi-group tile) run two spans; then 200
    one-channel receivers join, 100 in front of them and 100 behind, and two of them leave: the K1 tile becomes two
    groups over the budget.  Kept receivers continue against an oracle over their whole stream, new ones against an
    oracle started at the join, removed ones against one over what they brought."""
    old, _ = _ragged(0.2, 0x4F4A0000)
    new = one_channel_fleet([KINDS[r % len(KINDS)] for r in range(200)], 0.3, 0x4F4A0100, per_group=True,
                            centre0=136000000, spacing=2500, bursts_per_s=30.0)
    n_after = 3
    for r, x in enumerate(new["rx"]):                 # host buffers, as the multi-channel stations have
        x["buf"] = host_units(new, r, 0, n_after * W)
    st = old + new["rx"]                              # station ids: 0..8 the old fleet, 9..208 the new receivers
    members = list(range(9))
    g = vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"])) for x in old], max_chunk_bytes=W * 80,
                              flags=vd.FLAG_KEEP_DEC, ragged=True)
    pos = {i: 0 for i in range(len(st))}
    record = []                                       # per span: {station: (dec rows, decimated samples before)}
    frames = {i: [] for i in range(len(st))}
    counters = {}
    rng = np.random.default_rng(0x4F4A)

    def w_of(i):
        return st[i]["os"] * _bpp(st[i]["fmt"])

    def span(counts):
        bufs = [st[i]["buf"][pos[i] * w_of(i):(pos[i] + counts[i]) * w_of(i)] for i in members]
        g.submit_ragged(bufs)
        dec = g.read_dec(W + 2)
        record.append({i: (dec[:counts[i], g.channels_of(k)[0]:g.channels_of(k)[-1] + 1].copy(), pos[i]) for k, i in enumerate(members)})
        for i in members:
            pos[i] += counts[i]

    def drain():
        for f in g.flush():
            k = g.receiver_of(f.channel)
            f.channel -= g.channels_of(k)[0]
            frames[members[k]].append(f)
        cnt = g.channel_counters()
        return {i: cnt[g.channels_of(k)[0]:g.channels_of(k)[-1] + 1] for k, i in enumerate(members)}

    span({i: W for i in members})
    span({i: int(rng.integers(W // 2, W + 1)) for i in members})
    cnt = drain()
    joined = list(range(9, 209))
    gone = (3, 7)
    for i in gone:
        counters[i] = cnt[i]
    kept = [i for i in members if i not in gone]
    new_members = joined[:100] + kept + joined[100:]
    old_index = {i: k for k, i in enumerate(members)}
    g.update_receivers([(st[i]["centre"], st[i]["freqs"], st[i]["os"], _vfmt(st[i]["fmt"])) for i in new_members],
                       [old_index.get(i, -1) for i in new_members])
    members = new_members
    assert g.receiver_positions().tolist() == [pos[i] for i in members]
    span({i: W for i in members})
    span({i: 0 if i % 10 == 3 else int(rng.integers(0, W + 1)) for i in members})
    span({i: 1 + i % 3 for i in members})
    cnt = drain()
    counters.update(cnt)
    stats = g.stats()
    g.close()
    assert stats["pool_overflows"] == 0 and stats["out_overflows"] == 0
    n = 0
    for i in range(len(st)):
        x = st[i]
        o = po.Oracle(105000 * x["os"], x["os"], _ofmt(x["fmt"]), x["centre"], x["freqs"], dec_tap=True)
        o.process(x["buf"][:pos[i] * w_of(i)])
        what = f"station {i} (os {x['os']}, {x['fmt']}, {len(x['freqs'])} channels)"
        wd = o.dec_samples()
        assert wd.shape[0] == pos[i]
        for k, rec in enumerate(record):
            if i in rec:
                d, d0 = rec[i]
                assert _rows_equal(d, wd[d0:d0 + d.shape[0]]), f"{what}: span {k}: decimated samples"
        util.assert_frames_equal(frames[i], o.frames(), what)
        assert all(f.freq == x["freqs"][f.channel] for f in frames[i])
        assert np.array_equal(counters[i], o.counters()), f"{what}: counters"
        n += len(frames[i])
    assert n > 40


# ---- 6. the lanes kernel (one stream per channel) and the same streams as one-channel receivers ----
def _lanes_chunks(os_):
    return [65537, 2, 65535, 65536 + os_ // 2, 65537, 65537, 333]


@pytest.mark.parametrize("os_", [20, 10])
def test_lanes_kernel_decimated_samples_equal_the_receivers_form(os_):
    """40 streams, one channel each (24 lanes of the second warp idle): through k1_mix_iir_decimate_lanes (n_streams ==
    n_channels, one centre) and through k1_mix_iir_decimate_groups (40 one-channel receivers on that centre)"""
    S, centre = 40, 136975000
    F = one_channel_fleet([(os_, "u8")] * S, 0.3, 0x4F4C0000 + os_, per_group=False, on_centre=(3,), centre0=centre, spacing=0)
    chunks = _lanes_chunks(os_)
    res = [oracle(F, s, chunks) for s in range(S)]
    wdec = np.stack([oracle_dec(o)[:, 0] for o, _ in res], axis=1)
    want = [_expected(*x) for x in res]
    freqs = [x["freqs"][0] for x in F["rx"]]
    lanes = vd.Vdl2Channels(105000 * os_, os_, vd.FMT_U8, centre, freqs, max_chunk_bytes=2 * max(chunks), n_streams=S,
                            flags=vd.FLAG_KEEP_DEC)
    rx = vd.Vdl2Receivers(105000 * os_, os_, vd.FMT_U8, [(centre, [f]) for f in freqs], max_chunk_bytes=2 * max(chunks),
                          flags=vd.FLAG_KEEP_DEC)
    s0 = 0
    for k, n in enumerate(chunks):
        parts = [host_units(F, s, s0, s0 + n) for s in range(S)]
        lanes.submit(np.concatenate(parts))
        rx.submit(parts)
        da, db = lanes.read_dec(n // os_ + 2), rx.read_dec(n // os_ + 2)
        d0, d1 = s0 // os_, (s0 + n) // os_
        assert da.shape == db.shape == (d1 - d0, S, 2)
        bad = [s for s in range(S) if not _rows_equal(da[:, s], wdec[d0:d1, s])]
        assert not bad, f"os {os_}: chunk {k}: the lanes kernel's decimated samples differ for streams {bad}"
        assert _rows_equal(db, da), f"os {os_}: chunk {k}: the receivers form differs from the lanes form"
        s0 += n
    fa, fb = lanes.flush(), rx.flush()
    ca, cb = lanes.channel_counters(), rx.channel_counters()
    for g in (lanes, rx):
        st = g.stats()
        assert st["pool_overflows"] == 0 and st["out_overflows"] == 0
        g.close()
    assert sorted(util.frame_tuple(f) for f in fa) == sorted(util.frame_tuple(f) for f in fb)
    assert np.array_equal(ca, cb)
    assert np.array_equal(ca, np.concatenate([w[1] for w in want]).astype(np.uint64))
    assert check_frames(fa, list(range(S + 1)), F["rx"], want, f"lanes os {os_}") > 10


def test_lanes_kernel_decimated_samples_on_the_balanced_mapping():
    """9600 streams x 1 channel (17 or 18 per warp over all 528 warps): K0 places stream c in column slot(c); the
    decimated samples of sampled streams are checked after every chunk"""
    import torch
    S, centre, os_ = 9600, 136975000, 20
    F = one_channel_fleet([(os_, "u8")] * S, 0.3, 0x4F4C0100, per_group=False, on_centre=(), centre0=centre, spacing=0,
                          bursts_per_s=30.0)
    chunks = [65537, 65535, 65536]
    sample = (0, 1, 16, 17, 31, 32, 4799, 4800, 9215, 9216, 9599)
    g = vd.Vdl2Channels(105000 * os_, os_, vd.FMT_U8, centre, [x["freqs"][0] for x in F["rx"]], max_chunk_bytes=2 * max(chunks),
                        n_streams=S, flags=vd.FLAG_KEEP_DEC)
    st = torch.cuda.current_stream()
    res = {s: oracle(F, s, chunks)[0][0] for s in sample}
    s0 = 0
    for k, n in enumerate(chunks):
        buf = pack_lockstep(F, s0, n)
        g.submit_device(buf.data_ptr(), 2 * n, st.cuda_stream)
        dec = g.read_dec(n // os_ + 2)
        d0, d1 = s0 // os_, (s0 + n) // os_
        assert dec.shape == (d1 - d0, S, 2)
        for s in sample:
            assert _rows_equal(dec[:, s], res[s].dec_samples()[d0:d1, 0]), f"stream {s}: chunk {k}: decimated samples"
        s0 += n
        del buf, dec
    got = g.flush()
    cnt = g.channel_counters()
    g.close()
    checked = 0
    for s in sample:
        mine = [f for f in got if f.channel == s]
        for f in mine:
            f.channel = 0
        util.assert_frames_equal(mine, res[s].frames(), f"stream {s}")
        assert np.array_equal(cnt[s:s + 1], res[s].counters())
        checked += len(mine)
    assert checked > 2
