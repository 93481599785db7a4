"""-m gpu: receivers of different sample rates and formats in one context (vdl2gpu_create_mixed_receivers /
Vdl2MixedReceivers).  Every receiver must decode exactly what one reference process at its own rate, in its own format,
tuned to its own centre decodes from its own IQ stream: the oracle is run per receiver (po.Oracle(105000 os_r, os_r,
fmt_r, centre_r, freqs_r)), fed n_dec x os_r x bytes-per-sample_r bytes at a time, and compared frame for frame, counter
for counter and, for the last span, decimated sample for decimated sample."""
import ctypes as C
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth
from oracle import pyoracle as po
from tests import util

pytestmark = pytest.mark.gpu
EINVAL, ETOOBIG = -1, -5
SIZES = [1, 3, 8, 13, 32, 33, 40, 5, 17]       # 152 channels: blocks and warps straddle receivers (and rates)
KINDS = [(10, "u8"), (20, "s16"), (13, "u8"), (20, "u8"), (10, "s16")]
N_DEC = 3001                                   # odd: the last tile of every span ends on an odd sample at oversample 13


def _bpp(fmt):
    return 4 if fmt == "s16" else 2


def _vfmt(fmt):
    return vd.FMT_S16 if fmt == "s16" else vd.FMT_U8


def _ofmt(fmt):
    return po.FMT_S16 if fmt == "s16" else po.FMT_U8


def _ragged(seconds, seed):
    """receiver r: SIZES[r] channels, rate and format KINDS[r % 5], its own traffic, its own centre; all streams cut to the
    same number of decimated samples"""
    out = []
    for r, n in enumerate(SIZES):
        os_, fmt = KINDS[r % len(KINDS)]
        iq, offs, _ = synth.traffic_stream(105000 * os_, seconds, n + n % 2, 6.0, 24.0, -20.0, seed + 17 * r, fmt)
        centre = 136100000 + 125000 * r
        freqs = [centre + int(o) for o in offs[:n]]
        if r == 1:
            freqs[0] = centre
        out.append(dict(centre=centre, freqs=freqs, os=os_, fmt=fmt, buf=np.ascontiguousarray(iq).view(np.uint8).reshape(-1)))
    n_dec = min(x["buf"].size // (x["os"] * _bpp(x["fmt"])) for x in out)
    for x in out:
        x["buf"] = x["buf"][:n_dec * x["os"] * _bpp(x["fmt"])]
    return out, n_dec


def _oracle(x, n_dec):
    o = po.Oracle(105000 * x["os"], x["os"], _ofmt(x["fmt"]), x["centre"], x["freqs"], dec_tap=True)
    o.process_chunked(x["buf"], n_dec * x["os"] * _bpp(x["fmt"]))
    return o.frames(), o.counters(), o.dec_samples()


def _local(frames, first):
    for f in frames:
        f.channel -= first
    return frames


def _run_mixed(rxs, flags):
    g = vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"])) for x in rxs],
                              max_chunk_bytes=N_DEC * 80, flags=flags)
    g.process_chunked([x["buf"] for x in rxs], N_DEC)
    frames = g.flush()
    dec = g.read_dec(N_DEC + 2)
    st, cnt = g.stats(), g.channel_counters()
    assert st["pool_overflows"] == 0 and st["out_overflows"] == 0
    assert (st["graph_launches"] > 0) == (not flags & vd.FLAG_NO_GRAPH)
    assert st["iq_samples"] == sum(x["buf"].size // _bpp(x["fmt"]) for x in rxs)
    g.close()
    return frames, cnt, dec


@pytest.mark.parametrize("order", ["interleaved", "grouped"])
def test_ragged_mixed_receivers_match_the_oracle_per_receiver(order):
    rxs, total = _ragged(0.3, 0x4D580000)
    assert total % N_DEC != 0 and total > 3 * N_DEC                  # a few spans, then a short last span
    if order == "grouped":
        rxs = sorted(rxs, key=lambda x: (x["os"], x["fmt"]))         # stable: every warp on one rate but at the boundaries
    want = [_oracle(x, N_DEC) for x in rxs]
    first = np.concatenate([[0], np.cumsum([len(x["freqs"]) for x in rxs])])
    results = []
    for flags in (vd.FLAG_KEEP_DEC, vd.FLAG_KEEP_DEC | vd.FLAG_NO_GRAPH):
        frames, cnt, dec = _run_mixed(rxs, flags)
        assert dec.shape[0] == total % N_DEC
        n = 0
        for r, (wf, wc, wd) in enumerate(want):
            chans = range(int(first[r]), int(first[r + 1]))
            what = f"receiver {r} (os {rxs[r]['os']}, {rxs[r]['fmt']}, {order}, flags {flags})"
            mine = _local([f for f in frames if f.channel in chans], chans[0])
            util.assert_frames_equal(mine, wf, what)
            assert all(f.freq == rxs[r]["freqs"][f.channel] for f in mine)
            assert np.array_equal(cnt[chans[0]:chans[-1] + 1], wc), f"{what}: counters"
            assert np.array_equal(dec[:, chans[0]:chans[-1] + 1].view(np.uint32), wd[-dec.shape[0]:].view(np.uint32)), \
                f"{what}: decimated samples of the last span"
            n += len(mine)
        assert n > 40
        results.append((frames, cnt, dec))
    (fa, ca, da), (fb, cb, db) = results
    assert sorted(util.frame_tuple(f) for f in fa) == sorted(util.frame_tuple(f) for f in fb)
    assert np.array_equal(ca, cb) and np.array_equal(da.view(np.uint32), db.view(np.uint32))


@pytest.mark.parametrize("os_,fmt", [(20, "u8"), (10, "s16")])
def test_uniform_mix_equals_the_receivers_context(os_, fmt):
    """all receivers of one rate and format: a mixed context fed spans equals vdl2gpu_create_receivers fed the same bytes"""
    bpp, n_dec = _bpp(fmt), 2048
    streams, rx = [], []
    for r, n in enumerate([3, 8, 32, 1, 20]):
        iq, offs, _ = synth.traffic_stream(105000 * os_, 0.25, n + n % 2, 6.0, 24.0, -20.0, 0x4D580100 + r, fmt)
        centre = 136300000 + 100000 * r
        rx.append((centre, [centre + int(o) for o in offs[:n]]))
        streams.append(np.ascontiguousarray(iq).view(np.uint8).reshape(-1))
    m = min(s.size for s in streams) // (os_ * bpp) * (os_ * bpp)
    streams = [s[:m] for s in streams]
    a = vd.Vdl2Receivers(105000 * os_, os_, _vfmt(fmt), rx, max_chunk_bytes=n_dec * os_ * bpp, flags=vd.FLAG_KEEP_DEC)
    a.process_chunked(streams, n_dec * os_ * bpp)
    fa, ca, da = a.flush(), a.channel_counters(), a.read_dec(n_dec + 2)
    a.close()
    b = vd.Vdl2MixedReceivers([(c, f, os_, _vfmt(fmt)) for c, f in rx], max_chunk_bytes=n_dec * os_ * bpp, flags=vd.FLAG_KEEP_DEC)
    b.process_chunked(streams, n_dec)
    fb, cb, db = b.flush(), b.channel_counters(), b.read_dec(n_dec + 2)
    b.close()
    assert len(fa) > 20
    util.assert_frames_equal(fb, fa, f"uniform mix ({os_}, {fmt}) vs receivers context")
    assert np.array_equal(ca, cb)
    assert da.shape[0] > 0 and np.array_equal(da.view(np.uint32), db.view(np.uint32))


def test_2048_alternating_rate_receivers_on_the_balanced_mapping():
    """16384 channels = 2048 receivers x 8, rates alternating (10, cu8) / (20, cs16) receiver by receiver, so nearly every
    K1 warp runs two arms.  Receiver r is its class's base stream started 7919 r decimated samples later, tuned to its own
    centre; the spans are built on the device and fed through submit_span_device."""
    import torch
    R, n_dec, n_spans = 2048, 4000, 3
    kinds = [(10, "u8"), (20, "s16")]
    bases, offs = [], None
    for os_, fmt in kinds:
        iq, offs, _ = synth.traffic_stream(105000 * os_, 0.3, 8, 12.0, 24.0, -20.0, 0x4D580200, fmt)
        bases.append(np.ascontiguousarray(iq).view(np.uint8).reshape(-1))
    L = min(b.size // (os_ * _bpp(fmt)) for b, (os_, fmt) in zip(bases, kinds))          # decimated samples per base
    ar = torch.arange(n_spans * n_dec, device="cuda", dtype=torch.int64)
    widths = [os_ * _bpp(fmt) for os_, fmt in kinds]                                      # bytes per decimated sample
    per_pair = n_dec * sum(widths)
    raw = torch.empty(n_spans, R // 2, per_pair, dtype=torch.uint8, device="cuda")
    for k, (os_, fmt) in enumerate(kinds):
        b = torch.from_numpy(bases[k][:L * widths[k]].reshape(L, widths[k])).cuda()
        col = 0 if k == 0 else n_dec * widths[0]
        for p0 in range(0, R // 2, 128):
            r = 2 * torch.arange(p0, p0 + 128, device="cuda", dtype=torch.int64) + k
            blk = b[(ar[None, :] + (r[:, None] * 7919) % L) % L]                            # [128, n_spans x n_dec, width]
            for s in range(n_spans):
                raw[s, p0:p0 + 128, col:col + n_dec * widths[k]] = blk[:, s * n_dec:(s + 1) * n_dec].reshape(128, -1)
    centres = [135000000 + 1000 * r for r in range(R)]
    rx = [(centres[r], [centres[r] + int(o) for o in offs], *[(10, vd.FMT_U8), (20, vd.FMT_S16)][r % 2]) for r in range(R)]
    g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=n_dec * 80)
    st = torch.cuda.current_stream()
    for s in range(n_spans):
        g.submit_span_device(raw[s].data_ptr(), n_dec, st.cuda_stream)
    got = {}
    for f in g.flush():
        got.setdefault(g.receiver_of(f.channel), []).append(f)
    stats, cnt = g.stats(), g.channel_counters()
    g.close()
    assert stats["pool_overflows"] == 0 and stats["out_overflows"] == 0
    assert stats["msg_good"] > R // 4
    checked = 0
    # first and last; 63/64: block boundary after the four 32-channel blocks; 67: straddles warps 16/17; 79: straddles
    # blocks 4/5; 1023/1024: mid-machine; every pair covers both rate classes
    for r in (0, 1, 63, 64, 67, 79, 80, 1023, 1024, 2046, 2047):
        k = r % 2
        os_, fmt = kinds[k]
        sh = (7919 * r) % L
        iq = np.roll(bases[k][:L * widths[k]], -sh * widths[k])[:n_spans * n_dec * widths[k]]
        o = po.Oracle(105000 * os_, os_, _ofmt(fmt), centres[r], rx[r][1])
        o.process_chunked(iq, n_dec * widths[k])
        mine = _local(got.get(r, []), 8 * r)
        util.assert_frames_equal(mine, o.frames(), f"receiver {r} (os {os_}, {fmt})")
        assert all(f.freq == rx[r][1][f.channel] for f in mine)
        assert np.array_equal(cnt[8 * r:8 * r + 8], o.counters()), f"receiver {r}: counters"
        checked += len(mine)
    assert checked > 2


def test_live_context_errors():
    L = vd.load_library()
    rx = [(136975000, [136975000, 137000000], 10, vd.FMT_U8), (136500000, [136525000], 20, vd.FMT_S16)]
    g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=100 * 80)
    buf = np.zeros(101 * (20 + 80), np.uint8)
    assert L.vdl2gpu_submit(g.h, buf.ctypes.data, 2000) == EINVAL
    assert "vdl2gpu_submit_span" in L.vdl2gpu_last_error().decode()
    assert L.vdl2gpu_submit_device(g.h, C.c_void_p(1), 2000, None) == EINVAL
    assert L.vdl2gpu_submit_planar_s16(g.h, buf.ctypes.data, buf.ctypes.data, 100) == EINVAL
    assert L.vdl2gpu_submit_span(g.h, buf.ctypes.data, 101) == ETOOBIG
    assert L.vdl2gpu_submit_span(g.h, buf.ctypes.data, 0) == 0
    assert L.vdl2gpu_submit_span(g.h, buf.ctypes.data, 100) == 0
    assert L.vdl2gpu_get_tables(g.h, *[None] * 8) == EINVAL
    with pytest.raises(vd.Vdl2GpuError, match="submit_span"):
        g.submit([buf, buf])
    with pytest.raises(vd.Vdl2GpuError, match="receiver 1"):
        g.submit_span([np.zeros(2 * 10 * 5, np.uint8), np.zeros(4 * 20 * 4, np.uint8)])
    g.flush()
    assert g.stats()["iq_samples"] == 100 * 30
    g.close()
    f = vd.Vdl2Channels(2100000, 20, vd.FMT_U8, 136975000, [136975000], max_chunk_bytes=4096)
    assert L.vdl2gpu_submit_span(f.h, buf.ctypes.data, 10) == EINVAL
    assert L.vdl2gpu_submit_span_device(f.h, C.c_void_p(1), 10, None) == EINVAL
    f.close()
    s = vd.Vdl2Channels(2100000, 20, vd.FMT_U8, 136975000, [136975000 + 25000 * k for k in range(64)], max_chunk_bytes=4096, n_streams=2)
    assert L.vdl2gpu_submit_span(s.h, buf.ctypes.data, 10) == EINVAL
    s.close()
