"""-m gpu: many receivers in one context (vdl2gpu_create_receivers / Vdl2Receivers).  Every receiver must decode exactly
what one reference process tuned to its own centre frequency decodes from its own IQ stream: the oracle is run per
receiver (po.Oracle(fs, os, fmt, centre_r, freqs_r)) and compared frame for frame, counter for counter and, for the last
chunk, decimated sample for decimated sample."""
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth
from oracle import pyoracle as po
from tests import cases, util

pytestmark = pytest.mark.gpu
SIZES = [1, 3, 8, 13, 32, 33, 40]          # 130 channels: blocks and warps straddle receivers


def _receivers(fs, fmt, seconds, seed):
    """one traffic stream per receiver (its own seed), each receiver tuned to its own centre; receiver 1's first channel
    sits exactly on its centre"""
    out = []
    for r, n in enumerate(SIZES):
        iq, offs, _ = synth.traffic_stream(fs, seconds, n + n % 2, 6.0, 24.0, -20.0, seed + 17 * r, fmt)   # (slots come in pairs)
        centre = 136100000 + 125000 * r
        freqs = [centre + int(o) for o in offs[:n]]
        if r == 1:
            freqs[0] = centre
        out.append((centre, freqs, np.ascontiguousarray(iq).view(np.uint8).reshape(-1)))
    n = min(b.size for _, _, b in out)
    return [(c, f, b[:n]) for c, f, b in out]


def _local(frames, first):
    for f in frames:
        f.channel -= first
    return frames


@pytest.mark.parametrize("fmt,os_", [("u8", 20), ("s16", 10), ("u8", 13)])
def test_ragged_receivers_match_the_oracle_per_receiver(fmt, os_, monkeypatch):
    fs = 105000 * os_
    bpp = 4 if fmt == "s16" else 2
    rxs = _receivers(fs, fmt, 0.3, 0x52580000 + os_)
    chunk = (65536 + 7) * bpp                    # odd number of samples: the decimation phase moves on every chunk
    assert rxs[0][2].size % chunk != 0           # ... and the stream ends with a short tail chunk
    ofmt = po.FMT_S16 if fmt == "s16" else po.FMT_U8
    want = []
    for centre, freqs, b in rxs:
        o = po.Oracle(fs, os_, ofmt, centre, freqs, dec_tap=True)
        o.process_chunked(b, chunk)
        want.append((o.frames(), o.counters(), o.dec_samples()))
    results = []
    # the last leg without the symmetric-tap form of the filter (VDL2GPU_K1_VARIANT=4, read at create)
    for flags, k1_variant in ((vd.FLAG_KEEP_DEC, None), (vd.FLAG_KEEP_DEC | vd.FLAG_NO_GRAPH, None), (vd.FLAG_KEEP_DEC, "4")):
        if k1_variant:
            monkeypatch.setenv("VDL2GPU_K1_VARIANT", k1_variant)
        g = vd.Vdl2Receivers(fs, os_, vd.FMT_S16 if fmt == "s16" else vd.FMT_U8, [(c, f) for c, f, _ in rxs],
                             max_chunk_bytes=chunk, flags=flags)
        assert g.n_channels == sum(SIZES) and g.receiver_of(12) == 3 and list(g.channels_of(2)) == list(range(4, 12))
        g.process_chunked([b for _, _, b in rxs], chunk)
        frames = g.flush()
        dec = g.read_dec(chunk // bpp // os_ + 2)
        st, cnt = g.stats(), g.channel_counters()
        assert st["pool_overflows"] == 0 and st["out_overflows"] == 0
        assert (st["graph_launches"] > 0) == (not flags & vd.FLAG_NO_GRAPH)
        g.close()
        results.append((frames, cnt, dec))
        total = 0
        for r, (wf, wc, wd) in enumerate(want):
            chans = range(sum(SIZES[:r]), sum(SIZES[:r + 1]))
            mine = _local([f for f in frames if f.channel in chans], chans[0])
            util.assert_frames_equal(mine, wf, f"receiver {r} ({fmt}, os {os_}, flags {flags})")
            assert all(f.freq == rxs[r][1][f.channel] for f in mine)
            assert np.array_equal(cnt[chans[0]:chans[-1] + 1], wc), f"receiver {r}: counters"
            assert dec.shape[0] > 0 and np.array_equal(dec[:, chans[0]:chans[-1] + 1].view(np.uint32), wd[-dec.shape[0]:].view(np.uint32)), \
                f"receiver {r}: decimated samples of the last chunk"
            total += len(mine)
        assert total > 40
    fa, ca, da = results[0]
    for fb, cb, db in results[1:]:
        assert sorted(util.frame_tuple(f) for f in fa) == sorted(util.frame_tuple(f) for f in fb)
        assert np.array_equal(ca, cb) and np.array_equal(da.view(np.uint32), db.view(np.uint32))


def _pairs(chunk_bytes, b):
    return [b[o:o + chunk_bytes] for o in range(0, b.size, chunk_bytes)]


def test_one_receiver_equals_the_fan_out_context():
    fs, centre = 2100000, cases.CENTER
    iq, offs, _ = synth.traffic_stream(fs, 0.5, 48, 4.0, 22.0, -20.0, 0x52580001, "u8")
    freqs = [centre + int(o) for o in offs] + [centre]
    chunk = 131072
    a = vd.Vdl2Channels(fs, 20, vd.FMT_U8, centre, freqs, max_chunk_bytes=chunk)
    a.process_chunked(iq, chunk)
    fa, ca = a.flush(), a.channel_counters()
    b = vd.Vdl2Receivers(fs, 20, vd.FMT_U8, [(centre, freqs)], max_chunk_bytes=chunk)
    b.process_chunked([iq], chunk)
    fb, cb = b.flush(), b.channel_counters()
    assert len(fa) > 20
    util.assert_frames_equal(fb, fa, "one receiver vs fan-out")
    assert [f.freq for f in sorted(fb, key=lambda f: f.key())] == [f.freq for f in sorted(fa, key=lambda f: f.key())]
    assert np.array_equal(ca, cb)


def test_uniform_receivers_equal_the_independent_streams_mode():
    """4 receivers x 32 channels with one shared centre: the same as n_streams = 4 in the fan-out API"""
    fs, centre, S = 2100000, cases.CENTER, 4
    streams, freqs = [], None
    for s in range(S):
        iq, offs, _ = synth.traffic_stream(fs, 0.4, 32, 4.0, 22.0, -20.0, 0x52580100 + s, "u8")
        streams.append(np.ascontiguousarray(iq).view(np.uint8).reshape(-1))
        freqs = [centre + int(o) for o in offs]
    chunk = 131072
    a = vd.Vdl2Channels(fs, 20, vd.FMT_U8, centre, freqs * S, max_chunk_bytes=chunk, n_streams=S)
    for parts in zip(*[_pairs(chunk, b) for b in streams]):
        a.submit(np.concatenate(parts))
    fa, ca = a.flush(), a.channel_counters()
    b = vd.Vdl2Receivers(fs, 20, vd.FMT_U8, [(centre, freqs)] * S, max_chunk_bytes=chunk)
    b.process_chunked(streams, chunk)
    fb, cb = b.flush(), b.channel_counters()
    assert len(fa) > 20
    util.assert_frames_equal(fb, fa, "uniform receivers vs n_streams")
    assert np.array_equal(ca, cb)


def test_2048_receivers_of_8_channels_on_the_balanced_mapping():
    """16384 channels = 2048 receivers x 8: more than half a machine's worth, so the channels are dealt over all warps
    (32 or 31 per warp) and 4-warp blocks start and end inside receivers.  Receiver r is the base stream started 7919 r
    samples later, tuned to its own centre; the streams are built on the device and fed through submit_device."""
    import torch
    fs, pairs, R, n_chunks = 2100000, 65536, 2048, 3
    base, offs, _ = synth.traffic_stream(fs, 0.3, 8, 12.0, 24.0, -20.0, 0x52580200, "u8")
    L = base.size // 2
    b2 = torch.from_numpy(base[:2 * L].reshape(L, 2)).cuda()
    ar = torch.arange(n_chunks * pairs, device="cuda", dtype=torch.int64)
    raw = torch.empty(n_chunks, R, pairs, 2, dtype=torch.uint8, device="cuda")
    for r0 in range(0, R, 128):
        sh = (torch.arange(r0, r0 + 128, device="cuda", dtype=torch.int64) * 7919) % L
        blk = b2[(ar[None, :] + sh[:, None]) % L]
        for c in range(n_chunks):
            raw[c, r0:r0 + 128] = blk[:, c * pairs:(c + 1) * pairs]
    del blk
    centres = [135000000 + 1000 * r for r in range(R)]
    rx = [(centres[r], [centres[r] + int(o) for o in offs]) for r in range(R)]
    g = vd.Vdl2Receivers(fs, 20, vd.FMT_U8, rx, max_chunk_bytes=2 * pairs)
    st = torch.cuda.current_stream()
    for c in range(n_chunks):
        g.submit_device(raw[c].data_ptr(), 2 * pairs, st.cuda_stream)
    got = {}
    for f in g.flush():
        got.setdefault(g.receiver_of(f.channel), []).append(f)
    stats, cnt = g.stats(), g.channel_counters()
    g.close()
    assert stats["pool_overflows"] == 0 and stats["out_overflows"] == 0
    assert stats["msg_good"] > R // 4
    checked = 0
    # first and last; 63/64: the block boundary after the four 32-channel blocks; 67: straddles warps 16/17;
    # 79: straddles blocks 4/5; 1023/1024: mid-machine
    for r in (0, 1, 63, 64, 67, 79, 80, 1023, 1024, 2046, 2047):
        iq = np.roll(base[:2 * L], -2 * ((7919 * r) % L))[:2 * n_chunks * pairs]
        o = po.Oracle(fs, 20, po.FMT_U8, centres[r], rx[r][1])
        o.process_chunked(iq, 2 * pairs)
        mine = _local(got.get(r, []), 8 * r)
        util.assert_frames_equal(mine, o.frames(), f"receiver {r}")
        assert all(f.freq == rx[r][1][f.channel] for f in mine)
        assert np.array_equal(cnt[8 * r:8 * r + 8], o.counters()), f"receiver {r}: counters"
        checked += len(mine)
    assert checked > 2
