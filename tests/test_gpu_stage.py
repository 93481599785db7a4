"""-m gpu: the public launch stubs one stage at a time (include/vdl2gpu.h "raw launch stubs" / "stage stubs") against
the oracle's output for the same stage, plus the run-time variants of the pipeline (CUDA graphs on/off, K2a
evaluation, K2 walk variants, independent streams), which must not change a single bit."""
import ctypes as C
import os
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import api
from oracle import pyoracle as po
from tests import cases, util

pytestmark = pytest.mark.gpu


class Stage:
    """vdl2gpu_stage on a torch-allocated block of device memory"""

    def __init__(self, case, max_dec, flags=0):
        import torch
        self.L = vd.load_library()
        self.cfg, self._fr = api.make_config(case["fs"], case["oversample"], util.fmt_code(case), case["centerfreq"], case["freqs"],
                                             max_ppm=case.get("max_ppm", 0.0), flags=flags)
        self.n_ch = len(case["freqs"])
        self.stride = self.L.vdl2gpu_stage_row_stride(self.n_ch)
        nbytes = self.L.vdl2gpu_stage_device_bytes(self.n_ch, max_dec, flags)
        self.mem = torch.zeros(nbytes + 256, dtype=torch.uint8, device="cuda")
        base = (self.mem.data_ptr() + 255) & ~255
        self.h = C.c_void_p()
        rc = self.L.vdl2gpu_stage_create(C.byref(self.cfg), max_dec, C.c_void_p(base), nbytes, C.byref(self.h))
        assert rc == 0, self.L.vdl2gpu_last_error()
        self.max_dec = max_dec

    def levels(self):
        p = C.c_void_p()
        assert self.L.vdl2gpu_stage_levels(self.h, C.byref(p)) == 0
        return p.value

    def close(self):
        self.L.vdl2gpu_stage_destroy(self.h)


def _convert(st, case, raw_bytes):
    import torch
    fmt = util.fmt_code(case)
    n_pairs = raw_bytes.size // (4 if fmt == po.FMT_S16 else 2)
    d_raw = torch.from_numpy(raw_bytes.copy()).cuda()
    s4 = torch.empty(n_pairs, 2, dtype=torch.float32, device="cuda")
    assert st.L.vdl2gpu_launch_convert(d_raw.data_ptr(), n_pairs, fmt, st.levels(), s4.data_ptr(), None) == 0
    return s4, n_pairs


def test_convert_stub():
    import torch
    L = vd.load_library()
    rng = np.random.default_rng(3)
    raw = rng.integers(0, 256, 2 * 5000, dtype=np.uint8)
    lv = po.levels_u8()
    d_raw = torch.from_numpy(raw).cuda(); d_lv = torch.from_numpy(lv).cuda()
    out = torch.zeros(5000, 2, dtype=torch.float32, device="cuda")
    assert L.vdl2gpu_launch_convert(d_raw.data_ptr(), 5000, 0, d_lv.data_ptr(), out.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), lv[raw].reshape(-1, 2))
    s16 = rng.integers(-32768, 32768, 2 * 5000, dtype=np.int16)
    d_s = torch.from_numpy(s16).cuda()
    assert L.vdl2gpu_launch_convert(d_s.data_ptr(), 5000, 1, None, out.data_ptr(), None) == 0
    torch.cuda.synchronize()
    want = (s16.astype(np.float32) / np.float32(32768.0)).reshape(-1, 2)
    assert np.array_equal(out.cpu().numpy(), want)


@pytest.mark.parametrize("name", ["cfg2", "mixed_s16"])
def test_stage_stubs_k1_k2_k3_against_the_oracle(name):
    """K0 -> K1 -> (K2a + K2) -> K3 through the four launch stubs, buffer by buffer: decimated samples bit-exact,
    sync/header events bit-exact, frames + metadata identical."""
    import torch
    c = cases.ALL_GOLDEN[name]()
    o = util.run_oracle(c, trace=True, dec_tap=True)
    odec = o.dec_samples()
    b = util.case_bytes(c)
    chunk = c["chunk"]
    bpp = 4 if c["fmt"] == "s16" else 2
    max_dec = chunk // bpp // c["oversample"] + 2
    st = Stage(c, max_dec, flags=vd.FLAG_TRACE)
    dec = torch.zeros(max_dec, st.stride, 2, dtype=torch.float32, device="cuda")
    region = torch.zeros(4 << 20, dtype=torch.uint8, device="cuda")
    frames, pos = [], 0
    for off in range(0, b.size, chunk):
        s4, n_pairs = _convert(st, c, b[off:off + chunk])
        n_dec = C.c_uint32(0)
        assert st.L.vdl2gpu_launch_mix_iir_decimate(st.h, s4.data_ptr(), n_pairs, dec.data_ptr(), C.byref(n_dec), None) == 0
        n = n_dec.value
        torch.cuda.synchronize()
        got = dec[:n, :st.n_ch].cpu().numpy()
        want = odec[pos:pos + n]
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{name}: K1 stub output differs at byte {off}"
        pos += n
        assert st.L.vdl2gpu_launch_sync_slice(st.h, dec.data_ptr(), n, None) == 0
        assert st.L.vdl2gpu_launch_burst_fec(st.h, region.data_ptr(), region.numel(), None) == 0
        torch.cuda.synchronize()
        frames += api.parse_records(region.cpu().numpy().tobytes(), c["fs"] // c["oversample"])
    assert pos == odec.shape[0]
    util.assert_frames_equal(frames, o.frames(), f"stage stubs [{name}]")
    ev = (api._Event * (1 << 16))()
    n = st.L.vdl2gpu_stage_read_events(st.h, C.cast(ev, C.c_void_p), 1 << 16)
    got_ev = [dict(channel=ev[k].channel, kind=ev[k].kind, dec_index=ev[k].dec_index, i=list(ev[k].i),
                   f=np.array(list(ev[k].f), np.float32)) for k in range(n)]
    util.assert_events_equal(got_ev, o.events(), f"stage stubs events [{name}]")
    st.close()


def test_sync_slice_stub_on_the_oracles_decimated_samples():
    """K2 alone: the oracle's own decimated samples in, the oracle's sync/header events and frames out."""
    import torch
    c = cases.ALL_GOLDEN["noisy"]()
    o = util.run_oracle(c, trace=True, dec_tap=True)
    odec = o.dec_samples()                                   # [n_dec][n_ch][2]
    n_total, n_ch = odec.shape[0], odec.shape[1]
    step = 4000
    st = Stage(c, step, flags=vd.FLAG_TRACE)
    region = torch.zeros(4 << 20, dtype=torch.uint8, device="cuda")
    frames = []
    for m in range(0, n_total, step):
        blk = odec[m:m + step]
        padded = np.zeros((blk.shape[0], st.stride, 2), np.float32)
        padded[:, :n_ch] = blk
        d = torch.from_numpy(padded).cuda()
        assert st.L.vdl2gpu_launch_sync_slice(st.h, d.data_ptr(), blk.shape[0], None) == 0
        assert st.L.vdl2gpu_launch_burst_fec(st.h, region.data_ptr(), region.numel(), None) == 0
        torch.cuda.synchronize()
        frames += api.parse_records(region.cpu().numpy().tobytes(), c["fs"] // c["oversample"])
    util.assert_frames_equal(frames, o.frames(), "K2/K3 stubs on oracle dec")
    st.close()


def _phase_inputs(rng, n):
    parts = []
    a = rng.uniform(0, 2 * np.pi, n); r = rng.uniform(1e-3, 0.5, n)
    parts.append(np.stack([r * np.cos(a), r * np.sin(a)], 1))
    parts.append(0.01 * rng.standard_normal((n, 2)))
    a = rng.integers(0, 8, n) * (np.pi / 4) + (rng.uniform(-0.5, 0.5, n) * 1e-3 * 10.0 ** (-6 * rng.uniform(0, 1, n)))
    parts.append(np.stack([0.3 * np.cos(a), 0.3 * np.sin(a)], 1))
    parts.append(rng.integers(-16, 17, (n, 2)).astype(np.float64))
    lv = (np.arange(256) - 127.5) / 127.5 * 0.01
    parts.append(lv[rng.integers(0, 256, (n, 2))])
    parts.append(np.exp(rng.uniform(np.log(1e-8), np.log(1e3), (n, 2))) * rng.choice([-1.0, 1.0], (n, 2)))
    sp = np.array([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, np.nan, 1e-38, 1e-45, 3e38])
    parts.append(np.array([[x, y] for x in sp for y in sp]))
    return np.concatenate(parts).astype(np.float32)


def test_phase_mag_stub_fast_equals_libm_equals_glibc():
    """K2a: the Ziv-guarded short atan2 == libdevice atan2 == glibc atan2 after narrowing to float, bit for bit;
    hypot likewise (src/demod.c:232,238,256)."""
    import torch
    L = vd.load_library()
    rng = np.random.default_rng(0x56444C32)
    x = _phase_inputs(rng, 400000)
    d = torch.from_numpy(x).cuda()
    n = x.shape[0]
    res = []
    for exact in (0, 1):
        ph = torch.zeros(n, dtype=torch.float32, device="cuda"); mg = torch.zeros(n, dtype=torch.float32, device="cuda")
        assert L.vdl2gpu_launch_phase_mag(d.data_ptr(), n, ph.data_ptr(), mg.data_ptr(), exact, None) == 0
        torch.cuda.synchronize()
        res.append((ph.cpu().numpy(), mg.cpu().numpy()))
    re, im = x[:, 0].astype(np.float64), x[:, 1].astype(np.float64)
    with np.errstate(all="ignore"):
        want_ph = np.arctan2(im, re).astype(np.float32)
        want_mg = np.sqrt(re * re + im * im).astype(np.float32)

    def same(a, b):
        return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))
    assert same(res[0][0], res[1][0]).all(), "fast and libdevice phases differ"
    bad = ~same(res[0][0], want_ph)
    assert bad.sum() == 0, f"{bad.sum()} phases differ from glibc, first: {x[bad][:4]} {res[0][0][bad][:4]} {want_ph[bad][:4]}"
    assert same(res[0][1], res[1][1]).all()
    finite = np.isfinite(want_mg) & (np.abs(re) < 1e18) & (np.abs(im) < 1e18)
    assert same(res[0][1][finite], want_mg[finite]).all()


def _frames_of(case, env=None, flags=0, chunk=None):
    old = {k: os.environ.get(k) for k in (env or {})}
    try:
        for k, v in (env or {}).items():
            os.environ[k] = str(v)
        g = vd.Vdl2Channels(case["fs"], case["oversample"], util.fmt_code(case), case["centerfreq"], case["freqs"],
                            max_ppm=case.get("max_ppm", 0.0), max_chunk_bytes=max(chunk or case["chunk"], 1 << 16), flags=flags)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    g.process_chunked(util.case_bytes(case), chunk or case["chunk"])
    fr = g.flush()
    st = g.stats()
    cnt = g.channel_counters()
    g.close()
    return fr, st, cnt


def test_cuda_graph_replay_equals_direct_launches():
    c = cases.case_replicas(n_slots=16, n_rep=4, duration=1.0)
    o = util.run_oracle(c)
    f_graph, st_graph, cnt_graph = _frames_of(c, chunk=200000)
    f_direct, st_direct, cnt_direct = _frames_of(c, flags=vd.FLAG_NO_GRAPH, chunk=200000)
    assert st_graph["graph_launches"] >= 3 * (st_graph["chunks_submitted"] - 1) and st_direct["graph_launches"] == 0
    util.assert_frames_equal(f_graph, o.frames(), "graph replay vs oracle")
    util.assert_frames_equal(f_direct, o.frames(), "direct launches vs oracle")
    assert np.array_equal(cnt_graph, cnt_direct) and np.array_equal(cnt_graph, o.counters())
    assert len(f_graph) > 20


@pytest.mark.parametrize("env", [dict(VDL2GPU_K2A=0), dict(VDL2GPU_STAGES=3), dict(VDL2GPU_K2_VARIANT=1), dict(VDL2GPU_K2_VARIANT=3),
                                 dict(VDL2GPU_K2_VARIANT=4), dict(VDL2GPU_K2_VARIANT=5), dict(VDL2GPU_K2_VARIANT=0), dict(VDL2GPU_K1_VARIANT=0),
                                 dict(VDL2GPU_K1_VARIANT=8),
                                 dict(VDL2GPU_K1_VARIANT=4)])
def test_kernel_variants_do_not_change_results(env):
    c = cases.ALL_GOLDEN["noisy"]()
    o = util.run_oracle(c)
    fr, st, cnt = _frames_of(c, env=env)
    util.assert_frames_equal(fr, o.frames(), f"variant {env}")
    assert np.array_equal(cnt, o.counters())
    c2 = cases.case_stress()
    o2 = util.run_oracle(c2)
    fr2, _, cnt2 = _frames_of(c2, env=env)
    util.assert_frames_equal(fr2, o2.frames(), f"variant {env} [stress]")
    assert np.array_equal(cnt2, o2.counters())


def test_independent_streams_mode():
    """4 different IQ streams x 32 channels in one context: stream s feeds channels [32 s, 32 s + 32) and every one of
    them must equal the oracle run on that stream alone (src/demod.c:302-329: each channel thread reads its buffer)."""
    from dumpvdl2_b200 import synth
    fs, center = 2100000, cases.CENTER
    S, Cn, chunk = 4, 32, 262144
    streams, want = [], []
    offs = synth.slot_offsets(Cn, 25e3)
    freqs_one = [center + int(o) for o in offs]
    for s in range(S):
        iq, _, _ = synth.traffic_stream(fs, 0.75, Cn, 6.0, 22.0, -20.0, 0x56444C40 + s, "u8")
        n = (iq.size // chunk) * chunk
        streams.append(iq[:n])
        o = po.Oracle(fs, 20, po.FMT_U8, center, freqs_one)
        o.process_chunked(iq[:n], chunk)
        want.append(o)
    n = min(x.size for x in streams)
    g = vd.Vdl2Channels(fs, 20, vd.FMT_U8, center, freqs_one * S, max_chunk_bytes=chunk, n_streams=S)
    for off in range(0, n, chunk):
        g.process_buf_uchar(np.concatenate([x[off:off + chunk] for x in streams]))
    got = g.flush()
    st = g.stats()
    assert st["pool_overflows"] == 0 and st["out_overflows"] == 0
    total = 0
    for s in range(S):
        mine = [f for f in got if s * Cn <= f.channel < (s + 1) * Cn]
        for f in mine:
            f.channel -= s * Cn
        util.assert_frames_equal(mine, want[s].frames(), f"stream {s}")
        total += len(mine)
    assert total > 40
    cnt = g.channel_counters()
    for s in range(S):
        assert np.array_equal(cnt[s * Cn:(s + 1) * Cn], want[s].counters())
    g.close()


@pytest.mark.parametrize("n_streams,os_", [(32, 20), (40, 20), (40, 10)], ids=["32", "40", "40-os10"])
def test_one_stream_per_channel_mode(n_streams, os_):
    """n_streams == n_channels: every channel demodulates its OWN IQ stream (the reference's traffic model, one buffer
    per channel thread); K0 lays the samples out time-major across streams and K1 runs one lane per stream.  Each
    channel must equal the oracle run on its stream alone; 40 streams leave 24 lanes of the second warp idle."""
    from dumpvdl2_b200 import synth
    fs, center, chunk = 105000 * os_, cases.CENTER, 131072
    base, offs, _ = synth.traffic_stream(fs, 0.6, 8, 8.0, 24.0, -20.0, 0x56444C50, "u8")
    n = (base.size // chunk) * chunk
    base = base[:n]
    streams, freqs, want = [], [], []
    for s in range(n_streams):
        iq = np.roll(base, 2 * 7919 * s)                     # the same traffic, shifted in time: a different stream per channel
        f = center + int(offs[s % len(offs)])
        o = po.Oracle(fs, os_, po.FMT_U8, center, [f])
        o.process_chunked(iq, chunk)
        streams.append(iq); freqs.append(f); want.append(o)
    g = vd.Vdl2Channels(fs, os_, vd.FMT_U8, center, freqs, max_chunk_bytes=chunk, n_streams=n_streams)
    for off in range(0, n, chunk):
        g.process_buf_uchar(np.concatenate([x[off:off + chunk] for x in streams]))
    got = g.flush()
    total = 0
    for s in range(n_streams):
        mine = [f for f in got if f.channel == s]
        for f in mine:
            f.channel = 0
        util.assert_frames_equal(mine, want[s].frames(), f"stream {s}")
        total += len(mine)
    assert total > 20
    cnt = g.channel_counters()
    for s in range(n_streams):
        assert np.array_equal(cnt[s:s + 1], want[s].counters())
    st = g.stats()
    assert st["pool_overflows"] == 0 and st["out_overflows"] == 0
    g.close()


def test_one_stream_per_channel_with_the_balanced_slot_mapping():
    """9600 streams x 1 channel: more than half a machine's worth, so the channels are dealt out over all 592 warps (17 or
    16 per warp) and K0 has to place stream c in column slot(c).  The streams are built on the device (stream s = the base
    stream started 7919 s samples later) and fed through submit_device; a sample of channels is checked against the oracle."""
    import torch
    from dumpvdl2_b200 import synth
    fs, center, pairs = 2100000, cases.CENTER, 65536
    S, n_chunks = 9600, 3
    base, offs, _ = synth.traffic_stream(fs, 0.3, 8, 12.0, 24.0, -20.0, 0x56444C51, "u8")
    L = base.size // 2
    b2 = torch.from_numpy(base[:2 * L].reshape(L, 2)).cuda()
    ar = torch.arange(n_chunks * pairs, device="cuda", dtype=torch.int64)
    raw = torch.empty(n_chunks, S, pairs, 2, dtype=torch.uint8, device="cuda")
    for s0 in range(0, S, 128):
        sh = (torch.arange(s0, min(s0 + 128, S), device="cuda", dtype=torch.int64) * 7919) % L
        idx = (ar[None, :] + sh[:, None]) % L                      # [streams][time]
        blk = b2[idx]                                              # [streams][time][2]
        for c in range(n_chunks):
            raw[c, s0:s0 + idx.shape[0]] = blk[:, c * pairs:(c + 1) * pairs]
    freqs = [center + int(offs[s % len(offs)]) for s in range(S)]
    g = vd.Vdl2Channels(fs, 20, vd.FMT_U8, center, freqs, max_chunk_bytes=2 * pairs, n_streams=S)
    st = torch.cuda.current_stream()
    for c in range(n_chunks):
        g.submit_device(raw[c].data_ptr(), 2 * pairs, st.cuda_stream)
    got = {}
    for f in g.flush():
        got.setdefault(f.channel, []).append(f)
    cnt = g.channel_counters()
    g.close()
    checked = 0
    for s in (0, 1, 16, 17, 31, 32, 4799, 4800, 9215, 9216, 9599):
        iq = np.roll(base[:2 * L], -2 * ((7919 * s) % L))[:2 * n_chunks * pairs]
        o = po.Oracle(fs, 20, po.FMT_U8, center, [freqs[s]])
        o.process_chunked(iq, 2 * pairs)
        mine = got.get(s, [])
        for f in mine:
            f.channel = 0
        util.assert_frames_equal(mine, o.frames(), f"stream {s}")
        assert np.array_equal(cnt[s:s + 1], o.counters())
        checked += len(mine)
    assert checked > 2
