"""-m gpu: what a context owns over its lifetime.  A case decodes like the oracle through one stream for all stages
(VDL2GPU_FLAG_NO_OVERLAP, where the middle and back streams are the front stream) and through three
(VDL2GPU_STAGES=3).  Every kind of context - fan-out, independent streams, one stream per channel, receivers, mixed
receivers, ragged receivers with pushed input - is created and destroyed several times, and decoding afterwards still
matches the oracle.  The process's own device memory, as NVML reports it, comes back to where it was after those
cycles, after vdl2gpu_update_receivers grow/shrink cycles on a ragged context with pushed rings, and after an update
refused (ETOOBIG) before anything was allocated."""
import os
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from oracle import pyoracle as po
from tests import cases, util
from tests.test_gpu_mixed_receivers import _bpp, _local, _ofmt, _ragged, _vfmt

pytestmark = pytest.mark.gpu
ETOOBIG = -5
MiB = 1 << 20
SLACK = 8 * MiB          # the driver's own bookkeeping; a layout or ring set leaked on every cycle adds more than that
W = 3001                 # the largest span of the ragged contexts (max_chunk_bytes = W x 80)


def _own_device_bytes():
    """device memory NVML charges to this process, summed over the devices; skips when NVML cannot see the process"""
    try:
        import pynvml
    except ImportError:
        pytest.skip("pynvml is not installed")
    try:
        pynvml.nvmlInit()
        total, seen = 0, False
        for i in range(pynvml.nvmlDeviceGetCount()):
            for p in pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(i)):
                if p.pid == os.getpid() and p.usedGpuMemory is not None:
                    total, seen = total + p.usedGpuMemory, True
    except pynvml.NVMLError as e:
        pytest.skip(f"NVML: {e}")
    if not seen:
        pytest.skip("NVML does not list this process's device memory (another PID namespace, or no permission)")
    return total


def _cfg2_channels(c, flags=0, **kw):
    return vd.Vdl2Channels(c["fs"], c["oversample"], util.fmt_code(c), c["centerfreq"], c["freqs"], flags=flags, **kw)


def _decode_cfg2(c, flags=0):
    g = _cfg2_channels(c, flags)
    g.process_chunked(util.case_bytes(c), c["chunk"])
    fr, cnt = g.flush(), g.channel_counters()
    g.close()
    return fr, cnt


def _desc(x):
    return (x["centre"], x["freqs"], x["os"], _vfmt(x["fmt"]))


def _w(x):
    return x["os"] * _bpp(x["fmt"])


def _push_decode(rxs, piece=7777):
    """every receiver's bytes pushed in odd pieces, drained after each round; frames per receiver, counters, bytes"""
    g = vd.Vdl2MixedReceivers([_desc(x) for x in rxs], max_chunk_bytes=W * 80, ragged=True)
    sent = [0] * len(rxs)
    while any(s < x["buf"].size for s, x in zip(sent, rxs)):
        for r, x in enumerate(rxs):
            g.push(r, x["buf"][sent[r]:sent[r] + piece])
            sent[r] = min(sent[r] + piece, x["buf"].size)
        g.submit_pushed()
    fr, cnt = g.flush(), g.channel_counters()
    first = [g.channels_of(r)[0] for r in range(len(rxs))] + [g.n_channels]
    g.close()
    return fr, cnt, first, sent


def _check_pushed(rxs, what):
    fr, cnt, first, sent = _push_decode(rxs)
    n = 0
    for r, x in enumerate(rxs):
        o = po.Oracle(105000 * x["os"], x["os"], _ofmt(x["fmt"]), x["centre"], x["freqs"])
        o.process(x["buf"][:sent[r] // _w(x) * _w(x)])
        mine = _local([f for f in fr if first[r] <= f.channel < first[r + 1]], first[r])
        util.assert_frames_equal(mine, o.frames(), f"{what}: receiver {r}")
        assert np.array_equal(cnt[first[r]:first[r + 1]], o.counters()), f"{what}: receiver {r} counters"
        n += len(mine)
    return n


@pytest.fixture(scope="module")
def fleet():
    rxs, _ = _ragged(0.3, 0x4C494600)
    return rxs[:4]


def _kinds(fleet):
    """one create / feed / destroy of every kind of context, with the optional per-input and per-channel buffers"""
    c = cases.case_cfg2(0.2)
    data = util.case_bytes(c)
    rng = np.random.default_rng(0x4C494601)
    noise = rng.integers(0, 256, 1 << 18, dtype=np.uint8)
    meters = dict(levels=True, channel_levels=True, spectrum=True)
    rx = [(x["centre"], x["freqs"]) for x in fleet]

    def fan_out(flags=0):
        g = _cfg2_channels(c, flags, **meters)
        g.process_chunked(data, c["chunk"])
        return g

    def streams():
        g = vd.Vdl2Channels(2100000, 20, vd.FMT_U8, cases.CENTER, [cases.CENTER + 25000 * (k - 32) for k in range(64)],
                            n_streams=2, **meters)
        g.submit(noise)
        return g

    def lanes():
        g = vd.Vdl2Channels(2100000, 20, vd.FMT_U8, cases.CENTER, [cases.CENTER + 25000 * k for k in range(4)], n_streams=4,
                            **meters)
        g.submit(noise)
        return g

    def receivers():
        g = vd.Vdl2Receivers(2100000, 20, vd.FMT_U8, rx, **meters)
        g.submit([noise[:1 << 16]] * len(rx))
        return g

    def mixed():
        g = vd.Vdl2MixedReceivers([_desc(x) for x in fleet], **meters)
        g.submit_span([x["buf"][:1000 * _w(x)] for x in fleet])
        return g

    def ragged():
        g = vd.Vdl2MixedReceivers([_desc(x) for x in fleet], max_chunk_bytes=W * 80, ragged=True, **meters)
        for r, x in enumerate(fleet):
            g.push(r, x["buf"][:5000 + 13 * r])
        g.submit_pushed()
        return g

    return [fan_out, lambda: fan_out(vd.FLAG_NO_OVERLAP), lambda: fan_out(vd.FLAG_NO_GRAPH), streams, lanes, receivers,
            mixed, ragged]


def _cycle(kinds, monkeypatch, times):
    for _ in range(times):
        for k in kinds:
            g = k()
            g.flush()
            g.close()
        monkeypatch.setenv("VDL2GPU_STAGES", "3")          # three streams: K2a on a stream of its own
        for k in kinds[:3]:
            g = k()
            g.flush()
            g.close()
        monkeypatch.delenv("VDL2GPU_STAGES")


def test_aliased_and_three_streams_decode_like_the_oracle(monkeypatch):
    c = cases.case_cfg2()
    o = util.run_oracle(c)
    fr, cnt = _decode_cfg2(c, vd.FLAG_NO_OVERLAP)
    util.assert_frames_equal(fr, o.frames(), "one stream for all stages")
    assert np.array_equal(cnt, o.counters())
    monkeypatch.setenv("VDL2GPU_STAGES", "3")
    fr, cnt = _decode_cfg2(c)
    util.assert_frames_equal(fr, o.frames(), "three streams")
    assert np.array_equal(cnt, o.counters())
    assert len(fr) >= 8


def test_every_kind_survives_create_destroy_cycles(fleet, monkeypatch):
    _cycle(_kinds(fleet), monkeypatch, 3)
    c = cases.case_cfg2()
    o = util.run_oracle(c)
    for flags in (0, vd.FLAG_NO_OVERLAP):
        fr, cnt = _decode_cfg2(c, flags)
        util.assert_frames_equal(fr, o.frames(), f"after the cycles, flags {flags}")
        assert np.array_equal(cnt, o.counters())
    _check_pushed(fleet, "pushed, after the cycles")


def test_create_destroy_cycles_return_device_memory(fleet, monkeypatch):
    kinds = _kinds(fleet)
    _cycle(kinds, monkeypatch, 1)                            # loads every kernel and the driver's lazy state
    before = _own_device_bytes()
    _cycle(kinds, monkeypatch, 5)
    after = _own_device_bytes()
    assert after - before <= SLACK, f"{(after - before) / MiB:.1f} MiB more after 5 create/destroy cycles of every kind"


def test_update_cycles_and_a_refused_update_return_device_memory(fleet):
    """a ragged context with pushed rings: a receiver joins and leaves 20 times, with partial groups queued across every
    update; then an update whose layout exceeds the kernels' 32-bit element index is refused before it allocates"""
    g = vd.Vdl2MixedReceivers([_desc(x) for x in fleet[:3]], max_chunk_bytes=W * 80, ragged=True,
                              levels=True, channel_levels=True, spectrum=True)
    sent = [0] * 4

    def feed(n_rx, n):
        for r in range(n_rx):
            x = fleet[r]
            g.push(r, x["buf"][sent[r]:sent[r] + n + 3 * r])
            sent[r] += n + 3 * r
        g.submit_pushed()
        g.flush()

    def grow_shrink():
        sent[3] = 0
        g.add_receivers([_desc(fleet[3])])
        feed(4, 2345)
        g.remove_receivers([3])
        feed(3, 1234)

    feed(3, 4000)
    grow_shrink()
    before = _own_device_bytes()
    for _ in range(20):
        grow_shrink()
    mid = _own_device_bytes()
    assert mid - before <= SLACK, f"{(mid - before) / MiB:.1f} MiB more after 20 update cycles"
    n_ch = 700000                                           # (max_span + 2 + 160) x n_ch >= 2^32 at max_chunk_bytes W x 80
    rx = (vd.api._ReceiverEx * 1)()
    rx[0].centerfreq, rx[0].n_channels, rx[0].oversample, rx[0].sample_fmt = cases.CENTER, n_ch, 20, vd.FMT_U8
    src = np.full(1, -1, np.int32)
    freqs = np.full(n_ch, cases.CENTER, np.uint32)
    assert g.L.vdl2gpu_update_receivers(g.h, rx, src.ctypes.data, 1, freqs.ctypes.data) == ETOOBIG
    assert "32-bit element index" in g.L.vdl2gpu_last_error().decode()
    assert _own_device_bytes() - mid <= SLACK
    pos = g.receiver_positions().tolist()
    feed(3, 3000)
    assert [int(p) for p in g.receiver_positions()] == [sent[r] // _w(fleet[r]) for r in range(3)]
    assert all(b > a for a, b in zip(pos, g.receiver_positions().tolist()))
    g.close()
