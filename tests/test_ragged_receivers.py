"""CPU: ragged spans on a mixed-receivers context (VDL2GPU_FLAG_RAGGED, vdl2gpu_submit_ragged) without a GPU - every
refusal (EINVAL, ETOOBIG) that needs no device, ENODEV for valid ragged configurations - the per-span receiver table and the
ragged K1's per-row copy sizes of vdl2_core.cuh compiled for the host (tests/hostsim/layout_ragged.cpp, TEST-ONLY), and
the contract the GPU tests rely on: the oracle fed one receiver's stream in ragged cuts equals the oracle on the whole
stream."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import api, synth
from oracle import pyoracle as po
from tests import util

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "dumpvdl2_b200", "csrc")
EINVAL, ENODEV, ETOOBIG = -1, -2, -5


@pytest.fixture(scope="module")
def lay(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("layout_ragged") / "liblayout.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I", CSRC, "-o", so, os.path.join(HERE, "hostsim", "layout_ragged.cpp")])
    L = C.CDLL(so)
    L.ragged_span_table.restype = C.c_uint64
    L.ragged_span_table.argtypes = [C.c_void_p] * 2 + [C.c_uint32] + [C.c_void_p] * 4
    L.ragged_tile_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    L.ragged_span_entry_bytes.restype = C.c_size_t
    return L


class Stepper:
    """the library's per-receiver bookkeeping, stepped span by span through vdl2_rx_span_table"""

    def __init__(self, lay, os_, fmt):
        self.lay = lay
        self.os = np.ascontiguousarray(os_, np.uint32)
        self.fmt = np.ascontiguousarray(fmt, np.uint32)
        self.pos = np.zeros(self.os.size, np.uint64)
        self.prev = np.zeros(self.os.size, np.uint32)

    def span(self, counts):
        n = np.ascontiguousarray(counts, np.uint32)
        out = np.zeros((self.os.size, 4), np.uint64)
        b = self.lay.ragged_span_table(self.os.ctypes.data, self.fmt.ctypes.data, self.os.size, n.ctypes.data,
                                       self.pos.ctypes.data, self.prev.ctypes.data, out.ctypes.data)
        return b, out


def test_span_entry_is_24_bytes(lay):
    assert lay.ragged_span_entry_bytes() == 24


def test_table_across_spans_with_zero_counts(lay):
    mix = [(10, 0), (20, 1), (13, 0), (20, 0), (10, 1)]
    widths = [o * (4 if f else 2) for o, f in mix]
    st = Stepper(lay, [m[0] for m in mix], [m[1] for m in mix])
    rng = np.random.default_rng(7)
    spans = [[0, 0, 0, 0, 0], [5, 0, 1, 160, 11], [0, 0, 0, 159, 0], [300, 12, 0, 0, 7], [0, 3001, 2, 1, 0]]
    spans += [list(rng.integers(0, 400, 5) * (rng.random(5) > 0.3)) for _ in range(40)]
    pos, prev = np.zeros(5, np.int64), np.zeros(5, np.int64)
    for counts in spans:
        b, t = st.span(counts)
        assert b == sum(n * w for n, w in zip(counts, widths))
        assert t[:, 0].tolist() == [sum(counts[q] * widths[q] for q in range(r)) for r in range(5)]
        assert t[:, 1].tolist() == list(counts)
        assert t[:, 2].tolist() == prev.tolist()
        assert t[:, 3].tolist() == pos.tolist()
        pos += np.asarray(counts)
        prev = np.asarray(counts, np.int64)
    assert st.pos.tolist() == pos.tolist() and st.prev.tolist() == prev.tolist()


def test_table_offsets_pass_4_gib(lay):
    """65535 cs16 receivers at oversample 20 bringing 13107 decimated samples each (the largest 1 MiB allows), except
    every third receiver, which brings nothing: offsets run far past 4 GiB"""
    n = 65535
    counts = np.where(np.arange(n) % 3 == 0, 0, 13107).astype(np.uint32)
    st = Stepper(lay, [20] * n, [1] * n)
    b, t = st.span(counts)
    want = np.concatenate([[0], np.cumsum(counts.astype(np.uint64) * np.uint64(80))])
    assert b == int(want[-1]) and b > 1 << 32
    assert np.array_equal(t[:, 0], want[:-1])
    assert int(t[-1, 0]) > 1 << 32


@pytest.mark.parametrize("seed", range(6))
def test_k1_row_copies_for_random_counts(lay, seed):
    rng = np.random.default_rng(seed)
    G = int(rng.integers(1, 129))
    os_ = np.ascontiguousarray(rng.choice([10, 13, 20], G), np.uint32)
    counts = rng.integers(0, 100, G) * (rng.random(G) > 0.25)
    if seed == 0:
        counts[:] = 0
        counts[1 % G] = 1
    n = np.ascontiguousarray(counts, np.uint32)
    TG = int(rng.choice([2, 4, 10, 38]))
    width = int(n.max())
    staged = np.zeros(G, np.int64)
    for g0 in range(0, width, TG):
        out = np.zeros((G, 4), np.uint32)
        lay.ragged_tile_rows(n.ctypes.data, os_.ctypes.data, G, g0, TG, out.ctypes.data)
        groups, samples, nbytes, odd = (out[:, k].astype(np.int64) for k in range(4))
        want = np.clip(n.astype(np.int64) - g0, 0, TG)
        assert np.array_equal(groups, want)
        assert np.array_equal(samples, want * os_)
        assert np.array_equal(nbytes, (samples & ~1) * 8)
        assert np.array_equal(odd, samples & 1)
        assert np.all(nbytes[groups == 0] == 0)                      # a row with nothing left issues no copy
        assert np.all(nbytes[groups > 0] > 0) and np.all(nbytes % 16 == 0)
        # the tile's expected transaction bytes (what warp 0 reduces) = the bytes of the copies issued
        assert int(nbytes.sum()) == sum(int(b) for b in nbytes if b)
        assert np.all(odd[os_ != 13] == 0)                          # only an odd factor can end on an odd sample
        assert np.all(groups.max() > 0)                             # no tile of the block's loop is empty
        staged += groups
    assert np.array_equal(staged, n)


def test_odd_tail_at_oversample_13(lay):
    n = np.array([3, 1, 0, 2], np.uint32)
    os_ = np.array([13, 13, 13, 13], np.uint32)
    out = np.zeros((4, 4), np.uint32)
    lay.ragged_tile_rows(n.ctypes.data, os_.ctypes.data, 4, 0, 10, out.ctypes.data)
    assert out.tolist() == [[3, 39, 38 * 8, 1], [1, 13, 12 * 8, 1], [0, 0, 0, 0], [2, 26, 26 * 8, 0]]


# ---- the contract: where a receiver's stream is cut does not change what it decodes ----
@pytest.mark.parametrize("os_,fmt", [(10, "u8"), (20, "s16"), (13, "u8")])
def test_oracle_in_ragged_cuts_equals_the_whole_stream(os_, fmt):
    bpp = 4 if fmt == "s16" else 2
    iq, offs, _ = synth.traffic_stream(105000 * os_, 0.6, 4, 6.0, 24.0, -20.0, 0x52414700 + os_, fmt)
    buf = np.ascontiguousarray(iq).view(np.uint8).reshape(-1)
    w = os_ * bpp
    buf = buf[:buf.size // w * w]
    total = buf.size // w
    centre = 136500000
    freqs = [centre + int(o) for o in offs[:4]]
    whole = po.Oracle(105000 * os_, os_, po.FMT_S16 if fmt == "s16" else po.FMT_U8, centre, freqs, dec_tap=True)
    whole.process(buf)
    cut = po.Oracle(105000 * os_, os_, po.FMT_S16 if fmt == "s16" else po.FMT_U8, centre, freqs, dec_tap=True)
    rng = np.random.default_rng(os_)
    pattern = [0, 1, 11, 159, 160, 0, 0, 12, 3001, 1, 0, 159]
    pos = 0
    while pos < total:
        n = pattern.pop(0) if pattern else int(rng.choice([0, 1, 11, 159, 160, int(rng.integers(0, 5000))]))
        n = min(n, total - pos)
        cut.process(buf[pos * w:(pos + n) * w])
        pos += n
    assert len(whole.frames()) > 5
    util.assert_frames_equal(cut.frames(), whole.frames(), f"ragged cuts os {os_} {fmt}")
    assert np.array_equal(cut.counters(), whole.counters())
    assert np.array_equal(cut.dec_samples().view(np.uint32), whole.dec_samples().view(np.uint32))


# ---- refusals that need no device ----
def _cfg(freqs, flags, **kw):
    fr = np.ascontiguousarray(freqs, np.uint32)
    cfg = api._Config()
    cfg.n_channels, cfg.freqs = fr.size, fr.ctypes.data_as(C.POINTER(C.c_uint32))
    cfg.device, cfg.flags = -1, flags
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg, fr


def test_ragged_flag_is_refused_outside_mixed_receivers():
    L = vd.load_library()
    assert vd.FLAG_RAGGED == 32
    h = C.c_void_p()
    cfg, _k = _cfg([136975000], vd.FLAG_RAGGED, sample_rate=2100000, oversample=20, centerfreq=136975000)
    assert L.vdl2gpu_create(C.byref(cfg), C.byref(h)) == EINVAL
    assert "VDL2GPU_FLAG_RAGGED" in L.vdl2gpu_last_error().decode() and "vdl2gpu_create" in L.vdl2gpu_last_error().decode()
    rx = (api._Receiver * 1)()
    rx[0].centerfreq, rx[0].n_channels = 136975000, 1
    assert L.vdl2gpu_create_receivers(C.byref(cfg), rx, 1, C.byref(h)) == EINVAL
    assert "VDL2GPU_FLAG_RAGGED" in L.vdl2gpu_last_error().decode() and "vdl2gpu_create_receivers" in L.vdl2gpu_last_error().decode()
    mem = (C.c_uint8 * 4096)()
    assert L.vdl2gpu_stage_create(C.byref(cfg), 16, mem, 4096, C.byref(h)) == EINVAL
    with pytest.raises(vd.Vdl2GpuError, match="VDL2GPU_FLAG_RAGGED"):
        vd.Vdl2Receivers(2100000, 20, vd.FMT_U8, [(136975000, [136975000])], flags=vd.FLAG_RAGGED)


def test_ragged_calls_refuse_without_a_context():
    L = vd.load_library()
    n = np.zeros(2, np.uint32)
    assert L.vdl2gpu_submit_ragged(None, None, n.ctypes.data) == EINVAL
    assert L.vdl2gpu_submit_ragged_device(None, None, n.ctypes.data, None) == EINVAL
    assert L.vdl2gpu_get_receiver_positions(None, n.ctypes.data, 1) == EINVAL


def test_valid_ragged_configurations_reach_the_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = vd.load_library()
    fr = [136975000, 136700000, 136725000]
    a = (api._ReceiverEx * 2)()
    for k, (cf, nc, os_, fmt) in enumerate([(136975000, 1, 10, 0), (136700000, 2, 20, 1)]):
        a[k].centerfreq, a[k].n_channels, a[k].oversample, a[k].sample_fmt = cf, nc, os_, fmt
    for flags in (vd.FLAG_RAGGED, vd.FLAG_RAGGED | vd.FLAG_NO_GRAPH | vd.FLAG_TRACE):
        cfg, _k = _cfg(fr, flags)
        h = C.c_void_p()
        assert L.vdl2gpu_create_mixed_receivers(C.byref(cfg), a, 2, C.byref(h)) == ENODEV
    with pytest.raises(vd.Vdl2GpuError, match="no usable CUDA device"):
        vd.Vdl2MixedReceivers([(136975000, [136975000], 13, vd.FMT_U8), (136500000, [136525000], 13, vd.FMT_S16)], ragged=True)


def test_python_checks_whole_groups_before_the_library():
    """submit_ragged refuses a buffer that is not a whole number of decimation groups (ValueError) before any call"""
    g = vd.Vdl2MixedReceivers.__new__(vd.Vdl2MixedReceivers)
    g.n_receivers, g.bytes_per_dec = 2, [20, 80]
    with pytest.raises(ValueError, match="receiver 1"):
        g.submit_ragged([np.zeros(40, np.uint8), np.zeros(81, np.uint8)])
    with pytest.raises(ValueError, match="receiver 0"):
        g.submit_ragged([np.zeros(19, np.uint8), np.zeros(0, np.uint8)])
    with pytest.raises(ValueError, match="3 buffers"):
        g.submit_ragged([np.zeros(20, np.uint8)] * 3)
