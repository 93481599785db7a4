"""CPU: receivers of different sample rates and formats in one context (vdl2gpu_create_mixed_receivers) without a GPU -
every malformed configuration is refused with VDL2GPU_EINVAL before the device is touched - and the span layout and tile
sizing functions of vdl2_core.cuh the context is built with, compiled for the host (tests/hostsim/layout_mixed.cpp, TEST-ONLY)."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import api

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "dumpvdl2_b200", "csrc")
EINVAL, ENODEV = -1, -2


@pytest.fixture(scope="module")
def lay(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("layout_mixed") / "liblayout.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I", CSRC, "-o", so, os.path.join(HERE, "hostsim", "layout_mixed.cpp")])
    L = C.CDLL(so)
    u32 = C.c_uint32
    for n in ("layout_rx_mixed_tile_groups", "layout_rx_mixed_smem_max", "layout_rx_class", "layout_rx_k1_smem_bytes",
              "layout_rx_k1_smem_budget", "layout_rx_tile_stride"):
        getattr(L, n).restype = u32
    L.layout_rx_span_offsets.restype = C.c_uint64
    L.layout_rx_span_offsets.argtypes = [C.c_void_p, C.c_void_p, u32, u32, C.c_void_p]
    return L


@pytest.mark.parametrize("os_max", [10, 13, 20])
def test_tile_groups_are_the_largest_even_count_within_the_budget(lay, os_max):
    budget = lay.layout_rx_k1_smem_budget()
    assert budget == 110 * 1024
    last = None
    for g in range(1, 129):
        tg = lay.layout_rx_mixed_tile_groups(g, os_max)
        assert tg >= 2 and tg % 2 == 0, (g, tg)
        smem = lay.layout_rx_k1_smem_bytes(g, tg * os_max)
        assert lay.layout_rx_tile_stride(tg * os_max) >= tg * os_max
        if smem > budget:
            # only where not even two groups fit: 100 or more receivers of oversample 20 in one block
            assert tg == 2 and os_max == 20 and g >= 100, (g, tg, smem)
            assert smem <= lay.layout_rx_mixed_smem_max()
        assert lay.layout_rx_k1_smem_bytes(g, (tg + 2) * os_max) > budget, (g, tg)    # the largest such count
        assert last is None or tg <= last
        last = tg
    assert lay.layout_rx_mixed_tile_groups(128, 20) == 2
    assert lay.layout_rx_mixed_smem_max() == lay.layout_rx_k1_smem_bytes(128, 40) <= 227 * 1024


def test_rate_classes(lay):
    assert [lay.layout_rx_class(o) for o in (10, 13, 20)] == [0, 1, 2]


def _offsets(lay, os_, fmt, n_dec):
    os_ = np.ascontiguousarray(os_, np.uint32)
    fmt = np.ascontiguousarray(fmt, np.uint32)
    off = np.zeros(os_.size, np.uint64)
    per_dec = lay.layout_rx_span_offsets(os_.ctypes.data, fmt.ctypes.data, os_.size, n_dec, off.ctypes.data)
    return per_dec, off


@pytest.mark.parametrize("n_dec", [1, 7, 13107, 65535])
def test_span_offsets_of_a_ragged_mix(lay, n_dec):
    mix = [(10, 0), (20, 1), (13, 0), (20, 0), (10, 1), (13, 1), (13, 0)]
    os_, fmt = [m[0] for m in mix], [m[1] for m in mix]
    per_dec, off = _offsets(lay, os_, fmt, n_dec)
    widths = [o * (4 if f else 2) for o, f in mix]
    assert per_dec == sum(widths)
    assert off.tolist() == [n_dec * sum(widths[:r]) for r in range(len(mix))]


def test_span_offsets_need_64_bits(lay):
    """65535 cs16 receivers at oversample 20 at the largest span 1 MiB allows (13107 decimated samples): the last buffer
    starts 65534 x 13107 x 80 bytes in, far beyond 4 GiB"""
    n, n_dec = 65535, (1 << 20) // 80
    per_dec, off = _offsets(lay, [20] * n, [1] * n, n_dec)
    assert per_dec == 80 * n
    assert int(off[-1]) == (n - 1) * n_dec * 80 > 1 << 32
    assert np.array_equal(off, np.arange(n, dtype=np.uint64) * np.uint64(n_dec * 80))


def test_receiver_struct_is_16_bytes():
    assert C.sizeof(api._ReceiverEx) == 16
    assert [f for f, _ in api._ReceiverEx._fields_] == ["centerfreq", "n_channels", "oversample", "sample_fmt"]


# ---- vdl2gpu_create_mixed_receivers argument checks (no GPU needed) ----
FREQS3 = (136975000, 136700000, 136725000)


def _cfg(freqs=(136975000,), n_streams=0, flags=0, **per_rx):
    fr = np.ascontiguousarray(freqs, np.uint32)
    cfg = api._Config()
    cfg.n_channels, cfg.freqs = fr.size, fr.ctypes.data_as(C.POINTER(C.c_uint32))
    cfg.device, cfg.flags, cfg.n_streams = -1, flags, n_streams
    for k, v in per_rx.items():
        setattr(cfg, k, v)
    return cfg, fr


def _rx(*quads):
    a = (api._ReceiverEx * max(len(quads), 1))()
    for k, (cf, n, os_, fmt) in enumerate(quads):
        a[k].centerfreq, a[k].n_channels, a[k].oversample, a[k].sample_fmt = cf, n, os_, fmt
    return a


def _create(cfg, rx, n_rx):
    L = vd.load_library()
    h = C.c_void_p()
    rc = L.vdl2gpu_create_mixed_receivers(C.byref(cfg), rx, n_rx, C.byref(h))
    return rc, L.vdl2gpu_last_error().decode()


ONE = (136975000, 1, 20, 1)


@pytest.mark.parametrize("what,kw,rx,n_rx,msg", [
    ("no receivers", {}, _rx(ONE), 0, "no receivers"),
    ("null receivers", {}, None, 1, "no receivers"),
    ("oversample 8", {}, _rx((136975000, 1, 8, 0)), 1, "oversample 8"),
    ("oversample 0", {}, _rx((136975000, 1, 0, 0)), 1, "oversample 0"),
    ("oversample 26", dict(freqs=FREQS3), _rx((136975000, 1, 10, 0), (136700000, 2, 26, 1)), 2, "receiver 1: oversample 26"),
    ("format 2", {}, _rx((136975000, 1, 10, 2)), 1, "sample format 2"),
    ("empty receiver", dict(freqs=FREQS3), _rx((136975000, 1, 10, 0), (136700000, 0, 20, 1), (136700000, 2, 20, 1)), 3,
     "receiver 1 has no channels"),
    ("sum too small", dict(freqs=FREQS3), _rx((136975000, 1, 10, 0), (136700000, 1, 20, 1)), 2, "add up"),
    ("sum too large", dict(freqs=FREQS3), _rx((136975000, 2, 10, 0), (136700000, 2, 20, 1)), 2, "add up"),
    ("n_streams", dict(freqs=FREQS3, n_streams=3), _rx((136975000, 1, 10, 0), (136700000, 2, 20, 1)), 2, "n_streams"),
    ("sample_rate", dict(sample_rate=2100000), _rx(ONE), 1, "must be 0"),
    ("cfg oversample", dict(oversample=20), _rx(ONE), 1, "must be 0"),
    ("cfg format", dict(sample_fmt=1), _rx(ONE), 1, "must be 0"),
    ("cfg centre", dict(centerfreq=136975000), _rx(ONE), 1, "must be 0"),
    ("k1 scalar", dict(flags=vd.FLAG_K1_SCALAR), _rx(ONE), 1, "K1_SCALAR"),
    ("no channels", dict(freqs=()), _rx(ONE), 1, "no channels"),
])
def test_bad_mixed_configurations_are_refused(what, kw, rx, n_rx, msg):
    cfg, _keep = _cfg(**kw)
    rc, err = _create(cfg, rx, n_rx)
    assert rc == EINVAL, what
    assert msg in err and "vdl2gpu_create_mixed_receivers" in err, err


def test_more_receivers_than_k0_grid_rows_are_refused():
    n = 65536
    cfg, _keep = _cfg(freqs=[136975000] * n)
    rc, err = _create(cfg, _rx(*[ONE] * n), n)
    assert rc == EINVAL and "65535" in err


def test_valid_mixed_configurations_reach_the_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    for n_streams in (0, 2):
        cfg, _keep = _cfg(freqs=FREQS3, n_streams=n_streams)
        assert _create(cfg, _rx((136975000, 1, 10, 0), (136700000, 2, 20, 1)), 2)[0] == ENODEV
    cfg, _keep = _cfg(freqs=FREQS3)
    assert _create(cfg, _rx((136975000, 1, 13, 0), (136700000, 1, 13, 1), (136700000, 1, 10, 1)), 3)[0] == ENODEV
    with pytest.raises(vd.Vdl2GpuError, match="no usable CUDA device"):
        vd.Vdl2MixedReceivers([(136975000, [136975000, 137000000], 10, vd.FMT_U8), (136500000, [136525000], 20, vd.FMT_S16)])
    with pytest.raises(vd.Vdl2GpuError, match="invalid argument"):
        vd.Vdl2MixedReceivers([(136975000, [136975000], 10, vd.FMT_U8), (136500000, [136525000], 16, vd.FMT_S16)])


def test_spans_need_a_receivers_context():
    L = vd.load_library()
    assert L.vdl2gpu_submit_span(None, None, 0) == EINVAL
    assert L.vdl2gpu_submit_span_device(None, None, 0, None) == EINVAL
