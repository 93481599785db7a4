"""CPU: the multi-receiver context (vdl2gpu_create_receivers) without a GPU - every malformed configuration is refused
with VDL2GPU_EINVAL before the device is touched - and the layout functions of vdl2_core.cuh it builds its K1 tables
with, compiled for the host (tests/hostsim/layout.cpp, TEST-ONLY)."""
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
H100_SMS = 132


@pytest.fixture(scope="module")
def lay(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("layout") / "liblayout.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I", CSRC, "-o", so, os.path.join(HERE, "hostsim", "layout.cpp")])
    L = C.CDLL(so)
    u32 = C.c_uint32
    L.layout_slot_channel.argtypes = [u32, u32, u32, u32, C.POINTER(u32)]
    L.layout_rx_of_channel.restype = u32
    L.layout_rx_of_channel.argtypes = [u32, C.c_void_p, u32]
    L.layout_rx_tables.restype = u32
    L.layout_rx_tables.argtypes = [u32, u32, u32, u32, C.c_void_p, u32, C.c_void_p, C.c_void_p]
    for n in ("layout_rx_tile_samples", "layout_rx_tile_stride", "layout_rx_k1_smem_bytes", "layout_rx_k1_smem_budget"):
        getattr(L, n).restype = u32
    return L


def _slot_mapping(n_ch, n_sms=H100_SMS):
    """(lanes, full_warps, n_chp) as the context chooses them (create_impl): more than half a machine of warps' worth of
    channels are dealt out evenly over all 4 x SMs warps"""
    warps_all = 4 * n_sms
    if 16 * warps_all < n_ch <= 32 * warps_all:
        lanes = (n_ch + warps_all - 1) // warps_all
        return lanes, n_ch - (lanes - 1) * warps_all, warps_all * 32
    return 32, 0xFFFFFFFF, (n_ch + 31) // 32 * 32


def _tables(L, sizes):
    n_ch = int(sum(sizes))
    lanes, full, n_chp = _slot_mapping(n_ch)
    first = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    n_blocks = (n_chp + 127) // 128
    slot_rx = np.zeros(n_blocks * 128, np.uint32)
    block_rx = np.zeros((n_blocks, 2), np.uint32)
    g_max = L.layout_rx_tables(n_blocks, lanes, full, n_ch, first.ctypes.data, len(sizes), slot_rx.ctypes.data, block_rx.ctypes.data)
    chan = np.full(n_blocks * 128, -1, np.int64)
    c = C.c_uint32()
    for s in range(n_blocks * 128):
        if L.layout_slot_channel(s, lanes, full, n_ch, C.byref(c)):
            chan[s] = c.value
    return first, lanes, slot_rx, block_rx, g_max, chan


RAGGED = [1, 3, 8, 13, 32, 33, 40]


@pytest.mark.parametrize("sizes", [RAGGED, [8] * 2048, [1] * 9000, "random"], ids=["ragged7", "2048x8", "9000x1", "random"])
def test_every_active_slot_maps_to_its_channels_receiver(lay, sizes):
    if sizes == "random":
        sizes = list(np.random.default_rng(7).integers(1, 60, 400))            # ~12000 channels: balanced mapping, 23 per warp
    first, lanes, slot_rx, block_rx, g_max, chan = _tables(lay, sizes)
    n_ch = int(first[-1])
    active = chan >= 0
    assert sorted(chan[active].tolist()) == list(range(n_ch))                  # the slots hold every channel exactly once
    want_rx = np.searchsorted(first, chan[active], side="right") - 1
    assert np.array_equal(slot_rx[active], want_rx)
    for ch in (0, n_ch - 1) + tuple(first[1:-1]) + tuple(first[1:-1] - 1):
        assert lay.layout_rx_of_channel(int(ch), first.ctypes.data, len(sizes)) == np.searchsorted(first, ch, side="right") - 1
    gs = []
    for b in range(block_rx.shape[0]):
        mine = slot_rx[b * 128:(b + 1) * 128][active[b * 128:(b + 1) * 128]]
        if mine.size == 0:
            assert block_rx[b, 1] == 0
            continue
        assert (block_rx[b, 0], block_rx[b, 1]) == (mine.min(), mine.max() - mine.min() + 1), f"block {b}"
        # a block covers a contiguous channel range, so every receiver of its range has a channel in it
        assert set(mine.tolist()) == set(range(mine.min(), mine.max() + 1))
        assert (slot_rx[b * 128:(b + 1) * 128][~active[b * 128:(b + 1) * 128]] == block_rx[b, 0]).all()
        gs.append(int(block_rx[b, 1]))
    assert g_max == max(gs)


def test_block_ranges_at_the_balanced_mapping_warp_boundaries(lay):
    """2048 receivers x 8 channels on an H100: 16384 channels dealt over 528 warps, the first 16 with 32 channels, the rest
    31; a 4-warp block then spans 128 or 124 channels, i.e. 16 receivers, and every other 124-channel block starts and ends
    in the middle of a receiver."""
    first, lanes, slot_rx, block_rx, g_max, chan = _tables(lay, [8] * 2048)
    assert lanes == 32 and block_rx.shape[0] == H100_SMS
    for b in (0, 3, 4, 5, H100_SMS - 1):                # blocks 0-3 hold the 32-channel warps, block 4 the first 31-channel one
        ch = chan[b * 128:(b + 1) * 128]
        ch = ch[ch >= 0]
        assert ch.max() - ch.min() + 1 == ch.size == (128 if b < 4 else 124)
        assert block_rx[b, 0] == ch.min() // 8 and block_rx[b, 0] + block_rx[b, 1] - 1 == ch.max() // 8
    assert block_rx[4, 0] == 64 and chan[4 * 128] == 512
    assert chan[5 * 128] == 636 and block_rx[5, 0] == 79 and block_rx[4, 0] + block_rx[4, 1] - 1 == 79     # receiver 79 straddles
    assert block_rx[-1, 0] + block_rx[-1, 1] == 2048 and set(block_rx[:, 1].tolist()) == {16} and g_max == 16


@pytest.mark.parametrize("oversample", [20, 10, 13])
def test_tile_length_respects_the_shared_memory_budget(lay, oversample):
    budget = lay.layout_rx_k1_smem_budget()
    assert budget == 110 * 1024
    step = oversample if oversample % 2 == 0 else 2 * oversample
    last = None
    for g in range(1, 129):
        t = lay.layout_rx_tile_samples(g, oversample)
        assert t > 0 and t % oversample == 0 and t % 2 == 0, (g, t)
        r = lay.layout_rx_tile_stride(t)
        assert r >= t + 2 and r % 16 == 2
        assert lay.layout_rx_k1_smem_bytes(g, t) <= budget, (g, t)
        assert lay.layout_rx_k1_smem_bytes(g, t + step) > budget, (g, t)     # the largest such tile
        assert last is None or t <= last
        last = t


# ---- vdl2gpu_create_receivers argument checks (no GPU needed) ----
def _cfg(rate=2100000, os_=20, freqs=(136975000,), n_streams=0, flags=0):
    fr = np.ascontiguousarray(freqs, np.uint32)
    cfg = api._Config()
    cfg.sample_rate, cfg.oversample, cfg.sample_fmt, cfg.centerfreq = rate, os_, vd.FMT_U8, 0
    cfg.n_channels, cfg.freqs = fr.size, fr.ctypes.data_as(C.POINTER(C.c_uint32))
    cfg.device, cfg.flags, cfg.n_streams = -1, flags, n_streams
    return cfg, fr


def _rx(*pairs):
    a = (api._Receiver * max(len(pairs), 1))()
    for k, (cf, n) in enumerate(pairs):
        a[k].centerfreq, a[k].n_channels = cf, n
    return a


def _create(cfg, rx, n_rx):
    L = vd.load_library()
    h = C.c_void_p()
    rc = L.vdl2gpu_create_receivers(C.byref(cfg), rx, n_rx, C.byref(h))
    return rc, L.vdl2gpu_last_error().decode()


FREQS3 = (136975000, 136700000, 136725000)


@pytest.mark.parametrize("what,kw,rx,n_rx,msg", [
    ("no receivers", {}, _rx((136975000, 1)), 0, "no receivers"),
    ("null receivers", {}, None, 1, "no receivers"),
    ("empty receiver", dict(freqs=FREQS3), _rx((136975000, 1), (136700000, 0), (136700000, 2)), 3, "no channels"),
    ("sum too small", dict(freqs=FREQS3), _rx((136975000, 1), (136700000, 1)), 2, "add up"),
    ("sum too large", dict(freqs=FREQS3), _rx((136975000, 2), (136700000, 2)), 2, "add up"),
    ("n_streams", dict(freqs=FREQS3, n_streams=3), _rx((136975000, 1), (136700000, 2)), 2, "n_streams"),
    ("oversample 8", dict(rate=840000, os_=8), _rx((136975000, 1)), 1, "oversample"),
    ("k1 scalar", dict(flags=vd.FLAG_K1_SCALAR), _rx((136975000, 1)), 1, "K1_SCALAR"),
    ("bad rate", dict(rate=2000000), _rx((136975000, 1)), 1, "sample_rate"),
])
def test_bad_receiver_configurations_are_refused(what, kw, rx, n_rx, msg):
    cfg, _keep = _cfg(**kw)
    rc, err = _create(cfg, rx, n_rx)
    assert rc == EINVAL, what
    assert msg in err, err


def test_more_receivers_than_k0_grid_rows_are_refused():
    n = 65536
    cfg, _keep = _cfg(freqs=[136975000] * n)
    rc, err = _create(cfg, _rx(*[(136975000, 1)] * n), n)
    assert rc == EINVAL and "65535" in err


def test_valid_receiver_configurations_reach_the_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    for n_streams in (0, 2):
        cfg, _keep = _cfg(freqs=FREQS3, n_streams=n_streams)
        assert _create(cfg, _rx((136975000, 1), (136700000, 2)), 2)[0] == ENODEV
    cfg, _keep = _cfg(rate=1365000, os_=13)
    assert _create(cfg, _rx((136975000, 1)), 1)[0] == ENODEV
    with pytest.raises(vd.Vdl2GpuError, match="no usable CUDA device"):
        vd.Vdl2Receivers(2100000, 20, vd.FMT_U8, [(136975000, [136975000, 137000000]), (136500000, [136525000])])
    with pytest.raises(vd.Vdl2GpuError, match="invalid argument"):
        vd.Vdl2Receivers(2100000, 20, vd.FMT_U8, [(136975000, [136975000]), (136500000, [])])
