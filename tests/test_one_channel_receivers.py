"""CPU: the fleets of one-channel receivers of test_gpu_one_channel_receivers.py reach the K1 shapes they are there to
test - G = 128 receivers per block, tiles of one decimation group (T = 20 / 26 / 30), two-group tiles of the mixed and
ragged kernels above the shared-memory budget (VDL2_RX_MIXED_SMEM_MAX), G >= 124 under the balanced mapping - computed
with the layout and sizing functions of vdl2_core.cuh compiled for the host (tests/hostsim/layout.cpp and
layout_mixed.cpp, TEST-ONLY), so that a change to the sizing rules cannot quietly turn those tests into easy ones.  The
fleet builders and chunk and span schedules are rehearsed at a tiny size against the oracle."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from oracle import pyoracle as po
from tests.test_gpu_mixed_receivers import KINDS, SIZES
from tests.test_receivers import _slot_mapping, _tables
from tests import test_gpu_one_channel_receivers as oc

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "dumpvdl2_b200", "csrc")


def _compile(tmp_path_factory, name):
    so = str(tmp_path_factory.mktemp(name) / "liblayout.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I", CSRC, "-o", so, os.path.join(HERE, "hostsim", f"{name}.cpp")])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def lay(tmp_path_factory):
    L = _compile(tmp_path_factory, "layout")
    u32 = C.c_uint32
    L.layout_slot_channel.argtypes = [u32, u32, u32, u32, C.POINTER(u32)]
    L.layout_rx_tables.restype = u32
    L.layout_rx_tables.argtypes = [u32, u32, u32, u32, C.c_void_p, u32, C.c_void_p, C.c_void_p]
    for n in ("layout_rx_tile_samples", "layout_rx_tile_stride", "layout_rx_k1_smem_bytes", "layout_rx_k1_smem_budget"):
        getattr(L, n).restype = u32
    return L


@pytest.fixture(scope="module")
def laym(tmp_path_factory):
    L = _compile(tmp_path_factory, "layout_mixed")
    for n in ("layout_rx_mixed_tile_groups", "layout_rx_mixed_smem_max", "layout_rx_k1_smem_bytes", "layout_rx_k1_smem_budget"):
        getattr(L, n).restype = C.c_uint32
    return L


def _blocks(lay, sizes):
    """G of every block with channels, and the largest"""
    first, lanes, slot_rx, block_rx, g_max, chan = _tables(lay, sizes)
    return [int(g) for g in block_rx[:, 1] if g], int(g_max)


def _mixed_tile(laym, g_max, os_max):
    tg = laym.layout_rx_mixed_tile_groups(g_max, os_max)
    return tg, laym.layout_rx_k1_smem_bytes(g_max, tg * os_max)


# ---- the shapes the GPU fleets reach ----
@pytest.mark.parametrize("os_", [20, 13, 10])
def test_groups_fleet_has_128_receivers_per_block_and_one_group_tiles(lay, os_):
    gs, g_max = _blocks(lay, [1] * oc.N_FLEET)
    assert gs == [128, 128, 44] and g_max == 128
    t = lay.layout_rx_tile_samples(g_max, os_)
    assert t == oc.TILE[os_] == {20: 20, 13: 26, 10: 30}[os_]
    assert t // os_ == (1 if os_ == 20 else 2 if os_ == 13 else 3)
    assert lay.layout_rx_k1_smem_bytes(g_max, t) <= lay.layout_rx_k1_smem_budget()
    # rows past 32: warp 0 issues four bulk copies per lane
    assert (g_max + 31) // 32 == 4


def test_mixed_and_ragged_fleet_take_two_groups_over_the_budget(lay, laym):
    kinds_of = [KINDS[r % len(KINDS)] for r in range(oc.N_FLEET)]
    assert max(o for o, _ in kinds_of) == 20
    gs, g_max = _blocks(lay, [1] * oc.N_FLEET)            # one channel each: the grouped order has the same blocks
    assert g_max == 128
    tg, smem = _mixed_tile(laym, g_max, 20)
    assert tg == 2 and smem == laym.layout_rx_mixed_smem_max() == 135312 > laym.layout_rx_k1_smem_budget()
    # every block of 128 interleaved receivers holds all five kinds; the grouped order puts the rate boundaries inside blocks
    for b in range(2):
        assert set(kinds_of[128 * b:128 * (b + 1)]) == set(KINDS)
    grouped = sorted(kinds_of)
    assert any(len(set(o for o, _ in grouped[128 * b:128 * (b + 1)])) > 1 for b in range(3))


def test_balanced_fleets_have_124_to_128_receivers_per_block(lay, laym):
    lanes, full, n_chp = _slot_mapping(oc.BALANCED)
    assert (lanes, full) == (32, 16)
    gs, g_max = _blocks(lay, [1] * oc.BALANCED)
    assert set(gs) == {124, 128} and g_max == 128 and len(gs) == 132
    assert lay.layout_rx_tile_samples(g_max, 20) == 20
    tg, smem = _mixed_tile(laym, g_max, 20)                # the alternating (10, cu8) / (20, cs16) ragged fleet
    assert tg == 2 and smem == laym.layout_rx_mixed_smem_max()
    # the sampled receivers sit where they say: slot of channel c
    slot = {}
    c = C.c_uint32()
    for s in range(n_chp):
        if lay.layout_slot_channel(s, lanes, full, oc.BALANCED, C.byref(c)):
            slot[c.value] = s
    warp = {r: slot[r] // 32 for r in oc.BALANCED_SAMPLE}
    block = {r: slot[r] // 128 for r in oc.BALANCED_SAMPLE}
    assert (block[127], block[128]) == (0, 1)
    assert (warp[511], warp[512], block[511], block[512]) == (15, 16, 3, 4)
    assert (warp[542], warp[543]) == (16, 17) and slot[543] == 17 * 32
    assert (block[635], block[636]) == (4, 5)
    assert block[8191] != block[0] and block[16383] == 131


def test_join_goes_from_a_multi_group_tile_to_two_groups_over_the_budget(lay, laym):
    before = list(SIZES)
    _, g0 = _blocks(lay, before)
    tg0, smem0 = _mixed_tile(laym, g0, 20)
    assert tg0 > 2 and smem0 <= laym.layout_rx_k1_smem_budget()
    kept = [n for k, n in enumerate(SIZES) if k not in (3, 7)]
    after = [1] * 100 + kept + [1] * 100
    gs, g1 = _blocks(lay, after)
    assert g1 >= 100
    tg1, smem1 = _mixed_tile(laym, g1, 20)
    assert tg1 == 2 and laym.layout_rx_k1_smem_budget() < smem1 <= laym.layout_rx_mixed_smem_max()


def test_lanes_fleets(lay):
    assert _slot_mapping(40)[:2] == (32, 0xFFFFFFFF)
    assert _slot_mapping(9600)[:2] == (19, 9600 - 18 * 528)
    gs, g_max = _blocks(lay, [1] * 40)                      # the same streams as 40 one-channel receivers
    assert gs == [40] and g_max == 40                       # one block, rows past 32


# ---- the schedules have the edges they are meant to have ----
@pytest.mark.parametrize("os_", [20, 13, 10])
def test_chunk_schedule_edges(os_):
    chunks = oc.chunk_schedule(os_)
    tg = oc.TILE[os_] // os_
    s, seen = 0, set()
    for n in chunks:
        cnt0 = s % os_
        head = min(n, (os_ - cnt0) % os_)
        groups = (n - head) // os_
        tail = n - head - groups * os_
        if n % 2:
            seen.add("odd")
        if groups == 0 and tail == 0 and head == n:
            seen.add("head only")
        if n > os_ and n < oc.TILE[os_] and groups < tg:
            seen.add("under a tile")
        if groups:
            seen.add(f"mis {head & 1}")
        if (s + n) % os_:
            seen.add("mid-group end")
        s += n
    assert chunks[-1] < 1000 and max(chunks) == 65537
    want = {"odd", "head only", "mis 0", "mis 1", "mid-group end"} | ({"under a tile"} if tg > 1 else set())
    assert want <= seen, want - seen


def test_span_schedules_edges():
    assert {1, 2, 3, 7, oc.W} <= set(oc.mixed_spans()) and oc.W % 2 == 1
    spans = oc.ragged_spans(oc.N_FLEET, 0x4F52)
    a = np.asarray(spans)
    assert a.max() == oc.W and a.min() == 0 and (a == oc.W).all(axis=1).any()
    assert all(((a[:, r] == 0).sum() >= 3) for r in range(4, oc.N_FLEET, 11))               # absent for whole spans
    assert {0, 1, 2, 3} <= set(a.ravel().tolist()) and (a % 2 == 1).any()
    one = [k for k in range(len(spans)) if (a[k, :128] > 0).sum() == 1]                     # one receiver of block 0
    assert one and a[one[0], oc.ALONE] == 3 and a[one[0], 128:].max() > 0
    assert all(a[oc.RESTART_SPAN, r] == 0 for r in oc.IDLE_AT_RESTART)
    assert all(a[:oc.RESTART_SPAN, r].sum() > 0 for r in oc.RESTARTED)
    c = oc.balanced_counts(oc.BALANCED, 4, 2000, 0x4F47)
    assert c.max() == 2000 and 0.08 < (c == 0).mean() < 0.15


# ---- the builders and schedules at a tiny size, against the oracle ----
def test_lockstep_builder_and_chunk_positions():
    torch = pytest.importorskip("torch")
    os_ = 13
    F = oc.one_channel_fleet([(os_, "u8")] * 5, 0.05, 0x4F540000, per_group=False, on_centre=(1,))
    L = F["bases"][(os_, "u8")].shape[0]
    assert F["rx"][1]["freqs"] == [F["rx"][1]["centre"]] and F["rx"][2]["freqs"] != [F["rx"][2]["centre"]]
    assert [x["shift"] for x in F["rx"]] == [(7919 * r) % L for r in range(5)]
    chunks = [5000, 3, 25, 6500, 41]
    s0 = 0
    for n in chunks:
        buf = oc.pack_lockstep(F, s0, n, device="cpu")
        assert buf.shape == (5, n, 2) and buf.dtype == torch.uint8
        want = np.concatenate([oc.host_units(F, r, s0, s0 + n) for r in range(5)])
        assert np.array_equal(buf.numpy().reshape(-1), want)
        s0 += n
    # receiver 3's stream is the base rolled by 7919 x 3 samples
    base = F["bases"][(os_, "u8")].reshape(-1)
    assert np.array_equal(oc.host_units(F, 3, 0, L), np.roll(base, -2 * F["rx"][3]["shift"]))
    # the oracle fed chunk by chunk yields floor(S / os) decimated samples after S samples (the rows read_dec returns)
    o = po.Oracle(105000 * os_, os_, po.FMT_U8, F["rx"][2]["centre"], F["rx"][2]["freqs"], dec_tap=True)
    s0 = 0
    for n in chunks:
        o.process(oc.host_units(F, 2, s0, s0 + n))
        s0 += n
        assert o.dec_samples().shape == (s0 // os_, 1, 2)
    (whole,), bounds = oc.oracle(F, 2, chunks)
    assert bounds == [0, sum(chunks)]
    assert np.array_equal(whole.dec_samples().view(np.uint32), o.dec_samples().view(np.uint32))


def test_span_builder_and_segmented_oracles():
    torch = pytest.importorskip("torch")
    F = oc.one_channel_fleet([KINDS[r % len(KINDS)] for r in range(7)], 0.05, 0x4F550000, per_group=True)
    widths = [x["os"] * (4 if x["fmt"] == "s16" else 2) for x in F["rx"]]
    assert [F["bases"][(x["os"], x["fmt"])].shape[1] for x in F["rx"]] == widths
    spans = [[3] * 7, [0, 1, 2, 0, 5, 0, 7], [0] * 7, [11, 0, 0, 0, 0, 0, 1]]
    pos = np.zeros(7, np.int64)
    for c in spans:
        buf = oc.pack_span(F, c, pos, device="cpu")
        assert buf.dtype == torch.uint8 and buf.numel() == sum(n * w for n, w in zip(c, widths))
        want = np.concatenate([oc.host_units(F, r, pos[r], pos[r] + c[r]) for r in range(7)])
        assert np.array_equal(buf.numpy(), want)
        pos += c
    # a restart after the first two spans: two oracles whose decimated samples make up the receiver's stream
    r = 4
    per = [s[r] for s in spans]
    (a, b), bounds = oc.oracle(F, r, per, cuts=[sum(per[:2])])
    assert bounds == [0, 8, 8] and a.dec_samples().shape[0] == 8 and b.dec_samples().shape[0] == 0
    assert oc.oracle_dec([a, b]).shape == (8, 1, 2)
