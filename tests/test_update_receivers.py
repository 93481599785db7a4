"""CPU: receivers joining and leaving a ragged mixed-receivers context (vdl2gpu_update_receivers,
Vdl2MixedReceivers.update_receivers / add_receivers / remove_receivers) without a GPU.  The slot map of vdl2_core.cuh
compiled for the host (tests/hostsim/update_receivers.cpp, TEST-ONLY) is stepped over adding, removing and reordering
receivers, one-channel receivers, and lists that cross the balanced slot mapping's threshold (8448 channels on 132 SMs)
both ways: every kept channel must map to its own old slot, its counters to its own old channel, and nothing else to an
old slot.  Then the refusal that needs no device and the Python ValueErrors."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
import dumpvdl2_b200 as vd

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "dumpvdl2_b200", "csrc")
EINVAL = -1
FRESH, NONE = -1, -2
SMS = 132


@pytest.fixture(scope="module")
def um(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("update") / "libupdate.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I", CSRC, "-o", so, os.path.join(HERE, "hostsim", "update_receivers.cpp")])
    L = C.CDLL(so)
    L.update_slot_map.argtypes = [C.c_uint32] * 4 + [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 3
    L.update_slot_channel.argtypes = [C.c_uint32] * 4 + [C.POINTER(C.c_uint32)]
    L.update_migrate_entry_bytes.restype = C.c_size_t
    return L


def _layout(n_ch):
    """(n_chp, lanes, full_warps) of create's slot mapping for n_ch channels of a receivers context on 132 SMs"""
    w = 4 * SMS
    if 16 * w < n_ch <= 32 * w:
        lanes = (n_ch + w - 1) // w
        return w * 32, lanes, n_ch - (lanes - 1) * w
    return (n_ch + 31) // 32 * 32, 32, 0xFFFFFFFF


def _first(counts):
    return np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)


def _slots(um, n_ch):
    """channel -> slot of the layout, from the slot -> channel function the kernels use"""
    n_chp, lanes, fw = _layout(n_ch)
    out = {}
    ch = C.c_uint32(0)
    for s in range(n_chp):
        if um.update_slot_channel(s, lanes, fw, n_ch, C.byref(ch)):
            out[ch.value] = s
    assert sorted(out) == list(range(n_ch))
    return out


def _check(um, old_counts, new_counts, from_):
    old_first, new_first = _first(old_counts), _first(new_counts)
    n_old, n_new = int(old_first[-1]), int(new_first[-1])
    n_chp, lanes, fw = _layout(n_new)
    _, olanes, ofw = _layout(n_old)
    fr = np.ascontiguousarray(from_, np.int32)
    slot_from, chan_from = np.zeros(n_chp, np.int32), np.zeros(n_chp, np.int32)
    um.update_slot_map(n_chp, lanes, fw, n_new, new_first.ctypes.data, len(new_counts), fr.ctypes.data, olanes, ofw,
                       old_first.ctypes.data, slot_from.ctypes.data, chan_from.ctypes.data)
    old_slot, new_slot = _slots(um, n_old), _slots(um, n_new)
    want_slot = np.full(n_chp, NONE, np.int64)
    want_chan = np.full(n_chp, -1, np.int64)
    for r, k in enumerate(from_):
        for j in range(new_counts[r]):
            ch = int(new_first[r]) + j
            if k < 0:
                want_slot[new_slot[ch]] = FRESH
            else:
                assert new_counts[r] == old_counts[k]
                want_slot[new_slot[ch]] = old_slot[int(old_first[k]) + j]
                want_chan[ch] = int(old_first[k]) + j
    assert slot_from.tolist() == want_slot.tolist()
    assert chan_from.tolist() == want_chan.tolist()
    kept = slot_from[slot_from >= 0]
    assert np.unique(kept).size == kept.size                    # nothing else maps to an old slot
    kept_old = {old_slot[int(old_first[k]) + j] for k in from_ if k >= 0 for j in range(old_counts[k])}
    assert set(kept.tolist()) == kept_old
    return lanes


def test_migrate_entry_is_20_bytes(um):
    assert um.update_migrate_entry_bytes() == 20


@pytest.mark.parametrize("case", ["grow", "shrink", "reorder", "swap_kind", "one_channel", "drop_first", "drop_last", "replace_all"])
def test_slot_map_small_fleets(um, case):
    old = [3, 8, 1, 33, 5, 1, 64, 2]
    n = len(old)
    if case == "grow":
        new, src = old[:3] + [7, 1] + old[3:] + [40], [0, 1, 2, -1, -1, 3, 4, 5, 6, 7, -1]
    elif case == "shrink":
        new, src = [old[k] for k in (0, 3, 6)], [0, 3, 6]
    elif case == "reorder":
        src = [7, 2, 5, 0, 6, 1, 4, 3]
        new = [old[k] for k in src]
    elif case == "swap_kind":                                    # receiver 3 removed, a new one of another kind in its place
        new, src = old[:3] + [12] + old[4:], [0, 1, 2, -1, 4, 5, 6, 7]
    elif case == "one_channel":
        new, src = [1, 1, 1, 1], [5, -1, 2, -1]
    elif case == "drop_first":
        new, src = old[1:], list(range(1, n))
    elif case == "drop_last":
        new, src = old[:-1], list(range(n - 1))
    else:
        new, src = [4, 4], [-1, -1]
    _check(um, old, new, src)


def test_slot_map_crosses_the_balanced_threshold_both_ways(um):
    """1050 receivers x 8 = 8400 channels (32 lanes per warp), + 10 receivers = 8480 > 8448 (balanced, 17 lanes), then
    back under it by removing 11 receivers, including the first and the last"""
    old = [8] * 1050
    assert _check(um, old, old, list(range(1050))) == 32
    grown = old[:500] + [8] * 10 + old[500:]
    src_grow = list(range(500)) + [-1] * 10 + list(range(500, 1050))
    assert _check(um, old, grown, src_grow) == 17
    gone = {0, 1059, 3, 250, 503, 700, 701, 702, 900, 1000, 1058}
    keep = [k for k in range(1060) if k not in gone]
    assert _check(um, grown, [grown[k] for k in keep], keep) == 32
    # 2048 x 8 = 16384 (balanced, 32 or 31 lanes) + 72 receivers: 16960 > 16896 leaves the balanced mapping
    big = [8] * 2048
    assert _check(um, big, big + [8] * 72, list(range(2048)) + [-1] * 72) == 32
    assert _check(um, big + [8] * 72, big[:-1], list(range(2047))) == 32       # 16376 channels: balanced again, 32 or 31 lanes


# ---- refusals that need no device ----
def test_update_refuses_without_a_context():
    L = vd.load_library()
    rx = (vd.api._ReceiverEx * 1)()
    rx[0].centerfreq, rx[0].n_channels, rx[0].oversample, rx[0].sample_fmt = 136500000, 1, 10, 0
    fr = np.array([136525000], np.uint32)
    src = np.array([-1], np.int32)
    assert L.vdl2gpu_update_receivers(None, rx, src.ctypes.data, 1, fr.ctypes.data) == EINVAL
    assert "no context" in L.vdl2gpu_last_error().decode()
    assert L.vdl2gpu_update_receivers(None, None, None, 0, None) == EINVAL


def _detached(receivers):
    """a Vdl2MixedReceivers with the bookkeeping update_receivers checks, but no library context behind it"""
    g = vd.Vdl2MixedReceivers.__new__(vd.Vdl2MixedReceivers)
    g.L, g.h = None, None
    g._describe(vd.Vdl2MixedReceivers._normalise(receivers))
    return g


FLEET = [(136500000, [136525000, 136550000], 10, vd.FMT_U8), (136900000, [136975000], 20, vd.FMT_S16),
         (137100000, [137100000], 13, vd.FMT_U8)]


@pytest.mark.parametrize("args,msg", [
    (([FLEET[0]], [0, 1]), "2 entries in from_ for 1 receivers"),
    (([], []), "no receivers"),
    (([FLEET[0], FLEET[1]], [0, 3]), "entry 1 continues receiver 3 of 3"),
    (([FLEET[0], FLEET[1]], [0, -2]), "entry 1 continues receiver -2 of 3"),
    (([FLEET[0], FLEET[0]], [0, 0]), "entry 1 continues receiver 0, which an earlier entry continues"),
    (([(136500000, [136550000, 136525000], 10, vd.FMT_U8)], [0]), "entry 0 does not repeat receiver 0's description"),
    (([(136500000, [136525000, 136550000], 20, vd.FMT_U8)], [0]), "entry 0 does not repeat receiver 0's description"),
    (([(136900000, [136975000], 20, vd.FMT_U8)], [1]), "entry 0 does not repeat receiver 1's description"),
    (([FLEET[2], (136800000, [136975000], 20, vd.FMT_S16)], [2, 1]), "entry 1 does not repeat receiver 1's description"),
])
def test_python_checks_update_before_the_library(args, msg):
    g = _detached(FLEET)
    with pytest.raises(ValueError, match=msg):
        g.update_receivers(*args)
    assert g.n_receivers == 3 and g.freqs.tolist() == [136525000, 136550000, 136975000, 137100000]      # nothing changed


def test_python_checks_add_and_remove_before_the_library():
    g = _detached(FLEET)
    with pytest.raises(ValueError, match="position 4 of 3 receivers"):
        g.add_receivers([FLEET[0]], at=4)
    with pytest.raises(ValueError, match="position -1 of 3 receivers"):
        g.add_receivers([FLEET[0]], at=-1)
    with pytest.raises(ValueError, match="receiver 3 of 3"):
        g.remove_receivers([0, 3])
    with pytest.raises(ValueError, match="no receivers"):
        g.remove_receivers([0, 1, 2])
    assert g.n_receivers == 3 and g.receivers[0] == (136500000, [136525000, 136550000])
