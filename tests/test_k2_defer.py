"""CPU: the default K2 walk slices a burst's data symbols after the block loop (vdl2_defer in vdl2_core.cuh) instead of
inline.  A host build of the device functions (tests/hostsim/defer.cpp, TEST-ONLY) runs the walk both ways, launch by
launch, and after every launch every field of every channel, the phase rings, the whole burst pool, the free list, the
queue counters and the events must be equal.  The schedules and pool sizes put the deferred path's own cases in reach: a
burst ending on every offset of a block and in the per-sample tail, a burst completing on a launch's last sample, bursts
spanning many launches and one-sample launches inside a burst, more bursts per channel and launch than the queue holds,
and bursts without a pool slot."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from tests import k2_corpus as kc

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "dumpvdl2_b200", "csrc")
STATS = ["end_at_block_offset_%d" % k for k in range(12)] + ["end_in_tail", "queued", "sliced_at_once", "no_pool_slot",
                                                              "open_completed_on_last_sample"]

# (stage, channels, launch schedule, pool slots or None for the usual 3 per channel + 16)
CASES = {
    "main": ("main", None, kc.LAUNCHES, None),
    "ppm": ("ppm", None, kc.LAUNCHES, None),
    "long": ("long", None, kc.LAUNCHES, None),
    # a launch of a whole stage: back-to-back bursts overrun the one-burst queue
    "main_one_launch": ("main", 256, (8000,), None),
    "long_one_launch": ("long", None, (60000,), None),
    # one-sample launches (and a few longer ones), so that a burst spans hundreds of launches
    "main_one_sample_launches": ("main", 64, (1,) * 30 + (37,), None),
    # launches around the symbol period and the block
    "main_short_launches": ("main", 128, (9, 10, 11, 12, 13, 19, 20, 21, 24, 25), None),
    # a pool of eight slots: most headers find it empty (slot = -1)
    "main_pool_overflow": ("main", 256, kc.LAUNCHES, 8),
}


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("defer") / "libdefer.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I", CSRC, "-o", so, os.path.join(HERE, "hostsim", "defer.cpp")])
    L = C.CDLL(so)
    L.hostsim_k2_defer_check.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_float, C.c_uint32,
                                         C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    return L


def _run(lib, case):
    """-> (first launch whose state differs or -1, its first differing channel or -1, {STATS name: count})"""
    name, n_ch, launches, n_slots = CASES[case]
    s = kc.stage(name)
    dec, freqs = s["dec"], s["freqs"]
    if n_ch is not None:
        dec, freqs = dec[:, :n_ch], freqs[:n_ch]
    d = np.ascontiguousarray(dec, np.float32)
    f = np.ascontiguousarray(freqs, np.uint32)
    sched = np.ascontiguousarray(launches, np.uint32)
    stats = np.zeros(len(STATS), np.uint64)
    bad_ch = C.c_int32(-1)
    bad = lib.hostsim_k2_defer_check(d.ctypes.data, d.shape[0], d.shape[1], f.ctypes.data, 2100000, s["max_ppm"],
                                     n_slots if n_slots is not None else 3 * d.shape[1] + 16, sched.ctypes.data, sched.size,
                                     stats.ctypes.data, C.byref(bad_ch))
    return bad, bad_ch.value, dict(zip(STATS, (int(x) for x in stats)))


@pytest.mark.parametrize("case", list(CASES))
def test_deferred_data_symbols_leave_every_launch_as_the_inline_walk(lib, case):
    bad, ch, stats = _run(lib, case)
    print(case, stats)
    assert bad == -1, f"{case}: launch {bad} differs (channel {ch})"
    assert stats["queued"] > 0


def test_deferred_walk_reaches_its_own_cases(lib):
    """the cases above hit every way a deferred burst can end"""
    total = {}
    for case in CASES:
        for k, v in _run(lib, case)[2].items():
            total[k] = total.get(k, 0) + v
    print(total)
    empty = [k for k, v in total.items() if v == 0]
    assert not empty, f"not reached: {empty}"
