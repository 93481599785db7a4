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
                                                              "open_completed_on_last_sample", "end_on_last_sample_but_one",
                                                              "last_symbol_on_next_first_sample", "two_ends_in_a_launch",
                                                              "three_ends_in_a_launch", "open_across_an_empty_span",
                                                              "one_sample_span_in_data"]

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
    for f in (L.hostsim_k2_defer_check, L.hostsim_k2_defer_check_spans):
        f.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_float, C.c_uint32, C.c_void_p, C.c_uint32,
                      C.c_void_p, C.c_void_p]
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
    """the cases above hit every way a deferred burst can end (an empty span takes per-receiver spans, below)"""
    total = {}
    for case in CASES:
        for k, v in _run(lib, case)[2].items():
            total[k] = total.get(k, 0) + v
    print(total)
    empty = [k for k, v in total.items() if v == 0 and k != "open_across_an_empty_span"]
    assert not empty, f"not reached: {empty}"


def test_ragged_deferral_plan_leaves_every_span_as_the_inline_walk_and_reaches_every_cell(lib):
    """k2_corpus.defer_spans: 64 one-receiver channels, each on its own span counts (zeros included), planned from the
    oracle's burst ends so that spans end on, one before and one after a burst's last symbol, come empty or one sample
    long while a burst is open, and hold two and three burst ends.  After every span the deferred walk leaves what the
    inline walk leaves, and every cell of the plan is reached."""
    oracles = kc.defer_oracles()
    dec = np.ascontiguousarray(np.concatenate([o.dec_samples() for o in oracles], axis=1), np.float32)
    freqs = np.ascontiguousarray([x["freqs"][0] for x in kc.defer_fleet()], np.uint32)
    spans = np.ascontiguousarray(kc.defer_spans(oracles, [dec.shape[0]] * dec.shape[1]), np.uint32)
    stats = np.zeros(len(STATS), np.uint64)
    bad_ch = C.c_int32(-1)
    bad = lib.hostsim_k2_defer_check_spans(dec.ctypes.data, dec.shape[0], dec.shape[1], freqs.ctypes.data, 2100000, 0.0,
                                           3 * dec.shape[1] + 16, spans.ctypes.data, spans.shape[0], stats.ctypes.data,
                                           C.byref(bad_ch))
    cells = dict(zip(STATS, (int(x) for x in stats)))
    for k, v in cells.items():
        print(f"{k:40s} {v}")
    assert bad == -1, f"span {bad} differs (channel {bad_ch.value})"
    assert (spans == 0).any() and (spans == 1).any()
    empty = [k for k, v in cells.items() if v == 0 and k != "no_pool_slot"]
    assert not empty, f"not reached: {empty}"
