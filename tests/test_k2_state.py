"""CPU: the state a K2 launch leaves behind, in every walk form the kernels use.

A host build of the device functions (tests/hostsim/k2_state.cpp, TEST-ONLY) walks a whole stage of channels launch by
launch, in one walk form per run.  The simplest form, the plain per-sample step (vdl2_demod_step_pm), is the reference.
After every launch the other forms must leave the same state:
- every K2_* field of every channel, in the plane encoding of vdl2_chan_store, the slot number included;
- the 160 ring floats, and the phase history the next launch starts from;
- the queue counters, and every ready burst's header and words;
- for a channel inside a burst with a slot, the slot words written so far.
The forms are the blocked walks on the phase plane (two unwraps), the ring walks (inputs one block ahead, staged), the
default walk with data symbols sliced inline, and the default walk with data symbols sliced after the walk (vdl2_defer).
The same helper restates a stage's device layout, pinned here against vdl2gpu_stage_device_bytes; the device tests
(test_gpu_k2_state.py) read a stage's planes through it."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from tests import k2_corpus as kc
from tests import test_k2_defer as kd

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "dumpvdl2_b200", "csrc")
INCLUDE = os.path.join(HERE, "..", "include")
PER_SAMPLE, DEFAULT_INLINE, DEFERRED = 0, 5, 6
FORMS = {"block_twosum": 1, "block_table": 2, "ring_regs": 3, "ring_staged": 4, "default_inline": DEFAULT_INLINE,
         "deferred": DEFERRED}
K2 = dict(PREV_PHI=0, PREV_DPHI=1, DPHI=2, PHERR0=3, PHERR1=4, PHERR2=5, PPM=6, MAG_LP=7, MAG_NF=8, FRAME_PWR=9,
          RING_POS=10, SCLK=11, NFCNT=12, FRAME_PWR_CNT=13, STATE=14, ACC_LO=15, ACC_HI=16, NBITS=17, NEED_BITS=18,
          DATALEN=19, SYNDROME=20, SLOT=21, BURST_SEQ=22, SYNC_LO=23, SYNC_HI=24, FREQ=25, CNT_SYNC=26,
          CNT_HDR_GOOD=27, PURE_RUN=28)
LAYOUT = ("tab", "k1", "k2", "counters", "ring", "phase", "mag", "hist", "pool", "free_list", "ready", "ctl", "events")
CTL = ("free_top", "n_ready", "pool_overflows", "out_overflows", "out_used", "out_records", "n_events", "pad")
DEC_DATA = 1


def build(tmpdir):
    so = os.path.join(str(tmpdir), "libk2state.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I", CSRC, "-I", INCLUDE, "-o", so, os.path.join(HERE, "hostsim", "k2_state.cpp")])
    L = C.CDLL(so)
    L.k2_state_open.restype = C.c_void_p
    L.k2_state_open.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_float, C.c_uint32, C.c_int,
                                C.c_int]
    L.k2_state_step.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.k2_state_read.argtypes = [C.c_void_p] + [C.c_void_p] * 4
    L.k2_state_ready.restype = C.c_uint32
    L.k2_state_ready.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.k2_state_slot.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    L.k2_state_phase_rows.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    L.k2_state_close.argtypes = [C.c_void_p]
    L.k2_state_sizes.argtypes = [C.c_void_p]
    L.k2_state_stage_layout.restype = C.c_uint32
    L.k2_state_stage_layout.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    sz = np.zeros(4, np.uint32)
    L.k2_state_sizes(sz.ctypes.data)
    L.slot_words, L.slot_header_words, L.n_fields, L.ctl_bytes = int(sz[0]) // 4, int(sz[1]) // 4, int(sz[2]), int(sz[3])
    assert L.n_fields == len(K2) and L.ctl_bytes == 4 * len(CTL)
    return L


def stage_layout(L, n_ch, max_dec, flags):
    """({part: byte offset}, total bytes, pool slots) of a stage's device memory"""
    off = np.zeros(14, np.uint64)
    n_slots = L.k2_state_stage_layout(n_ch, max_dec, flags, off.ctypes.data)
    return dict(zip(LAYOUT, (int(x) for x in off[:13]))), int(off[13]), int(n_slots)


def slot_words_used(nbits, complete):
    """words of a slot that hold the burst: all ceil(nbits / 32) of a completed burst; the full words of an open one (its
    partial last word is written when the burst completes, and its header too)"""
    return (int(nbits) + 31) // 32 if complete else int(nbits) // 32


class HostStage:
    """one host walk of a stage: open, step a launch, read"""

    def __init__(self, L, dec, freqs, max_ppm, n_slots, form=PER_SAMPLE, trace=True):
        self.L = L
        self.dec = np.ascontiguousarray(dec, np.float32)
        self.n_dec, self.n_ch = self.dec.shape[:2]
        f = np.ascontiguousarray(freqs, np.uint32)
        self.h = L.k2_state_open(self.dec.ctypes.data, self.n_dec, self.n_ch, f.ctypes.data, kc.DEC_RATE * 20, max_ppm,
                                 n_slots, form, int(trace))
        assert self.h
        self.n_slots = n_slots

    def step(self, n=0, counts=None):
        c = None if counts is None else np.ascontiguousarray(counts, np.uint32)
        assert self.L.k2_state_step(self.h, None if c is None else c.ctypes.data, n) == 0

    def read(self):
        """dict(k2=[K2_NFIELDS][n_ch] u32, ring=[160][n_ch] f32, hist=[160][n_ch] f32, ctl={name: value})"""
        k2 = np.zeros((self.L.n_fields, self.n_ch), np.uint32)
        ring = np.zeros((kc.RING, self.n_ch), np.float32)
        hist = np.zeros((kc.RING, self.n_ch), np.float32)
        ctl = np.zeros(len(CTL), np.uint32)
        self.L.k2_state_read(self.h, k2.ctypes.data, ring.ctypes.data, hist.ctypes.data, ctl.ctypes.data)
        return dict(k2=k2, ring=ring, hist=hist, ctl=dict(zip(CTL, (int(x) for x in ctl))))

    def ready(self):
        """[u32 slot] of the ready list (in slot order)"""
        buf = np.zeros((self.n_slots, self.L.slot_words), np.uint32)
        n = self.L.k2_state_ready(self.h, buf.ctypes.data, self.n_slots)
        return list(buf[:n])

    def slot(self, i):
        buf = np.zeros(self.L.slot_words, np.uint32)
        assert self.L.k2_state_slot(self.h, int(i), buf.ctypes.data) == 0
        return buf

    def phase_rows(self, row0, n_rows):
        """rows [row0, row0 + n_rows) of the stream's phases with 160 zero rows in front"""
        out = np.zeros((n_rows, self.n_ch), np.float32)
        self.L.k2_state_phase_rows(self.h, row0, n_rows, out.ctypes.data)
        return out

    def open_words(self, k2):
        """{channel: words written so far} of every channel inside a burst with a slot"""
        H = self.L.slot_header_words
        out = {}
        for ch in np.flatnonzero(k2[K2["SLOT"]].view(np.int32) >= 0):
            out[int(ch)] = self.slot(k2[K2["SLOT"], ch])[H:H + slot_words_used(k2[K2["NBITS"], ch], False)]
        return out

    def close(self):
        if self.h:
            self.L.k2_state_close(self.h)
            self.h = None


def ready_key(L, s):
    """a ready burst as comparable bytes: header and the words that hold it"""
    H = L.slot_header_words
    return s[:H].tobytes() + s[H:H + slot_words_used(s[4], True)].tobytes()


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return build(tmp_path_factory.mktemp("k2state"))


def _first_difference(a, b):
    """None, or what differs between two reads"""
    if not np.array_equal(a["k2"], b["k2"]):
        f, ch = np.argwhere(a["k2"] != b["k2"])[0]
        name = [k for k, v in K2.items() if v == f][0]
        return f"K2_{name} of channel {ch}: {a['k2'][f, ch]:#x} != {b['k2'][f, ch]:#x}"
    for part in ("ring", "hist"):
        if a[part].tobytes() != b[part].tobytes():
            return f"{part} of channel {np.argwhere(a[part].view(np.uint32) != b[part].view(np.uint32))[0][1]}"
    if a["ctl"] != b["ctl"]:
        return f"ctl {a['ctl']} != {b['ctl']}"
    return None


def _case(name):
    stage, n_ch, launches, n_slots = kd.CASES[name]
    s = kc.stage(stage)
    dec, freqs = s["dec"], s["freqs"]
    if n_ch is not None:
        dec, freqs = dec[:, :n_ch], freqs[:n_ch]
    return dec, freqs, s["max_ppm"], launches, n_slots if n_slots is not None else 3 * dec.shape[1] + 16


@pytest.mark.parametrize("case", list(kd.CASES))
def test_every_walk_form_leaves_the_per_sample_state_after_every_launch(lib, case):
    dec, freqs, max_ppm, launches, n_slots = _case(case)
    ref = HostStage(lib, dec, freqs, max_ppm, n_slots, PER_SAMPLE)
    forms = {k: HostStage(lib, dec, freqs, max_ppm, n_slots, v) for k, v in FORMS.items()}
    in_data = 0
    try:
        for li, (a, n) in enumerate(kc.launch_bounds(dec.shape[0], launches)):
            ref.step(n)
            want = ref.read()
            want_ready = sorted(ready_key(lib, s) for s in ref.ready())
            want_open = ref.open_words(want["k2"])
            in_data += len(want_open)
            for k, H in forms.items():
                H.step(n)
                got = H.read()
                diff = _first_difference(got, want)
                assert diff is None, f"{case} {k}: launch {li} (samples {a}..{a + n}): {diff}"
                assert sorted(ready_key(lib, s) for s in H.ready()) == want_ready, f"{case} {k}: launch {li}: ready bursts"
                got_open = H.open_words(got["k2"])
                assert got_open.keys() == want_open.keys() and all(np.array_equal(got_open[c], w) for c, w in want_open.items()), \
                    f"{case} {k}: launch {li}: words of an open burst"
    finally:
        for H in [ref] + list(forms.values()):
            H.close()
    assert in_data > 0, f"{case}: no launch ended inside a burst"


@pytest.mark.parametrize("n_ch", [1, 31, 32, 33, 85, 86, 127, 1280, 1281, 4096])
@pytest.mark.parametrize("max_dec", [1, 12, 160, 2399, 8000])
def test_restated_stage_layout_matches_the_library(lib, n_ch, max_dec):
    """the layout the device tests read a stage through is the one vdl2gpu_stage_create lays out"""
    import dumpvdl2_b200 as vd
    V = vd.load_library()
    for flags in (0, vd.FLAG_TRACE, vd.FLAG_KEEP_DEC, vd.FLAG_TRACE | vd.FLAG_INPUT_LEVELS | vd.FLAG_CHANNEL_LEVELS):
        off, total, n_slots = stage_layout(lib, n_ch, max_dec, flags)
        assert total == V.vdl2gpu_stage_device_bytes(n_ch, max_dec, flags), (n_ch, max_dec, flags)
        assert n_slots == max(256, 3 * n_ch)
        assert all(v % 256 == 0 for v in off.values()) and list(off.values()) == sorted(off.values())
