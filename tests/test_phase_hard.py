"""CPU: the phase and magnitude evaluations on the inputs where they can go wrong.

tests/golden/phase_hard.json (made by tests/golden/make_phase_hard.py) holds samples whose exact atan2 lies within 4
double ulps of a float rounding boundary, samples either side of the fast path's guard, and samples whose magnitude is
an exact float midpoint or just off one.  Here:
- every entry is re-verified with mpmath at 200 bits (the phase: atan2 correctly rounded to double and narrowed, the
  float nearest to atan2, the distance from the midpoint) and with integer arithmetic (the magnitude);
- glibc's (float)atan2, which the oracle and the host simulations use, is compared with the phase;
- the host build of vdl2_fastmath.cuh (tests/hostsim/phase_hard.cpp, seeds perturbed by +-2^-18 as in
  tools/check_fastmath.cpp) must, on every entry and in each of vdl2_phase_fast, vdl2_phase_fast_nb, vdl2_mag_fast and
  vdl2_mag_fast_nb, either set *slow or return the expected float; vdl2_atan2_cr, the device's fall-back, must return
  the phase on every entry;
- two deliberately broken builds must fail on the fixture: a guard of 1 unit instead of 512, and a fall-back that keeps
  the fast float.  That is what shows the fixture reaches the boundary cases."""
import json
import math
import os
import subprocess
import sys
import ctypes as C

import mpmath as mp
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "dumpvdl2_b200", "csrc")
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_phase_hard as mk  # noqa: E402

FIXTURE = os.path.join(HERE, "golden", "phase_hard.json")
HARD = ("random", "near_pi", "near_pio2", "break", "pow2")         # classes searched within 4 double ulps of a midpoint
SEED_ERRS = (-2.0 ** -18, 0.0, 2.0 ** -18)
GLIBC_MISROUNDED = 2                                               # entries where glibc's double atan2 is not correctly rounded


def load():
    with open(FIXTURE) as f:
        return json.load(f)["cases"]


CASES = load()


def arrays(cases):
    u = lambda k: np.array([int(c[k], 16) for c in cases], np.uint32)      # noqa: E731
    return dict(re=u("re").view(np.float32), im=u("im").view(np.float32), phase=u("phase"), glibc=u("glibc"), mag=u("mag"))


def same(a, b):
    """bitwise equality of uint32 bit patterns, any NaN equal to any NaN"""
    fa, fb = a.view(np.float32), b.view(np.float32)
    return (a == b) | (np.isnan(fa) & np.isnan(fb))


def build(tmp, header_dir=CSRC, defines=()):
    so = os.path.join(str(tmp), "libphasehard.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           *[f"-D{d}" for d in defines], "-I", header_dir, "-o", so,
                           os.path.join(HERE, "hostsim", "phase_hard.cpp")])
    L = C.CDLL(so)
    L.phase_hard_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_void_p]
    return L


def evaluate(L, x, seed_err):
    n = x["re"].size
    val = np.zeros((n, 7), np.float32)
    slow = np.zeros((n, 4), np.int32)
    re, im = np.ascontiguousarray(x["re"]), np.ascontiguousarray(x["im"])
    L.phase_hard_eval(re.ctypes.data, im.ctypes.data, n, seed_err, val.ctypes.data, slow.ctypes.data)
    return val.view(np.uint32), slow


def contract_failures(val, slow, x):
    """{routine: indices where it neither set *slow nor returned the expected float}"""
    out = {}
    for j, name, want in ((0, "vdl2_phase_fast", x["phase"]), (1, "vdl2_phase_fast_nb", x["phase"]),
                          (2, "vdl2_mag_fast", x["mag"]), (3, "vdl2_mag_fast_nb", x["mag"])):
        out[name] = np.flatnonzero((slow[:, j] == 0) & ~same(val[:, j], want))
    return out


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return build(tmp_path_factory.mktemp("phasehard"))


def test_fixture_covers_every_class():
    hard = [c for c in CASES if c["cls"] in HARD]
    assert all(abs(c["dist"]) < 4 for c in hard)
    assert len(hard) >= 1000 and sum(abs(c["dist"]) < 1 for c in hard) >= 250, len(hard)
    per_octant = np.bincount([c["octant"] for c in hard], minlength=8)
    assert (per_octant >= 50).all(), per_octant
    n = {k: sum(c["cls"] == k for c in CASES) for k in {c["cls"] for c in CASES}}
    for k in HARD[1:] + ("mag_tie", "mag_near_tie", "special"):
        assert n.get(k, 0) >= 10, (k, n)
    assert n["zero"] == 4
    for c in CASES:
        re, im = float(mk.from_bits(c["re"])), float(mk.from_bits(c["im"]))
        if c["cls"] == "near_pi":
            assert re < 0 and abs(im) < 1e-6 * abs(re)
        if c["cls"] == "near_pio2":
            assert abs(re) < 1e-6 * abs(im)
        if c["cls"] == "break":
            q = min(abs(re), abs(im)) / max(abs(re), abs(im))
            assert min(abs(q - (k + 0.5) / 8) for k in range(8)) <= 2.0 ** -20
        if c["cls"] == "pow2":
            v = abs(float(mk.from_bits(c["phase"])))
            assert abs(v / 2.0 ** round(math.log2(v)) - 1) <= 2.0 ** -9
    guard = [abs(c["dist"]) for c in CASES if c["cls"] == "guard"]
    assert sum(400 <= d < 512 for d in guard) >= 10 and sum(512 <= d < 700 for d in guard) >= 10
    # results on either side of a power of two (where the float spacing changes)
    pw = [float(mk.from_bits(c["phase"])) for c in CASES if c["cls"] == "pow2"]
    assert any(abs(v) < 2.0 ** round(math.log2(abs(v))) for v in pw) and any(abs(v) > 2.0 ** round(math.log2(abs(v))) for v in pw)


def test_fixture_entries_are_exact():
    """the correctly rounded phase and its distance at 200 bits, the magnitude with integers, the octant"""
    for c in CASES:
        re, im = mk.from_bits(c["re"]), mk.from_bits(c["im"])
        again = mk.case(re, im, c["cls"])
        for k in ("phase", "nearest", "mag", "octant"):
            assert again[k] == c[k], (c, again)
        if c["dist"] is not None and abs(c["dist"]) < 1e3:
            assert again["dist"] == pytest.approx(c["dist"], abs=1e-3), (c, again)
    # a tie of the magnitude goes to the even float, a near-tie to the nearer one
    ties = [c for c in CASES if c["cls"] == "mag_tie"]
    assert all(int(c["mag"], 16) % 2 == 0 for c in ties)
    with mp.workprec(200):
        for c in ties:
            re, im = float(mk.from_bits(c["re"])), float(mk.from_bits(c["im"]))
            m = mp.sqrt(mp.mpf(re) ** 2 + mp.mpf(im) ** 2)
            f = float(mk.from_bits(c["mag"]))
            g = float(np.nextafter(np.float32(f), np.float32(m > f and np.inf or -np.inf)))
            assert (mp.mpf(f) + mp.mpf(g)) / 2 == m, c


def test_glibc_and_double_rounding():
    """glibc's (float)atan2 as recorded; where it differs from `phase` it misrounds the double (DESIGN.md §8a).  `phase`
    differs from the float nearest to atan2 exactly where atan2 lies within half a double ulp of a float midpoint."""
    x = arrays(CASES)
    got = np.array([mk.glibc_atan2(a, b) for a, b in zip(x["re"], x["im"])], np.float32).view(np.uint32)
    assert same(got, x["glibc"]).all()
    differ = [c for c in CASES if c["glibc"] != c["phase"]]
    assert len(differ) == GLIBC_MISROUNDED, differ
    assert all(c["cls"] in HARD and abs(c["dist"]) < 4 for c in differ)
    dr = [c for c in CASES if c["nearest"] != c["phase"]]
    assert len(dr) > 0 and all(abs(c["dist"]) < 0.5 for c in dr)
    for c in dr:                                       # the double is the midpoint; the narrowing took the even float
        assert int(c["phase"], 16) % 2 == 0


@pytest.mark.parametrize("seed_err", SEED_ERRS, ids=["seed-", "seed0", "seed+"])
def test_host_fast_paths_are_slow_or_correctly_rounded(lib, seed_err):
    x = arrays(CASES)
    val, slow = evaluate(lib, x, seed_err)
    for name, bad in contract_failures(val, slow, x).items():
        assert bad.size == 0, f"{name}: {bad.size} entries neither slow nor correctly rounded, first {[CASES[i] for i in bad[:3]]}"
    bad = np.flatnonzero(~same(val[:, 4], x["phase"]))
    assert bad.size == 0, f"vdl2_atan2_cr misrounds {bad.size} entries, first {[CASES[i] for i in bad[:3]]}"
    for j in (5, 6):                                   # what a kernel delivers: fast value or fall-back
        bad = np.flatnonzero(~same(val[:, j], x["phase"]))
        assert bad.size == 0, [CASES[i] for i in bad[:3]]
    # every hard entry next to a midpoint (within 1 unit) must have left the fast path
    near = np.array([c["cls"] in HARD and abs(c["dist"]) < 1 for c in CASES])
    inrange = np.array([c["cls"] in ("random", "break", "pow2") for c in CASES])
    assert slow[near & inrange, 0].all() and slow[near & inrange, 1].all()


def _hard_failures(L):
    """entries of the in-range hard classes on which a build delivers a wrong phase, over the three seeds"""
    x = arrays(CASES)
    inrange = np.array([c["cls"] in ("random", "break", "pow2") for c in CASES])
    n = 0
    for e in SEED_ERRS:
        val, slow = evaluate(L, x, e)
        wrong = ~same(val[:, 5], x["phase"]) | ~same(val[:, 6], x["phase"])
        n += int((wrong & inrange).sum())
    return n


def test_fixture_catches_a_narrow_guard(tmp_path):
    """the guard dist < 512u cut to dist < 1u (in a copy of the header): the fast paths return misrounded floats"""
    with open(os.path.join(CSRC, "vdl2_fastmath.cuh")) as f:
        src = f.read()
    assert src.count("dist < 512u") == 4
    (tmp_path / "vdl2_fastmath.cuh").write_text(src.replace("dist < 512u", "dist < 1u"))
    L = build(tmp_path, header_dir=str(tmp_path))
    assert _hard_failures(L) > 0
    x = arrays(CASES)
    val, slow = evaluate(L, x, 0.0)
    assert sum(b.size for b in contract_failures(val, slow, x).values()) > 0


def test_fixture_catches_a_fallback_that_keeps_the_fast_double(tmp_path):
    """the fall-back replaced by the fast path's own (float) of its double: misrounded floats on the hard entries"""
    L = build(tmp_path, defines=("PHASE_HARD_FALLBACK_FAST",))
    assert _hard_failures(L) > 0
