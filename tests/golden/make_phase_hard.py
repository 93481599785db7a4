"""Make tests/golden/phase_hard.json: samples whose phase or magnitude lies next to a float rounding boundary.

The demodulator consumes fl32(atan2((double)im, (double)re)) and fl32(sqrt(fl64(re^2 + im^2))) of every decimated sample
(src/demod.c:232,238,256).  An evaluation with an error of an ulp of a double or two delivers those floats except where
the exact value lies within that error of a float midpoint; this fixture collects such samples so that the tests can
feed every evaluation the library has (tests/test_phase_hard.py on the CPU, tests/test_gpu_phase_hard.py on the device)
exactly the inputs where it can go wrong.

atan2 cases: tools/find_hard_phases.c searches float pairs whose atan2l (64-bit mantissa) lies within 4 double ulps of a
float midpoint (classes random, near_pi, near_pio2, break, pow2; see the tool), or 400..700 units of the last double bit
from one (class guard: either side of vdl2_phase_fast's 512-unit guard).  Every candidate is confirmed here with mpmath at
200 bits.  Magnitude cases are made exactly: Pythagorean triples (u^2 - v^2, 2uv, u^2 + v^2) with an odd 25-bit
hypotenuse (an exact float midpoint, which the narrowing sends to the even neighbour), the same with one leg moved a float
ulp either way (just off the midpoint), zeros of both signs and the special values of tools/check_fastmath.cpp.

Each case records the input's float bits, its class and octant, the phase every evaluation must deliver (`phase`): atan2
correctly rounded to double and narrowed to float, the reference's float with a correctly rounded libm; the float nearest
to atan2 (`nearest`), which differs from `phase` where atan2 lies within half a double ulp of a float midpoint (the double
is then the midpoint and narrows to the even float); the signed distance of atan2 from the nearest float midpoint in
units of the last bit of a double there (`dist`); glibc's (float)atan2 (`glibc`); and fl32(sqrt(fl64(re^2 + im^2)))
computed with integers (`mag`).  Floats are 8-digit hex bit patterns.

    python tests/golden/make_phase_hard.py            # search (about 11 minutes on 8 threads) and write the fixture
    python tests/golden/make_phase_hard.py --check    # search again and compare with the committed file byte for byte

The search is deterministic: each block of 2^20 draws has its own generator seeded from (SEED, class, block), so the
candidates do not depend on the number of threads.  Made with SEED and SEARCH below; the search takes about 11 minutes on 8 CPU threads.
"""
import argparse
import json
import math
import os
import random
import subprocess
import sys
import tempfile
from fractions import Fraction

import mpmath as mp
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "phase_hard.json")
SEED = 0x56444C32
SEARCH = [(0, 20000), (1, 2700), (2, 2700), (3, 2700), (4, 2700), (5, 16)]     # (class, blocks of 2^20 draws)
CLASSES = {0: "random", 1: "near_pi", 2: "near_pio2", 3: "break", 4: "pow2", 5: "guard"}
SPECIALS = [0.0, -0.0, 1.0, -1.0, math.inf, -math.inf, math.nan, 1e-38, 1e-45, 3e38]     # tools/check_fastmath.cpp
PREC = 200


def f32(x):
    with np.errstate(over="ignore"):                       # hypot(3e38, 3e38) overflows a float, as it should
        return np.float32(x)


def bits(x):
    return f"{int(np.float32(x).view(np.uint32)):08x}"


def from_bits(h):
    return np.uint32(int(h, 16)).view(np.float32)


def octant(re, im):
    """0..3 in the upper half plane, counter-clockwise from +re (0: re > 0, |im| <= |re|; 1: re > 0, |im| > |re|; 2: re < 0,
    |im| > |re|; 3: re < 0, |im| <= |re|), 4..7 the same below (im's sign bit set)"""
    left = math.copysign(1.0, float(re)) < 0
    steep = abs(float(im)) > abs(float(re))
    o = (2 if steep else 3) if left else (1 if steep else 0)
    return o + (4 if math.copysign(1.0, float(im)) < 0 else 0)


def round_f32(x):
    """the float nearest the mpmath value x (ties cannot occur for atan2 of non-zero rational inputs; to even otherwise)"""
    f = f32(float(x))                                      # within a float ulp of the answer
    cand = [np.nextafter(f, f32(-np.inf)), f, np.nextafter(f, f32(np.inf))]
    best = min(cand, key=lambda c: (abs(mp.mpf(float(c)) - x), int(c.view(np.uint32)) & 1))
    return f32(best)


def midpoint_dist(x, f):
    """signed distance of x from the midpoint between f = round_f32(x) and its neighbour on x's side, in units of the last
    bit of a double at that midpoint"""
    g = np.nextafter(f, f32(np.inf) if x > mp.mpf(float(f)) else f32(-np.inf))
    mid = (mp.mpf(float(f)) + mp.mpf(float(g))) / 2
    e = math.frexp(float(mid))[1] - 1
    return (x - mid) / mp.ldexp(1, e - 52)


def exact_atan2(re, im):
    """(fl32 of the correctly rounded double, the float nearest, dist) of atan2(im, re) for finite inputs, other than
    (+-0, +-0)"""
    sign = -1.0 if math.copysign(1.0, float(im)) < 0 else 1.0     # atan2 takes im's sign, also a zero's (mpmath has no -0)
    with mp.workprec(PREC):
        x = mp.atan2(abs(mp.mpf(float(im))), mp.mpf(float(re))) * sign
        if x == 0:                                         # im == +-0, re > 0: exact
            z = f32(math.copysign(0.0, sign))
            return z, z, None
        f = round_f32(x)
        return f32(float(x)), f, float(mp.nstr(midpoint_dist(x, f), 6, strip_zeros=False))


def special_atan2(re, im):
    """atan2 of a zero or non-finite input, the C99 Annex F value (a multiple of pi/4, a zero or NaN), rounded to double
    and narrowed"""
    v = math.atan2(float(im), float(re)) if not (math.isnan(re) or math.isnan(im)) else math.nan
    if math.isnan(v) or v == 0.0:
        return f32(v)
    with mp.workprec(PREC):
        q = round(v / (math.pi / 4))
        return f32(float(mp.pi * q / 4))


def exact_mag(re, im):
    """fl32(sqrt(fl64(re^2 + im^2))): the sum rounded to double from exact rationals, the square root rounded to double
    with integers, then narrowed once to float"""
    re, im = float(re), float(im)
    if not (math.isfinite(re) and math.isfinite(im)):
        return f32(math.sqrt(re * re + im * im))
    s = float(Fraction(re) ** 2 + Fraction(im) ** 2)       # correctly rounded (int / int true division)
    if s == 0.0:
        return f32(0.0)
    if math.isinf(s):
        return f32(math.inf)
    m, e = math.frexp(s)                                   # s = m 2^e, m in [0.5, 1)
    M, E = int(m * 2 ** 53), e - 53                        # s = M 2^E exactly
    if E % 2:
        M, E = 2 * M, E - 1
    K = 30                                                 # sqrt(M 2^2K) has 57+ bits
    N = M << (2 * K)
    r = math.isqrt(N)
    sticky = r * r != N
    extra = r.bit_length() - 53
    q, rem, half = r >> extra, r & ((1 << extra) - 1), 1 << (extra - 1)
    if rem > half or (rem == half and (sticky or q & 1)):  # to nearest, ties (which cannot occur) to even
        q += 1
    root = math.ldexp(q, extra + E // 2 - K)
    assert root == math.sqrt(s)                            # the IEEE square root agrees
    return f32(root)


def glibc_atan2(re, im):
    return f32(math.atan2(float(im), float(re)))


def case(re, im, cls, want_dist=None):
    re, im = f32(re), f32(im)
    if math.isfinite(re) and math.isfinite(im) and (re != 0 or im != 0):
        ph, near, dist = exact_atan2(re, im)
    else:
        ph, dist = special_atan2(float(re), float(im)), None
        near = ph
    if want_dist is not None:
        assert dist is not None and abs(dist - want_dist) < 1e-2, (bits(re), bits(im), dist, want_dist)
    return dict(re=bits(re), im=bits(im), cls=cls, octant=octant(re, im), phase=bits(ph), nearest=bits(near), dist=dist,
                glibc=bits(glibc_atan2(re, im)), mag=bits(exact_mag(re, im)))


def search(threads, raw=None):
    """-> [(class, re bits, im bits, long double dist)] of tools/find_hard_phases.c, in (class, block, draw) order; with
    raw, read the tool's output for class c from raw/raw_c.txt instead of running it"""
    if raw is not None:
        rows = []
        for cls, _ in SEARCH:
            with open(os.path.join(raw, f"raw_{cls}.txt")) as f:
                for line in f.read().splitlines():
                    c, b, i, r, m, d = line.split()
                    rows.append((int(c), int(b), int(i), r, m, float(d)))
        rows.sort()
        return [(c, r, m, d) for c, _, _, r, m, d in rows]
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "find_hard_phases")
        subprocess.check_call(["cc", "-O2", "-std=c11", "-pthread", os.path.join(ROOT, "tools", "find_hard_phases.c"), "-o", exe, "-lm"])
        rows = []
        for cls, blocks in SEARCH:
            out = subprocess.run([exe, str(SEED), str(cls), str(blocks), str(threads)], check=True, capture_output=True, text=True).stdout
            for line in out.splitlines():
                c, b, i, r, m, d = line.split()
                rows.append((int(c), int(b), int(i), r, m, float(d)))
        rows.sort()
        return [(c, r, m, d) for c, _, _, r, m, d in rows]


def triples(rng, n):
    """n Pythagorean triples (a, b, c) = (u^2 - v^2, 2uv, u^2 + v^2), gcd(u, v) = 1, u - v odd, 2^24 < c < 2^25 (odd, so
    c is the midpoint between the floats c - 1 and c + 1), a < 2^24 (odd, so a float); b is even and below 2^25: a float"""
    out = [(2900, 2897)]
    while len(out) < n:
        v = rng.randrange(2897, 4000)
        u = v + rng.randrange(1, 64, 2)
        if math.gcd(u, v) == 1 and (u, v) not in out:
            out.append((u, v))
    res = []
    for u, v in out:
        a, b, c = u * u - v * v, 2 * u * v, u * u + v * v
        assert 2 ** 24 < c < 2 ** 25 and c % 2 == 1 and a < 2 ** 24 and b < 2 ** 25 and a * a + b * b == c * c
        res.append((a, b, c))
    return res


def magnitude_cases(rng):
    cases = []
    for a, b, c in triples(rng, 40):
        e = rng.randrange(0, 12)                           # |sample| = c 2^-(25 + e) in [2^-13, 1)
        x, y = f32(math.ldexp(a, -25 - e)), f32(math.ldexp(b, -25 - e))
        assert float(x) == math.ldexp(a, -25 - e) and float(y) == math.ldexp(b, -25 - e)
        if rng.random() < 0.5:
            x, y = y, x
        x, y = f32(x * rng.choice([-1, 1])), f32(y * rng.choice([-1, 1]))
        cases.append(case(x, y, "mag_tie"))
        for leg in (0, 1):
            for step in (-1, 1):
                p = [x, y]
                p[leg] = np.nextafter(p[leg], f32(math.copysign(math.inf, step * float(p[leg]))))
                cases.append(case(p[0], p[1], "mag_near_tie"))
    for re in (0.0, -0.0):
        for im in (0.0, -0.0):
            cases.append(case(re, im, "zero"))
    for re in SPECIALS:
        for im in SPECIALS:
            if not (re == 0 and im == 0):
                cases.append(case(re, im, "special"))
    return cases


def make(threads, raw=None):
    cases = []
    for cls, r, m, d in search(threads, raw):
        cases.append(case(from_bits(r), from_bits(m), CLASSES[cls], want_dist=d))
    cases += magnitude_cases(random.Random(SEED))
    head = dict(seed=SEED, search=SEARCH, note="floats as 8-digit hex bit patterns; dist in units of the last bit of a "
                "double at the nearest float midpoint, signed (positive: above); see make_phase_hard.py")
    lines = [json.dumps(c, sort_keys=True) for c in cases]
    return "{\"meta\": " + json.dumps(head, sort_keys=True) + ",\n\"cases\": [\n" + ",\n".join(lines) + "\n]}\n"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true", help="search again and compare with the committed fixture")
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 8)
    ap.add_argument("--raw", help="directory with the search tool's output per class (raw_<class>.txt) instead of a search")
    a = ap.parse_args()
    text = make(a.threads, a.raw)
    if a.check:
        with open(OUT) as f:
            same = f.read() == text
        print("phase_hard.json reproduced byte for byte" if same else "phase_hard.json DIFFERS from a fresh search")
        sys.exit(0 if same else 1)
    with open(OUT, "w") as f:
        f.write(text)
    print(f"wrote {OUT}: {text.count(chr(10)) - 3} cases")


if __name__ == "__main__":
    main()
