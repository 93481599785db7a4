"""CPU: channel levels (VDL2GPU_FLAG_CHANNEL_LEVELS) without a GPU - the power, bin and quantiser rules and the 128-bit fold
of vdl2_core.cuh compiled for the host (tests/hostsim/channel_levels.cpp, TEST-ONLY), the bound that keeps q within 64 bits
derived from the library's own filter taps, the ctypes mirror against the C layout of vdl2gpu_channel_levels, the refusals
that need no device, the Python metrics, and the oracle's noise floor (tests/nf_oracle.py) against what its bursts carry."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
import scipy.signal
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import api, synth
from oracle import pyoracle as po
from tests.nf_oracle import Oracle

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "dumpvdl2_b200", "csrc")
EINVAL = -1
U64 = (1 << 64) - 1
NBINS = 40


def sample_pow(dec):
    """p = fl32(fl32(re re) + fl32(im im)) of decimated samples [..., 2] (float32 throughout: no FMA)"""
    d = np.asarray(dec, np.float32)
    return d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]


def bins_of(p):
    """b = min(max(E - 90, 0), 39), E the biased exponent of p"""
    e = (np.asarray(p, np.float32).view(np.uint32) >> 23).astype(np.int64) & 0xFF
    return np.clip(e - 90, 0, NBINS - 1)


def q_of(p):
    """(uint64)(p 2^48), truncated (the scaling is exact in float32, the conversion exact in float64)"""
    return np.floor(np.asarray(p, np.float32).astype(np.float64) * 2.0 ** 48).astype(np.uint64)


def levels_of_dec(dec, counts=None):
    """numpy restatement of every channel's hist / pow / peak_pow over decimated samples [n][n_ch][2]; counts: per channel,
    how many of the rows are that channel's (ragged spans), default all of them.  -> list of dicts"""
    d = np.asarray(dec, np.float32)
    n, n_ch = d.shape[0], d.shape[1]
    p = sample_pow(d)
    live = np.ones((n, n_ch), bool) if counts is None else np.arange(n)[:, None] < np.asarray(counts, np.int64)[None, :]
    p = np.where(live, p, np.float32(0))
    b = np.where(live, bins_of(p), NBINS) + (NBINS + 1) * np.arange(n_ch)[None, :]
    hist = np.bincount(b.ravel(), minlength=(NBINS + 1) * n_ch).reshape(n_ch, NBINS + 1)[:, :NBINS].astype(np.uint64)
    q = q_of(p)
    lo = (q & np.uint64(0xFFFFFFFF)).sum(axis=0, dtype=np.uint64)       # exact: n < 2^32 addends below 2^32 each
    hi = (q >> np.uint64(32)).sum(axis=0, dtype=np.uint64)
    peak = p.max(axis=0) if n else np.zeros(n_ch, np.float32)
    return [dict(hist=hist[k], pow=(int(hi[k]) << 32) + int(lo[k]), peak_pow=np.float32(peak[k])) for k in range(n_ch)]


def add_levels(a, b):
    """the figures of two pieces of one channel's stream"""
    return dict(hist=a["hist"] + b["hist"], pow=a["pow"] + b["pow"], peak_pow=max(a["peak_pow"], b["peak_pow"]))


def zero_levels(n_ch):
    return [dict(hist=np.zeros(NBINS, np.uint64), pow=0, peak_pow=np.float32(0)) for _ in range(n_ch)]


@pytest.fixture(scope="module")
def cl(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("channel_levels") / "libchlevels.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I", CSRC, "-o", so, os.path.join(HERE, "hostsim", "channel_levels.cpp")])
    L = C.CDLL(so)
    L.cl_pow.restype = C.c_float
    L.cl_pow.argtypes = [C.c_float, C.c_float]
    L.cl_bin.restype = C.c_uint32
    L.cl_bin.argtypes = [C.c_float]
    L.cl_q.restype = C.c_uint64
    L.cl_q.argtypes = [C.c_float]
    L.cl_fold.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.cl_lpf.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p]
    L.cl_layout.argtypes = [C.c_void_p]
    L.cl_flag.restype = C.c_uint32
    L.cl_bins.restype = C.c_uint32
    return L


def _f32(bits):
    return np.array([bits], np.uint32).view(np.float32)[0]


def test_bin_rule_over_every_exponent_zero_and_subnormals(cl):
    assert cl.cl_bins() == NBINS
    for e in range(255):                                  # every finite exponent, at the bottom, middle and top of its octave
        for m in (0, 0x400000, 0x7FFFFF):
            p = _f32((e << 23) | m)
            want = min(max(e - 90, 0), NBINS - 1)
            assert cl.cl_bin(p) == want == bins_of([p])[0], (e, m)
    assert cl.cl_bin(0.0) == 0 and cl.cl_bin(_f32(1)) == 0 and cl.cl_bin(_f32(0x7FFFFF)) == 0     # zero, subnormals
    # both sides of 2^-36 and 2^2, and the bins' edges on the dBFS scale
    lo, hi = np.float32(2.0 ** -36), np.float32(4.0)
    assert cl.cl_bin(np.nextafter(lo, np.float32(0))) == 0 and cl.cl_bin(lo) == 1
    assert cl.cl_bin(np.nextafter(hi, np.float32(0))) == 38 and cl.cl_bin(hi) == 39 and cl.cl_bin(np.float32(3e38)) == 39
    for b in range(1, 39):
        assert cl.cl_bin(np.float32(2.0 ** (b - 37))) == b and cl.cl_bin(np.nextafter(np.float32(2.0 ** (b - 36)), np.float32(0))) == b
    assert 10 * np.log10(2.0 ** -36) == pytest.approx(-108.37, abs=0.01) and 10 * np.log10(4.0) == pytest.approx(6.02, abs=0.01)


def test_sample_power_is_two_rounded_squares_and_a_rounded_sum(cl):
    rng = np.random.default_rng(5)
    d = np.concatenate([rng.standard_normal((3000, 2)), rng.standard_normal((3000, 2)) * 1e-7,
                        rng.uniform(-2, 2, (3000, 2))]).astype(np.float32)
    got = np.array([cl.cl_pow(float(a), float(b)) for a, b in d], np.float32)
    assert np.array_equal(got.view(np.uint32), sample_pow(d).view(np.uint32))
    # not the FMA form fl32(re re + fl32(im im)) nor the double sum: those differ on some of these samples
    exact = (d[:, 0].astype(np.float64) ** 2 + d[:, 1].astype(np.float64) ** 2).astype(np.float32)
    assert not np.array_equal(exact, got)


def test_quantiser_against_python_integers(cl):
    from fractions import Fraction
    rng = np.random.default_rng(9)
    ps = np.concatenate([rng.uniform(0, 4, 2000), 10.0 ** rng.uniform(-20, 4.5, 2000), [0.0, 2.0 ** -48, 2.0 ** -49, 1.0, 32767.998]])
    ps = ps.astype(np.float32)
    ps = np.concatenate([ps, [_f32(1), np.nextafter(np.float32(2.0 ** 15), np.float32(0))]]).astype(np.float32)
    for p in ps:
        want = int(Fraction(float(p)) * (1 << 48))         # floor of the exact product
        assert cl.cl_q(float(p)) == want == int(q_of([p])[0]), p
    assert cl.cl_q(np.nextafter(np.float32(2.0 ** 15), np.float32(0))) < 1 << 63


def _fold(cl, addends, lo=0, hi=0):
    a = np.ascontiguousarray(addends, np.uint64)
    l, h = C.c_uint64(lo), C.c_uint64(hi)
    cl.cl_fold(a.ctypes.data, a.size, C.byref(l), C.byref(h))
    return (h.value << 64) | l.value


def test_fold_across_2_64_in_any_order(cl):
    top = (1 << 63) - 1                                    # the largest q of a sample below 2^15
    assert _fold(cl, [top, top, top]) == 3 * top           # two loud samples already wrap 64 bits
    assert _fold(cl, [1], lo=U64) == 1 << 64
    rng = np.random.default_rng(13)
    # one slice's per-sample q of a loud channel (p ~ 1: q ~ 2^48, 2^16 of them pass 2^64), then slice totals
    a = np.concatenate([rng.integers(0, 1 << 49, 70000, dtype=np.uint64), rng.integers(0, 1 << 63, 3000, dtype=np.uint64)])
    want = sum(int(x) for x in a)
    assert want > 1 << 70
    assert _fold(cl, a) == want
    for seed in range(3):
        assert _fold(cl, np.random.default_rng(seed).permutation(a)) == want


@pytest.mark.parametrize("os_", list(range(1, 41)) + [52, 64, 100, 128, 200, 256])
def test_decimated_power_stays_below_2_15(cl, os_):
    """A decimated component is the input filter's output over mixed samples.  Input components lie within [-1, 1] (cu8
    levels and cs16 / 32768); the NCO's interpolated cos and sin lie within [-1, 1], so a mixed component within [-2, 2].
    The filter's output is then bounded by 2 x the L1 norm of its impulse response, and p by 2 x (2 L1)^2 = 8 L1^2.  The
    bound holds with a margin of over 2^8 for every oversample vdl2gpu_create takes here (the receivers take 10, 13, 20)."""
    A, B = np.zeros(3, np.float32), np.zeros(3, np.float32)
    cl.cl_lpf(105000 * os_, A.ctypes.data, B.ctypes.data)
    # y[n] = a0 x[n] + a1 x[n-1] + a2 x[n-2] + b1 y[n-1] + b2 y[n-2] (src/demod.c:74-79): denominator 1 - b1 z^-1 - b2 z^-2
    den = np.array([1.0, -float(B[1]), -float(B[2])])
    poles = np.roots(den)
    assert np.all(np.abs(poles) < 1)
    n = int(60 / -np.log(np.max(np.abs(poles)))) + 64      # the tail beyond decays below e^-60
    h = scipy.signal.lfilter(A.astype(np.float64), den, np.r_[1.0, np.zeros(n)])
    l1 = float(np.abs(h).sum())
    assert 8 * l1 * l1 < 2.0 ** 15 / 256, (os_, l1)


def test_ctypes_mirror_matches_the_c_layout(cl):
    out = np.zeros(8, np.uint64)
    cl.cl_layout(out.ctypes.data)
    names = ["hist", "pow_lo", "pow_hi", "peak_pow", "mag_lp", "mag_nf", "nf_pwr_dbfs"]
    mirror = [C.sizeof(api._ChannelLevels)] + [getattr(api._ChannelLevels, n).offset for n in names]
    assert mirror == out.tolist()
    assert mirror[0] == 352 and mirror[2] == 320
    assert cl.cl_flag() == vd.FLAG_CHANNEL_LEVELS == 1 << 7


def test_refusals_without_a_context():
    L = vd.load_library()
    out = (api._ChannelLevels * 2)()
    assert L.vdl2gpu_get_channel_levels(None, out, 1) == EINVAL
    assert "no context" in L.vdl2gpu_last_error().decode()
    assert L.vdl2gpu_get_channel_levels(None, None, 0) == EINVAL


def test_channel_level_metrics_against_numpy_float64():
    rng = np.random.default_rng(17)
    d = (rng.standard_normal((50003, 1, 2)) * 0.03).astype(np.float32)
    d[100, 0] = (0.9, -0.4)
    d[200, 0] = (0.0, 0.0)
    rec = levels_of_dec(d)[0]
    rec.update(mag_lp=np.float32(0.05), mag_nf=np.float32(0.031), nf_pwr_dbfs=np.float32(20 * np.log10(np.float32(0.031) + np.float32(0.001))))
    m = vd.channel_level_metrics(rec)
    p = sample_pow(d[:, 0]).astype(np.float64)
    assert m["samples"] == 50003 == int(rec["hist"].sum())
    # pow truncates p 2^48 per sample: at most 2^-48 below the sum, far inside 1e-12 relative
    assert m["power_dbfs"] == pytest.approx(10 * np.log10(p.mean()), rel=1e-12)
    assert m["peak_dbfs"] == 10 * np.log10(np.float64(np.float32(p.max())))
    assert m["nf_dbfs"] == float(rec["nf_pwr_dbfs"])
    edges = m["bin_floor_dbfs"]
    assert len(edges) == NBINS and edges[0] == -np.inf
    assert np.allclose(edges[1:], 10 * np.log10(2.0 ** (np.arange(1, NBINS) - 37.0)), rtol=0, atol=1e-12)
    assert edges[1] == pytest.approx(-108.37, abs=0.01) and edges[-1] == pytest.approx(6.02, abs=0.01)


def test_channel_level_metrics_of_empty_and_silent_channels():
    e = vd.channel_level_metrics(dict(zero_levels(1)[0], mag_lp=0.0, mag_nf=2.0, nf_pwr_dbfs=np.float32(20 * np.log10(2.001))))
    assert e["samples"] == 0 and e["power_dbfs"] is None and e["peak_dbfs"] is None
    z = levels_of_dec(np.zeros((640, 1, 2), np.float32))[0]
    assert z["hist"][0] == 640 and int(z["hist"][1:].sum()) == 0 and z["pow"] == 0
    m = vd.channel_level_metrics(dict(z, mag_lp=0.0, mag_nf=2.0, nf_pwr_dbfs=0.0))
    assert m["samples"] == 640 and m["power_dbfs"] == float("-inf") and m["peak_dbfs"] == float("-inf")


def test_oracle_noise_floor_is_what_its_bursts_carry():
    """the oracle's noise floor read at each burst end equals the mag_nf that burst's trace event and frames carry"""
    fs, os_, centre = 2100000, 20, 136975000
    offs = [-50e3, 25e3, 0.0]
    freqs = [int(centre + o) for o in offs]
    rng = np.random.default_rng(21)
    bursts = [synth.BurstSpec(t, offs[k % 2], synth.random_frames(rng), power_dbfs=-14.0) for k, t in enumerate((0.06, 0.16, 0.27))]
    iq = synth.synth_stream(fs, 0.36, bursts, es_n0_db=26, fmt="u8", seed=4)
    full = Oracle(fs, os_, po.FMT_U8, centre, freqs, trace=True, dec_tap=True)
    full.process(iq)
    dec = full.dec_samples()
    ends = [e for e in full.events() if e["kind"] == 3]
    frames = full.frames()
    assert len(ends) >= 3 and len(frames) >= 3
    o = Oracle(fs, os_, po.FMT_U8, centre, freqs)
    assert np.array_equal(o.noise_floor(), np.array([[0.0, 2.0]] * len(freqs), np.float32))   # src/demod.c:383
    at, seen = 0, []
    for e in sorted(ends, key=lambda e: e["dec_index"]):
        o.process_dec(dec[at:e["dec_index"] + 1])
        at = e["dec_index"] + 1
        nf = o.noise_floor()[e["channel"], 1]
        assert nf == e["f"][1]
        seen.append((e["channel"], float(nf)))
    o.process_dec(dec[at:])
    assert np.array_equal(o.noise_floor(), full.noise_floor())
    assert sorted({(f.channel, float(np.float32(f.mag_nf))) for f in frames}) == sorted(set(seen))
    assert len({v for _, v in seen}) > 1 and all(v != 2.0 for _, v in seen)   # the floor moved between bursts
