"""CPU: input levels (VDL2GPU_FLAG_INPUT_LEVELS) without a GPU - the per-component code, rail and magnitude rules and the
128-bit fold of the sum of squares of vdl2_core.cuh compiled for the host (tests/hostsim/input_levels.cpp, TEST-ONLY),
the ctypes mirror against the C layout of vdl2gpu_input_levels, the refusals that need no device, and the Python
helper that turns one record into dBFS and full-scale units."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import api

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "dumpvdl2_b200", "csrc")
EINVAL = -1
U64 = (1 << 64) - 1


def levels_of(buf, fmt):
    """numpy restatement of one input's record over the raw bytes buf (interleaved I, Q) in format fmt (vd.FMT_U8 or
    vd.FMT_S16); a trailing partial sample is not a sample"""
    b = np.ascontiguousarray(buf).view(np.uint8).reshape(-1)
    if fmt == vd.FMT_U8:
        v = b[:b.size // 2 * 2].astype(np.int64).reshape(-1, 2)
        c, rail, fs = 2 * v - 255, (v == 0) | (v == 255), 255
    else:
        v = b[:b.size // 4 * 4].view("<i2").astype(np.int64).reshape(-1, 2)
        c, rail, fs = v, (v == -32768) | (v == 32767), 32768
    return dict(samples=int(c.shape[0]), sum_i=int(c[:, 0].sum()), sum_q=int(c[:, 1].sum()), pow=int((c * c).sum()),
                clipped=int(rail.any(axis=1).sum()), peak=int(np.abs(c).max()) if c.size else 0, full_scale=fs)


def add_levels(a, b):
    """the record of two pieces of one stream"""
    out = {k: a[k] + b[k] for k in ("samples", "sum_i", "sum_q", "pow", "clipped")}
    out.update(peak=max(a["peak"], b["peak"]), full_scale=a["full_scale"])
    return out


@pytest.fixture(scope="module")
def lv(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("input_levels") / "liblevels.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I", CSRC, "-o", so, os.path.join(HERE, "hostsim", "input_levels.cpp")])
    L = C.CDLL(so)
    L.lv_code.restype = C.c_int32
    L.lv_code.argtypes = [C.c_uint32, C.c_int32]
    for f in (L.lv_rail, L.lv_full_scale):
        f.restype = C.c_uint32
        f.argtypes = [C.c_uint32, C.c_int32]
    L.lv_full_scale.argtypes = [C.c_uint32]
    L.lv_mag.restype = C.c_uint32
    L.lv_mag.argtypes = [C.c_int32]
    L.lv_pow.restype = C.c_uint32
    L.lv_pow.argtypes = [C.c_int32, C.c_int32]
    L.lv_carry.restype = C.c_uint32
    L.lv_carry.argtypes = [C.c_uint64, C.c_uint64]
    L.lv_fold.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.lv_layout.argtypes = [C.c_void_p]
    L.lv_flag.restype = C.c_uint32
    return L


def _fold(lv, addends, lo=0, hi=0):
    a = np.ascontiguousarray(addends, np.uint64)
    l, h = C.c_uint64(lo), C.c_uint64(hi)
    lv.lv_fold(a.ctypes.data, a.size, C.byref(l), C.byref(h))
    return (h.value << 64) | l.value


def test_cu8_codes_rails_and_magnitudes_over_all_256_values(lv):
    v = np.arange(256)
    code = 2 * v - 255
    assert [lv.lv_code(0, int(x)) for x in v] == code.tolist()
    # c / 255 is exactly the reference's level table entry (v - 127.5) / 127.5 (src/demod.c:349-354)
    assert np.array_equal(code / 255.0, (v - 127.5) / 127.5)
    assert [lv.lv_rail(0, int(x)) for x in v] == ((v == 0) | (v == 255)).astype(int).tolist()
    assert [lv.lv_mag(int(c)) for c in code] == np.abs(code).tolist()
    assert lv.lv_full_scale(0) == 255
    assert max(lv.lv_mag(int(c)) for c in code) == 255


@pytest.mark.parametrize("fmt", [1, 2], ids=["interleaved", "planar"])
def test_cs16_codes_rails_and_magnitudes_at_the_extremes(lv, fmt):
    v = np.array([-32768, -32767, -1, 0, 1, 12345, 32766, 32767])
    assert [lv.lv_code(fmt, int(x)) for x in v] == v.tolist()
    assert [lv.lv_rail(fmt, int(x)) for x in v] == ((v == -32768) | (v == 32767)).astype(int).tolist()
    assert [lv.lv_mag(int(x)) for x in v] == np.abs(v).tolist()
    assert lv.lv_mag(-32768) == 32768 and lv.lv_full_scale(fmt) == 32768


def test_sample_squares(lv):
    assert lv.lv_pow(-32768, -32768) == 1 << 31                      # the largest: fits 32 bits unsigned
    assert lv.lv_pow(32767, -32768) == 32767 ** 2 + 32768 ** 2
    assert lv.lv_pow(-255, 255) == 2 * 255 ** 2 and lv.lv_pow(0, 0) == 0
    rng = np.random.default_rng(3)
    for ci, cq in rng.integers(-32768, 32768, (200, 2)):
        assert lv.lv_pow(int(ci), int(cq)) == int(ci) ** 2 + int(cq) ** 2


def test_fold_carries_across_2_64(lv):
    assert lv.lv_carry(U64, 1) == 1 and lv.lv_carry(U64 - 1, 1) == 0 and lv.lv_carry(0, U64) == 0 and lv.lv_carry(1, U64) == 1
    assert _fold(lv, [1], lo=U64) == 1 << 64
    assert _fold(lv, [U64, U64, U64]) == 3 * U64
    assert _fold(lv, [5], lo=U64 - 2, hi=7) == (7 << 64) + U64 - 2 + 5


def test_many_folds_in_any_order_are_exact(lv):
    rng = np.random.default_rng(7)
    # per-block sums (at most 256 samples x 2^31) and whole chunks up to the largest one (2^30 cs16 samples x 2^31 = 2^61)
    a = np.concatenate([rng.integers(0, 1 << 39, 20000, dtype=np.uint64), rng.integers(0, 1 << 61, 3000, dtype=np.uint64)])
    want = sum(int(x) for x in a)
    assert want > 1 << 66
    assert _fold(lv, a) == want
    for seed in range(3):                                              # the order blocks run in does not matter
        assert _fold(lv, np.random.default_rng(seed).permutation(a)) == want


def test_the_largest_single_chunk_sum(lv):
    big = (1 << 30) * (1 << 31)                                        # 2^30 complex samples at -32768 / -32768 (4 GiB)
    assert big < 1 << 64
    n = 1 << 10
    assert _fold(lv, [big] * n) == big * n == 1 << 71
    assert _fold(lv, [big], lo=U64 - big + 1) == U64 + 1               # lands exactly on 2^64


def test_ctypes_mirror_matches_the_c_layout(lv):
    out = np.zeros(18, np.uint64)
    lv.lv_layout(out.ctypes.data)
    names = ["samples", "sum_i", "sum_q", "pow_lo", "pow_hi", "clipped", "peak", "full_scale"]
    mirror = [C.sizeof(api._InputLevels)] + [getattr(api._InputLevels, n).offset for n in names]
    assert mirror == out[:9].tolist() == out[9:].tolist()
    assert mirror[0] == 56 and mirror[-1] == 52
    assert lv.lv_flag() == vd.FLAG_INPUT_LEVELS == 1 << 6


def test_refusals_without_a_context():
    L = vd.load_library()
    out = (api._InputLevels * 2)()
    assert L.vdl2gpu_get_input_levels(None, out, 1) == EINVAL
    assert "no context" in L.vdl2gpu_last_error().decode()
    assert L.vdl2gpu_get_input_levels(None, None, 0) == EINVAL


@pytest.mark.parametrize("fmt", [vd.FMT_U8, vd.FMT_S16], ids=["cu8", "cs16"])
def test_level_metrics_against_numpy_float64(fmt):
    rng = np.random.default_rng(11 + fmt)
    n = 100003
    if fmt == vd.FMT_U8:
        raw = np.clip(np.round(127.5 + 40 * rng.standard_normal(2 * n) + 3), 0, 255).astype(np.uint8)
        x = (raw.astype(np.float64) - 127.5) / 127.5                  # src/demod.c:349-354
        rails = (raw == 0) | (raw == 255)
    else:
        raw = np.clip(np.round(9000 * rng.standard_normal(2 * n) - 50), -32768, 32767).astype("<i2")
        x = raw.astype(np.float64) / 32768.0                           # src/demod.c:361-363
        rails = (raw == -32768) | (raw == 32767)
    rec = levels_of(raw.view(np.uint8), fmt)
    m = vd.level_metrics(rec)
    i, q = x[0::2], x[1::2]
    assert rec["clipped"] > 0
    assert m["power_dbfs"] == pytest.approx(10 * np.log10(np.mean(i * i + q * q)), rel=1e-12)
    assert m["dc_i"] == pytest.approx(np.mean(i), rel=1e-9, abs=1e-15)
    assert m["dc_q"] == pytest.approx(np.mean(q), rel=1e-9, abs=1e-15)
    assert m["clipped_fraction"] == np.mean(rails[0::2] | rails[1::2])
    assert m["peak"] == np.max(np.abs(x))


def test_level_metrics_of_empty_and_silent_inputs():
    assert vd.level_metrics(dict(samples=0, sum_i=0, sum_q=0, pow=0, clipped=0, peak=0, full_scale=255))["power_dbfs"] is None
    z = vd.level_metrics(levels_of(np.zeros(64, np.uint8), vd.FMT_S16))
    assert z["power_dbfs"] == float("-inf") and z["dc_i"] == 0 and z["peak"] == 0 and z["clipped_fraction"] == 0
    rail = vd.level_metrics(levels_of(np.full(64, 0x80, np.uint8) * np.tile([0, 1], 32).astype(np.uint8), vd.FMT_S16))
    assert rail["peak"] == 1.0 and rail["clipped_fraction"] == 1.0    # every component at -32768
