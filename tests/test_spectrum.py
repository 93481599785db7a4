"""CPU: spectrum (VDL2GPU_FLAG_SPECTRUM) without a GPU - the segment arithmetic of vdl2_core.cuh compiled for the host
(tests/hostsim/spectrum.cpp, TEST-ONLY) against a numpy float64 windowed FFT, the tables against their definitions, the
bound on p and q, the segment grid against cutting the concatenated stream, the ctypes mirror against the C layout,
the refusals that need no device, and the Python metrics."""
import ctypes as C
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import api
from tests import spectrum_sim as ss

N = ss.N
# Relative to the segment's total power: the float32 FFT's rounding (10 stages, twiddles rounded once) stays far below
REL_TOL = 1e-5


def numpy_power(x):
    """float64 restatement: periodic Hann window, FFT, |X|^2, shifted so that bin 512 is DC"""
    a = ss.as_pairs(x).astype(np.float64)
    w = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N) / N)
    X = np.fft.fft((a[:, 0] + 1j * a[:, 1]) * w)
    return np.fft.fftshift(np.abs(X) ** 2)


def check_against_numpy(x):
    p = ss.segment(x).astype(np.float64)
    ref = numpy_power(x)
    total = max(ref.sum(), 1e-30)
    assert np.max(np.abs(p - ref)) <= REL_TOL * total, np.max(np.abs(p - ref)) / total
    return p


def tone(f_bins, amp=1.0, phase=0.3):
    n = np.arange(N)
    return (amp * np.exp(1j * (2 * np.pi * f_bins * n / N + phase))).astype(np.complex64)


@pytest.mark.parametrize("f", [0.0, 1.0, 37.0, -200.0, 511.0, -512.0, 0.5, 100.25, -300.75, 511.5])
def test_tone_matches_numpy_and_lands_in_its_bin(f):
    p = check_against_numpy(tone(f, 0.9))
    if float(f).is_integer():
        # a tone at offset f (in bins of fs / 1024) lands in stored bin 512 + f (mod 1024: -fs/2 is bin 0)
        assert int(np.argmax(p)) == (512 + int(f)) % N


def test_dc_and_half_rate_tones():
    dc = np.full(N, 0.5 + 0.25j, np.complex64)
    assert int(np.argmax(check_against_numpy(dc))) == 512
    alt = np.where(np.arange(N) % 2 == 0, 0.7, -0.7).astype(np.complex64)           # +-fs/2
    assert int(np.argmax(check_against_numpy(alt))) == 0


def test_white_noise_zeros_and_smallest_codes():
    rng = np.random.default_rng(5)
    for _ in range(4):
        check_against_numpy((rng.normal(0, 0.3, N) + 1j * rng.normal(0, 0.3, N)).astype(np.complex64))
    z = ss.segment(np.zeros((N, 2), np.float32))
    assert not np.any(z)
    # the smallest cs16 codes: +-1 / 32768
    v = rng.choice(np.array([-1, 0, 1], np.int16), 2 * N)
    check_against_numpy(ss.cs16_floats(v))


def test_full_scale_cu8_both_rails():
    rng = np.random.default_rng(9)
    for raw in (np.full(2 * N, 255, np.uint8), np.zeros(2 * N, np.uint8), rng.choice(np.array([0, 255], np.uint8), 2 * N),
                np.tile(np.array([255, 0, 0, 255], np.uint8), N // 2), rng.integers(0, 256, 2 * N).astype(np.uint8)):
        check_against_numpy(ss.cu8_floats(raw))


def test_largest_power_stays_below_2_20_and_q_below_2_60():
    # the largest |X_k| comes from a full-scale complex tone on a bin: sum(w) sqrt(2) = 512 sqrt(2), p = 2^19
    worst = 0.0
    x = ss.as_pairs(tone(0.0, np.sqrt(2.0), phase=np.pi / 4))
    x = np.clip(x, -1.0, 1.0)                                           # both components at full scale: x_n = (1 + 1j)
    worst = max(worst, float(ss.segment(x).max()))
    for raw in (np.full(2 * N, 255, np.uint8), np.zeros(2 * N, np.uint8)):
        worst = max(worst, float(ss.segment(ss.cu8_floats(raw)).max()))
    worst = max(worst, float(ss.segment(ss.cs16_floats(np.full(2 * N, -32768, np.int16))).max()))
    assert 2.0 ** 18 < worst < 2.0 ** 20
    L = ss.lib()
    assert L.sp_q(C.c_float(np.float32(worst))) < (1 << 60)
    assert L.sp_q(C.c_float(np.nextafter(np.float32(2.0 ** 20), np.float32(0)))) < (1 << 60)
    assert L.sp_q(C.c_float(1.0)) == 1 << 40 and L.sp_q(C.c_float(2.0 ** -41)) == 0      # p 2^40, truncated


def test_tables_equal_their_double_then_round_definition():
    win, tw = ss.tables()
    n = np.arange(N)
    assert np.array_equal(win, (0.5 - 0.5 * np.cos(2 * np.pi * n / N)).astype(np.float32))
    k = np.arange(N // 2)
    assert np.array_equal(tw[:, 0], np.cos(2 * np.pi * k / N).astype(np.float32))
    assert np.array_equal(tw[:, 1], (-np.sin(2 * np.pi * k / N)).astype(np.float32))
    assert abs(float(win.astype(np.float64).sum()) - 512.0) < 1e-5         # the window's rounding moves its sum by < 2^-20
    assert [ss.lib().sp_fft_bin(k) for k in (0, 511, 512, 1023)] == [512, 1023, 0, 511]


def cut_reference(x, restarts_at=()):
    """the figures of cutting the concatenated stream (from its last restart on) into whole segments"""
    a = ss.as_pairs(x)
    start = max(restarts_at) if restarts_at else 0
    a = a[start:]
    segs = a.shape[0] // N
    pw = np.zeros(N, dtype=object)
    pk = np.zeros(N, np.uint32)
    L = ss.lib()
    for j in range(segs):
        p = ss.segment(a[j * N:(j + 1) * N])
        pw += np.array([L.sp_q(C.c_float(v)) for v in p], dtype=object)
        pk = np.maximum(pk, p.view(np.uint32))
    return dict(segments=segs, pending=a.shape[0] % N, pow=pw, peak_bits=pk)


def check_same(a, b):
    assert a["segments"] == b["segments"] and a["pending"] == b["pending"]
    assert all(a["pow"][k] == b["pow"][k] for k in range(N))
    assert np.array_equal(a["peak_bits"], b["peak_bits"])


@pytest.mark.parametrize("cuts", [[4096], [1, 1023, 1024, 2048], [0, 1, 0, 1023, 0, 1, 3071],
                                  [1023, 1023, 1023, 1023, 4], [5, 3000, 0, 0, 1100, 12], [777] * 7 + [0]])
def test_grid_equals_cutting_the_concatenated_stream(cuts):
    rng = np.random.default_rng(sum(cuts))
    n = sum(cuts)
    x = (rng.normal(0, 0.2, n) + 1j * rng.normal(0, 0.2, n)).astype(np.complex64)
    check_same(ss.stream(x, cuts), cut_reference(x))
    pend, segs, rest = ss.grid(cuts)
    pos = np.concatenate([[0], np.cumsum(cuts)])
    assert np.array_equal(pend, pos[:-1] % N)
    assert np.array_equal(segs, (pos[1:] // N) - (pos[:-1] // N))
    assert np.array_equal(rest, pos[1:] % N)


def test_pushes_that_split_a_sample_count_whole_samples_only():
    # pushed bytes enter spans in whole decimation groups: a push that ends inside a sample adds nothing until the rest
    # arrives, so the grid sees the group counts of the spans, whatever the push lengths were
    rng = np.random.default_rng(3)
    os_, bpp = 13, 2
    pushes = [7, 1, 26 * 100 + 3, 5, 26 * 77 - 16, 26 * 90 + 13]
    total = sum(pushes)
    groups, queued, cuts = 0, 0, []
    for b in pushes:
        queued += b
        g = queued // (os_ * bpp)
        queued -= g * os_ * bpp
        cuts.append(g * os_)
    n = sum(cuts)
    assert n == total // (os_ * bpp) * os_
    x = (rng.normal(0, 0.2, n) + 1j * rng.normal(0, 0.2, n)).astype(np.complex64)
    check_same(ss.stream(x, cuts), cut_reference(x))


@pytest.mark.parametrize("cuts,restart", [([1500, 700, 3000], 1), ([1023, 1, 2048], 2), ([100, 0, 5000], 1), ([4096, 4096], 1)])
def test_restart_mid_segment_anchors_a_new_grid(cuts, restart):
    rng = np.random.default_rng(11)
    n = sum(cuts)
    x = (rng.normal(0, 0.2, n) + 1j * rng.normal(0, 0.2, n)).astype(np.complex64)
    got = ss.stream(x, cuts, restarts=[restart])
    check_same(got, cut_reference(x, restarts_at=[sum(cuts[:restart])]))
    pend, segs, rest = ss.grid(cuts, restarts=[restart])
    assert pend[restart] == 0


def test_update_receivers_mapping_carries_positions():
    # kept receivers carry their position (and waiting samples) to their new index, new ones start at zero: the grid of a
    # kept receiver is the grid of its whole stream, that of a new one starts with its first span
    rng = np.random.default_rng(13)
    old = {0: [1500, 300], 1: [1023], 2: [4000, 1]}
    after = {0: (2, [2000, 50]), 1: (None, [1200, 1300]), 2: (0, [1, 1023, 1024])}     # new index: (old index, spans)
    for new, (src, spans) in after.items():
        before = old[src] if src is not None else []
        cuts = before + spans
        n = sum(cuts)
        x = (rng.normal(0, 0.2, n) + 1j * rng.normal(0, 0.2, n)).astype(np.complex64)
        check_same(ss.stream(x, cuts), cut_reference(x))
    # removed receiver 1: its figures go with it; nothing to compare


def test_ctypes_mirror_matches_the_c_layout():
    L = ss.lib()
    out = np.zeros(7, np.uint64)
    L.sp_layout(out.ctypes.data)
    s = api._Spectrum
    assert out.tolist() == [C.sizeof(s), s.segments.offset, s.pending.offset, s.pow_lo.offset, s.pow_hi.offset, s.peak.offset, api.SPECTRUM_BINS]
    assert C.sizeof(s) == 20496
    assert L.sp_flag() == vd.FLAG_SPECTRUM == 1 << 8


def test_refusals_without_a_device():
    L = api.load_library()
    rec = (api._Spectrum * 1)()
    assert L.vdl2gpu_get_spectrum(None, 0, 1, rec) == -1
    assert b"no context" in L.vdl2gpu_last_error()


def test_metrics_of_a_full_scale_tone_read_0_dbfs():
    # a complex tone of amplitude a on a bin: p = (512 a)^2 in that bin every segment
    a = 0.5
    segs = 3
    p = np.float32((512 * a) ** 2)
    q = int(ss.lib().sp_q(C.c_float(p)))
    pw = np.zeros(N, dtype=object)
    pw[:] = 0
    pw[600] = q * segs
    peak = np.zeros(N, np.float32)
    peak[600] = p
    m = vd.spectrum_metrics(dict(segments=segs, pending=5, pow=pw, peak=peak), 136_975_000, 1_050_000)
    assert m["freq_hz"][512] == 136_975_000 and m["freq_hz"][600] == 136_975_000 + 88 * 1_050_000 / 1024
    assert abs(m["mean_dbfs"][600] - 20 * np.log10(a)) < 1e-9
    assert abs(m["peak_dbfs"][600] - 20 * np.log10(a)) < 1e-9
    assert m["mean_dbfs"][0] == -np.inf
    none = vd.spectrum_metrics(dict(segments=0, pending=7, pow=np.zeros(N, dtype=object), peak=np.zeros(N, np.float32)), 0, 1_050_000)
    assert none["mean_dbfs"] is None and none["peak_dbfs"] is None
