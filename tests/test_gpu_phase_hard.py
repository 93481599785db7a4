"""-m gpu: the device's phase and magnitude on the inputs where they can go wrong (tests/golden/phase_hard.json).

Every phase the device delivers must be atan2 correctly rounded to double and narrowed to float (the fixture's `phase`),
every magnitude fl32(sqrt(fl64(re^2 + im^2))) (`mag`), bit for bit, whichever evaluation produced it:
(a) vdl2gpu_launch_phase_mag with the fast path and without it, each sample at every position of a 256-thread block and
    as the last element of a launch whose size is not a multiple of 256; signed zeros on their own;
(b) the device functions the phase pass and the K2 walk use (tests/hostsim/phase_hard_device.cu): each fast routine
    sets *slow or returns the expected float, and the fall-backs vdl2_phase_of and vdl2_mag_of return it on every sample
    (the phase pass's tail rows call vdl2_phase_of for every sample);
(c) fixture samples as the decimated rows of 48 channels through vdl2gpu_launch_sync_slice: the phase plane's rows, and
    the K2 fields after every launch against the host walk (test_gpu_k2_state.py), which covers the walk's own
    magnitudes; with the default walk and with VDL2GPU_K2A=0.  Entries where glibc's atan2 is not correctly rounded are
    left out of (c): the host walk uses glibc."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import dumpvdl2_b200 as vd
from dumpvdl2_b200 import build as vb
from tests import k2_corpus as kc
from tests import test_gpu_k2_state as gs
from tests import test_k2_state as ks
from tests import test_phase_hard as ph

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
X = ph.arrays(ph.CASES)
N = X["re"].size
SAMPLES = np.stack([X["re"], X["im"]], 1)                          # [N][2] float32
same = ph.same


def _launch_phase_mag(L, d_x, n, d_ph, d_mg, exact):
    assert L.vdl2gpu_launch_phase_mag(d_x.data_ptr(), n, d_ph.data_ptr(), d_mg.data_ptr(), exact, None) == 0


@pytest.mark.parametrize("exact", [0, 1], ids=["fast", "libm"])
def test_phase_mag_stub_at_every_block_position(exact):
    import torch
    L = vd.load_library()
    rng = np.random.default_rng(0x56444C33)
    for shift in range(256):                           # case j at index shift + j: every residue mod 256 once
        filler = (0.1 * rng.standard_normal((shift, 2))).astype(np.float32)
        x = np.concatenate([filler, SAMPLES])
        n = x.shape[0]
        d_x = torch.from_numpy(x).cuda()
        d_ph = torch.empty(n, dtype=torch.float32, device="cuda")
        d_mg = torch.empty(n, dtype=torch.float32, device="cuda")
        _launch_phase_mag(L, d_x, n, d_ph, d_mg, exact)
        got_ph = d_ph[shift:].cpu().numpy().view(np.uint32)
        got_mg = d_mg[shift:].cpu().numpy().view(np.uint32)
        bad = np.flatnonzero(~same(got_ph, X["phase"]))
        assert bad.size == 0, f"exact={exact} shift={shift}: {bad.size} phases differ, first {[ph.CASES[i] for i in bad[:3]]} " \
                              f"got {[hex(v) for v in got_ph[bad[:3]]]}"
        bad = np.flatnonzero(~same(got_mg, X["mag"]))
        assert bad.size == 0, f"exact={exact} shift={shift}: {bad.size} magnitudes differ, first {[ph.CASES[i] for i in bad[:3]]}"


@pytest.mark.parametrize("exact", [0, 1], ids=["fast", "libm"])
def test_phase_mag_stub_with_each_case_last_in_a_ragged_launch(exact):
    """case j as the last element of a launch of 256 m + r elements, r != 0 (the preceding elements other cases)"""
    import torch
    L = vd.load_library()
    d_a = torch.from_numpy(SAMPLES).cuda()                        # case j at index j
    d_b = torch.from_numpy(np.concatenate([SAMPLES[:1], SAMPLES])).cuda()     # case j at index j + 1
    lengths = [j + 1 if (j + 1) % 256 else j + 2 for j in range(N)]
    off = np.concatenate([[0], np.cumsum(lengths)])
    d_ph = torch.empty(int(off[-1]), dtype=torch.float32, device="cuda")
    d_mg = torch.empty(int(off[-1]), dtype=torch.float32, device="cuda")
    for j, n in enumerate(lengths):
        src = d_a if n == j + 1 else d_b
        assert L.vdl2gpu_launch_phase_mag(src.data_ptr(), n, d_ph[off[j]:].data_ptr(), d_mg[off[j]:].data_ptr(), exact, None) == 0
    last = off[1:] - 1
    got_ph = d_ph.cpu().numpy().view(np.uint32)[last]
    got_mg = d_mg.cpu().numpy().view(np.uint32)[last]
    bad = np.flatnonzero(~same(got_ph, X["phase"]))
    assert bad.size == 0, f"{bad.size} phases differ, first {[ph.CASES[i] for i in bad[:3]]}"
    bad = np.flatnonzero(~same(got_mg, X["mag"]))
    assert bad.size == 0, f"{bad.size} magnitudes differ, first {[ph.CASES[i] for i in bad[:3]]}"


@pytest.mark.parametrize("exact", [0, 1], ids=["fast", "libm"])
def test_phase_mag_stub_signed_zeros(exact):
    """atan2(+-0, +x) = +-0, atan2(+-0, -x) = +-pi, atan2(+-y, +-0) = +-pi/2, atan2(+-0, +-0) by the same rules"""
    import torch
    L = vd.load_library()
    pi, pio2 = np.float32(np.pi), np.float32(np.pi / 2)
    rows = []
    for im in (0.0, -0.0):
        for re in (0.0, -0.0, 1.0, 0.25, -1.0, -0.25):
            s = -1.0 if np.signbit(im) else 1.0
            rows.append((re, im, np.float32(s * (pi if np.signbit(re) else 0.0)), np.float32(abs(re))))
    for re in (0.0, -0.0):
        for im in (1.0, -1.0, 3e-5, -3e-5):
            rows.append((re, im, np.float32(np.sign(im) * pio2), np.float32(abs(im))))
    x = np.array([(r[0], r[1]) for r in rows], np.float32)
    want_ph = np.array([r[2] for r in rows], np.float32).view(np.uint32)
    want_mg = np.array([r[3] for r in rows], np.float32).view(np.uint32)
    d_x = torch.from_numpy(x).cuda()
    d_ph = torch.empty(len(rows), dtype=torch.float32, device="cuda")
    d_mg = torch.empty(len(rows), dtype=torch.float32, device="cuda")
    _launch_phase_mag(L, d_x, len(rows), d_ph, d_mg, exact)
    got_ph, got_mg = d_ph.cpu().numpy().view(np.uint32), d_mg.cpu().numpy().view(np.uint32)
    for k, r in enumerate(rows):
        assert got_ph[k] == want_ph[k], (r[:2], hex(got_ph[k]), hex(want_ph[k]))
        assert got_mg[k] == want_mg[k], (r[:2], hex(got_mg[k]), hex(want_mg[k]))


@pytest.fixture(scope="module")
def device_functions(tmp_path_factory):
    d = tmp_path_factory.mktemp("phasehard_dev")
    so = os.path.join(str(d), "libphasehard_dev.so")
    subprocess.check_call([vb._nvcc()] + vb.NVCC_FLAGS + ["-shared", "-o", so, os.path.join(HERE, "hostsim", "phase_hard_device.cu")])
    L = C.CDLL(so)
    L.phase_hard_run.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return L


def test_device_functions_on_every_case(device_functions):
    x = np.ascontiguousarray(SAMPLES)
    val = np.zeros((N, 7), np.float32)
    slow = np.zeros((N, 4), np.int32)
    assert device_functions.phase_hard_run(x.ctypes.data, N, val.ctypes.data, slow.ctypes.data) == 0
    val = val.view(np.uint32)
    libdevice_bad = np.flatnonzero(~same(val[:, 6], X["phase"]))
    print(f"\nlibdevice's (float)atan2 differs from the narrowed correctly rounded double on {libdevice_bad.size} of {N} "
          f"fixture entries: {[(ph.CASES[i]['re'], ph.CASES[i]['im'], ph.CASES[i]['cls'], ph.CASES[i]['dist']) for i in libdevice_bad]}")
    for name, bad in ph.contract_failures(val, slow, X).items():
        assert bad.size == 0, f"device {name}: {bad.size} entries neither slow nor as expected, first {[ph.CASES[i] for i in bad[:3]]}"
    bad = np.flatnonzero(~same(val[:, 4], X["phase"]))
    assert bad.size == 0, f"device vdl2_phase_of: {bad.size} entries differ, first {[ph.CASES[i] for i in bad[:3]]}"
    bad = np.flatnonzero(~same(val[:, 5], X["mag"]))
    assert bad.size == 0, f"device vdl2_mag_of: {bad.size} entries differ, first {[ph.CASES[i] for i in bad[:3]]}"
    # the entries next to a midpoint must have left the fast paths (the guard, with the device's own seeds)
    near = np.array([c["cls"] in ("random", "break", "pow2") and abs(c["dist"]) < 1 for c in ph.CASES])
    assert slow[near, 0].all() and slow[near, 1].all()


N_CH = 48


def _stage_rows():
    """[n_dec][48][2]: the finite fixture entries glibc rounds like the device, three times in different orders"""
    keep = np.array([np.isfinite(c0) and np.isfinite(c1) and c["glibc"] == c["phase"]
                     for c0, c1, c in zip(X["re"], X["im"], ph.CASES)])
    s = SAMPLES[keep]
    want = X["phase"][keep]
    order = np.concatenate([np.arange(s.shape[0]), np.roll(np.arange(s.shape[0]), 17), np.roll(np.arange(s.shape[0]), 101)])
    order = np.concatenate([order, order[:(-order.size) % N_CH]])
    return np.ascontiguousarray(s[order].reshape(-1, N_CH, 2)), want[order].reshape(-1, N_CH)


@pytest.fixture(scope="module")
def k2lib(tmp_path_factory):
    return ks.build(tmp_path_factory.mktemp("k2state_hard"))


@pytest.mark.parametrize("env", [None, dict(VDL2GPU_K2A=0)], ids=["default", "k2a0"])
def test_stage_on_fixture_rows(k2lib, env):
    dec, want = _stage_rows()
    freqs = [kc.CENTER + 25000 * (c - N_CH // 2) for c in range(N_CH)]
    bounds = kc.launch_bounds(dec.shape[0])
    max_dec = max(n for _, n in bounds)
    dev = gs.DeviceStage(k2lib, dec, freqs, 0.0, vd.FLAG_TRACE, max_dec, env)
    host = ks.HostStage(k2lib, dec, freqs, 0.0, dev.n_slots, ks.PER_SAMPLE)
    what = f"fixture rows {env or 'default'}"
    try:
        gs.check_fresh(dev, host)
        for a, n in bounds:
            dev.sync_slice(a, n)
            host.step(n)
            rows = dev.plane("phase", kc.RING + n)[kc.RING:]
            bad = np.argwhere(rows != want[a:a + n])
            assert bad.size == 0, f"{what}: phase row {a + bad[0][0]} channel {bad[0][1]}: {rows[tuple(bad[0])]:#x}, " \
                                  f"expected {want[a + bad[0][0], bad[0][1]]:#x}"
            dslot = gs.check_launch(dev, host, a, n, what)
            dev.burst_fec()
            gs.check_no_leak(dev, dslot, what)
    finally:
        host.close()
        dev.close()
