"""The host build of the spectrum arithmetic of vdl2_core.cuh (tests/hostsim/spectrum.cpp, TEST-ONLY), compiled once per
process into a temporary directory, and numpy helpers shared by the CPU and GPU spectrum tests."""
import ctypes as C
import os
import subprocess
import tempfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "dumpvdl2_b200", "csrc")
N = 1024
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="spectrum_sim_"), "libspectrum.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                               "-I", CSRC, "-o", so, os.path.join(HERE, "hostsim", "spectrum.cpp")])
        L = C.CDLL(so)
        L.sp_q.restype = C.c_uint64
        L.sp_q.argtypes = [C.c_float]
        L.sp_fft_bin.restype = C.c_uint32
        L.sp_fft_bin.argtypes = [C.c_uint32]
        L.sp_flag.restype = C.c_uint32
        L.sp_stream.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
        L.sp_grid.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


def tables():
    win, tw = np.zeros(N, np.float32), np.zeros((N // 2, 2), np.float32)
    lib().sp_tab(win.ctypes.data, tw.ctypes.data)
    return win, tw


def segment(x):
    """x: 1024 complex samples (complex or (1024, 2) float32) -> the 1024 bin powers p in stored order (float32)"""
    a = as_pairs(x)
    assert a.shape == (N, 2)
    p = np.zeros(N, np.float32)
    lib().sp_segment(a.ctypes.data, p.ctypes.data)
    return p


def as_pairs(x):
    x = np.asarray(x)
    if np.iscomplexobj(x):
        x = np.stack([x.real, x.imag], axis=-1)
    return np.ascontiguousarray(x, np.float32).reshape(-1, 2)


def stream(x, cuts=None, restarts=None):
    """What the device keeps for one input fed the samples x in chunks of the lengths cuts (default: one chunk);
    restarts: indices of chunks that start a new grid.  -> dict(segments, pending, pow (object array of Python ints),
    peak_bits (uint32))"""
    a = as_pairs(x)
    cuts = np.ascontiguousarray([a.shape[0]] if cuts is None else cuts, np.uint32)
    assert int(cuts.sum()) == a.shape[0]
    rs = np.zeros(cuts.size, np.uint8)
    for k in restarts or ():
        rs[k] = 1
    lo, hi, pk = np.zeros(N, np.uint64), np.zeros(N, np.uint64), np.zeros(N, np.uint32)
    pos = C.c_uint64(0)
    lib().sp_stream(a.ctypes.data, cuts.ctypes.data, cuts.size, rs.ctypes.data, lo.ctypes.data, hi.ctypes.data, pk.ctypes.data, C.byref(pos))
    return dict(segments=pos.value // N, pending=pos.value % N, pow=(hi.astype(object) << 64) | lo.astype(object), peak_bits=pk)


def grid(cuts, restarts=None):
    cuts = np.ascontiguousarray(cuts, np.uint32)
    rs = np.zeros(cuts.size, np.uint8)
    for k in restarts or ():
        rs[k] = 1
    pend, segs, rest = (np.zeros(cuts.size, np.uint32) for _ in range(3))
    lib().sp_grid(cuts.ctypes.data, cuts.size, rs.ctypes.data, pend.ctypes.data, segs.ctypes.data, rest.ctypes.data)
    return pend, segs, rest


def cu8_floats(raw):
    """the floats K0 makes of cu8 bytes: the level table ((float)v - 127.5f) / 127.5f"""
    v = np.asarray(raw, np.uint8).reshape(-1).astype(np.float32)
    return ((v - np.float32(127.5)) / np.float32(127.5)).astype(np.float32).reshape(-1, 2)


def cs16_floats(raw):
    """the floats K0 makes of cs16 values: v / 32768 (exact)"""
    v = np.ascontiguousarray(raw).view("<i2").reshape(-1).astype(np.float32)
    return (v / np.float32(32768.0)).astype(np.float32).reshape(-1, 2)


def check_equal(dev, ref, what=""):
    """device record (spectrum()) against a stream() restatement, bit for bit"""
    assert dev["segments"] == ref["segments"], (what, dev["segments"], ref["segments"])
    assert dev["pending"] == ref["pending"], (what, dev["pending"], ref["pending"])
    bad = [k for k in range(N) if dev["pow"][k] != ref["pow"][k]]
    assert not bad, (what, "pow differs in bins", bad[:8])
    assert np.array_equal(np.asarray(dev["peak"], np.float32).view(np.uint32), ref["peak_bits"]), (what, "peak differs")
