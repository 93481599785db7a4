"""ctypes binding of tests/hostsim/libhostsim.so (TEST-ONLY host build of the device functions)."""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "..", "..", "dumpvdl2_b200", "csrc")
_LIB = None


class Rec(C.Structure):
    _fields_ = [("rec_bytes", C.c_uint32), ("channel", C.c_uint32), ("burst_seq", C.c_uint32), ("status", C.c_int32),
                ("n_frames", C.c_uint32), ("datalen_bits", C.c_uint32), ("syndrome", C.c_uint32),
                ("num_fec_corrections", C.c_int32), ("frame_pwr", C.c_float), ("mag_nf", C.c_float),
                ("ppm_error", C.c_float), ("num_blocks", C.c_uint32), ("sync_lo", C.c_uint32), ("sync_hi", C.c_uint32),
                ("freq", C.c_uint32), ("frame_bytes", C.c_uint32), ("rs_ret", C.c_int8 * 12), ("pad", C.c_uint32)]


class Ev(C.Structure):
    _fields_ = [("channel", C.c_uint32), ("kind", C.c_uint32), ("dec_index", C.c_uint64),
                ("i", C.c_int32 * 8), ("f", C.c_float * 8)]


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libhostsim.so")
        deps = [os.path.join(_HERE, "hostsim.cpp")] + [os.path.join(_CSRC, f) for f in ("vdl2_core.cuh", "vdl2_types.h", "vdl2_tables_host.h")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                                   "-I", _CSRC, "-o", so, deps[0]])
        _LIB = C.CDLL(so)
        _LIB.hostsim_rs_verify.argtypes = [C.c_void_p, C.c_int]
        _LIB.hostsim_rs_verify_lanes.argtypes = [C.c_void_p, C.c_int]
        _LIB.hostsim_crc16.restype = C.c_uint16
        _LIB.hostsim_crc16.argtypes = [C.c_void_p, C.c_uint32]
        _LIB.hostsim_header_fix.restype = C.c_uint32
        _LIB.hostsim_header_fix.argtypes = [C.c_uint32, C.POINTER(C.c_uint32)]
        _LIB.hostsim_synd_weight.restype = C.c_uint32
    return _LIB


def parse_records(buf, used):
    """-> list of dict(record fields..., frames=[(bytes, crc)])"""
    out, off = [], 0
    raw = bytes(buf[:used])
    while off + C.sizeof(Rec) <= used:
        r = Rec.from_buffer_copy(raw, off)
        tab = np.frombuffer(raw, np.uint32, r.n_frames, off + C.sizeof(Rec))
        p = off + C.sizeof(Rec) + 4 * r.n_frames
        frames = []
        for t in tab:
            ln, crc = int(t) & 0xFFFF, int(t) >> 16
            frames.append((raw[p:p + ln], crc)); p += ln
        out.append(dict(channel=r.channel, burst_seq=r.burst_seq, status=r.status, datalen_bits=r.datalen_bits,
                        syndrome=r.syndrome, num_fec_corrections=r.num_fec_corrections, frame_pwr=np.float32(r.frame_pwr),
                        mag_nf=np.float32(r.mag_nf), ppm_error=np.float32(r.ppm_error), num_blocks=r.num_blocks,
                        sync_dec_index=r.sync_lo | (r.sync_hi << 32), freq=r.freq, rs_ret=list(r.rs_ret)[:9], frames=frames))
        off += r.rec_bytes
    return out


def k1(samples, rate, oversample, centerfreq, freqs):
    s = np.ascontiguousarray(samples, np.float32).reshape(-1, 2)
    f = np.ascontiguousarray(freqs, np.uint32)
    n_dec = s.shape[0] // oversample
    dec = np.zeros((n_dec, len(f), 2), np.float32)
    nd = C.c_uint32(0)
    lib().hostsim_k1(s.ctypes.data_as(C.c_void_p), C.c_uint32(s.shape[0]), C.c_uint32(rate), C.c_uint32(oversample),
                     C.c_uint32(centerfreq), f.ctypes.data_as(C.c_void_p), C.c_uint32(len(f)), dec.ctypes.data_as(C.c_void_p), C.byref(nd))
    return dec


def k2k3(dec, freqs, rate, max_ppm=0.0, trace=True, use_pre=True, launches=None, event_cap=1 << 16):
    """K2 + K3 over a whole decimated stream, fed in launches of the given lengths (repeated; default 1024)"""
    d = np.ascontiguousarray(dec, np.float32)
    sched = np.ascontiguousarray(launches if launches is not None else [], np.uint32)
    f = np.ascontiguousarray(freqs, np.uint32)
    n_dec, n_ch = d.shape[0], d.shape[1]
    out = np.zeros(8 << 20, np.uint8)
    used, nrec, nev = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
    cap = event_cap
    ev = (Ev * cap)()
    cnt = np.zeros((n_ch, 2), np.uint32)
    rc = lib().hostsim_k2k3(d.ctypes.data_as(C.c_void_p), C.c_uint32(n_dec), C.c_uint32(n_ch), f.ctypes.data_as(C.c_void_p),
                            C.c_uint32(rate), C.c_float(max_ppm), out.ctypes.data_as(C.c_void_p), C.c_uint32(out.size),
                            C.byref(used), C.byref(nrec), C.cast(ev, C.c_void_p) if trace else None, C.c_uint32(cap), C.byref(nev),
                            cnt.ctypes.data_as(C.c_void_p), C.c_int(int(use_pre)),      # 0 per-sample, 1 blocked, 2 blocked + unwrap table, 3 ring walk
                            sched.ctypes.data_as(C.c_void_p) if sched.size else None, C.c_uint32(sched.size))
    assert rc == 0, f"hostsim pool overflow / error {rc}"
    assert nev.value < cap, "hostsim event buffer full"
    recs = parse_records(out, used.value)
    events = [dict(channel=ev[k].channel, kind=ev[k].kind, dec_index=ev[k].dec_index, i=list(ev[k].i),
                   f=np.array(list(ev[k].f), np.float32)) for k in range(nev.value)]
    return recs, events, cnt


def k3(bits, datalen_bits):
    """Run the K3 device functions on one burst (scrambled bits incl. the 25 header bits)."""
    b = np.ascontiguousarray(bits, np.uint8)
    out = np.zeros(4096, np.uint8); lens = np.zeros(1100, np.uint32); crcs = np.zeros(1100, np.uint16)
    n = C.c_uint32(0); corr = C.c_int32(0); rs = np.zeros(9, np.int8)
    st = lib().hostsim_k3(b.ctypes.data_as(C.c_void_p), C.c_uint32(b.size), C.c_uint32(datalen_bits), out.ctypes.data_as(C.c_void_p),
                          C.c_uint32(out.size), lens.ctypes.data_as(C.c_void_p), crcs.ctypes.data_as(C.c_void_p), C.c_uint32(1100),
                          C.byref(n), C.byref(corr), rs.ctypes.data_as(C.c_void_p))
    frames, off = [], 0
    for k in range(n.value):
        frames.append(bytes(out[off:off + lens[k]])); off += int(lens[k])
    return st, frames, corr.value, rs, crcs[:n.value].copy()
