"""CPU: restarting one receiver of a ragged mixed-receivers context (vdl2gpu_restart_receiver,
Vdl2MixedReceivers.restart_receiver) without a GPU.  The restart rule of vdl2_core.cuh - the fresh state create gives a
channel and a restart gives it, the three K2 fields a restart keeps, the burst-pool slot a dropped burst hands back - and
a host walk of the K2 / K3 device functions with restarts at cuts (tests/hostsim/restart.cpp, TEST-ONLY): per channel it
must equal the oracle on everything before the first cut followed by a fresh oracle per segment (frames, events,
counters), with a cut inside a burst and a cut within 160 samples of the previous one.  Then the refusals that need no
device and the Python ValueErrors."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth
from oracle import pyoracle as po
from tests import util
from tests.hostsim import pyhostsim as hs

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "dumpvdl2_b200", "csrc")
EINVAL = -1
K2_NFIELDS, K1_NFIELDS = 29, 10
(K2_PHERR1, K2_PHERR2, K2_MAG_NF, K2_STATE, K2_NEED_BITS, K2_SLOT, K2_BURST_SEQ, K2_FREQ, K2_CNT_SYNC, K2_CNT_HDR_GOOD,
 K2_PURE_RUN) = 4, 5, 8, 14, 18, 21, 22, 25, 26, 27, 28
K1_DPHI = 9
ABANDONED = 0x80000000


@pytest.fixture(scope="module")
def rs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("restart") / "librestart.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I", CSRC, "-o", so, os.path.join(HERE, "hostsim", "restart.cpp")])
    L = C.CDLL(so)
    L.hostsim_restart_k2k3.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                       C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                       C.c_void_p, C.c_void_p]
    L.hostsim_fresh_state.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.hostsim_restart_entry_bytes.restype = C.c_size_t
    return L


def _fresh(rs, centre, freq, rate, restart_from=None):
    k1, k2 = np.zeros(K1_NFIELDS, np.uint32), np.zeros(K2_NFIELDS, np.uint32)
    ready, n_ready = np.zeros(1, np.uint32), C.c_uint32(0)
    src = None if restart_from is None else np.ascontiguousarray(restart_from, np.uint32)
    rs.hostsim_fresh_state(centre, freq, rate, None if src is None else src.ctypes.data, k1.ctypes.data, k2.ctypes.data,
                           ready.ctypes.data, C.byref(n_ready))
    return k1, k2, ready[:n_ready.value].tolist()


def _f32(x):
    return int(np.float32(x).view(np.uint32))


def test_restart_entry_is_12_bytes(rs):
    assert rs.hostsim_restart_entry_bytes() == 12


@pytest.mark.parametrize("os_,off", [(10, 25000), (20, -75000), (13, 0), (10, -487500)])
def test_fresh_state_is_the_reference_start(rs, os_, off):
    """create's state (initial_state) comes from the same rule as a restart: zero filter and NCO with the step of
    src/demod.c:385, and vdl2_channel_init + demod_reset (src/demod.c:205-220,379-392)"""
    centre, rate = 136500000, 105000 * os_
    k1, k2, ready = _fresh(rs, centre, centre + off, rate)
    want_dphi = 0 if off == 0 else int(np.int32(np.float32(np.float32(np.float32(np.float32(centre) - np.float32(centre + off))
                                                                      / np.float32(rate)) * np.float32(256.0)) * np.float32(65536.0)))
    assert k1[K1_DPHI] == np.uint32(want_dphi & 0xFFFFFFFF)
    assert not k1[:K1_DPHI].any()
    want = np.zeros(K2_NFIELDS, np.uint32)
    want[K2_MAG_NF], want[K2_PHERR1], want[K2_PHERR2] = _f32(2.0), _f32(1000.0), _f32(1000.0)
    want[K2_NEED_BITS], want[K2_SLOT], want[K2_FREQ], want[K2_PURE_RUN] = 25, 0xFFFFFFFF, centre + off, 0x40000000
    assert k2.tolist() == want.tolist() and ready == []


@pytest.mark.parametrize("slot", [-1, 0, 17])
def test_restart_keeps_sequence_and_counters_and_hands_back_the_slot(rs, slot):
    rng = np.random.default_rng(slot + 5)
    old = rng.integers(1, 1 << 31, K2_NFIELDS).astype(np.uint32)
    old[K2_SLOT] = np.uint32(slot & 0xFFFFFFFF)
    _, k2, ready = _fresh(rs, 136500000, 136525000, 1050000, restart_from=old)
    _, want, _ = _fresh(rs, 136500000, 136525000, 1050000)
    for f in (K2_BURST_SEQ, K2_CNT_SYNC, K2_CNT_HDR_GOOD):
        want[f] = old[f]
    assert k2.tolist() == want.tolist()
    assert ready == ([] if slot < 0 else [slot | ABANDONED])


# ---- the host walk with restarts at cuts against one fresh oracle per segment ----
def _walk(rs, dec, freqs, cuts, rate):
    d = np.ascontiguousarray(dec, np.float32)
    n_dec, n_ch = d.shape[0], d.shape[1]
    fr = np.ascontiguousarray(freqs, np.uint32)
    cu = np.ascontiguousarray(cuts, np.uint32)
    out = np.zeros(8 << 20, np.uint8)
    used, nrec, nev = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
    cap = 1 << 16
    ev = (hs.Ev * cap)()
    cnt = np.zeros((n_ch, 2), np.uint32)
    pool = np.zeros(4, np.uint32)
    rc = rs.hostsim_restart_k2k3(d.ctypes.data, n_dec, n_ch, fr.ctypes.data, cu.ctypes.data, cu.size, rate, out.ctypes.data,
                                 out.size, C.byref(used), C.byref(nrec), C.cast(ev, C.c_void_p), cap, C.byref(nev),
                                 cnt.ctypes.data, pool.ctypes.data)
    assert rc == 0, f"hostsim restart walk: {rc}"
    recs = hs.parse_records(out, used.value)
    events = [dict(channel=ev[k].channel, kind=ev[k].kind, dec_index=ev[k].dec_index, i=list(ev[k].i),
                   f=np.array(list(ev[k].f), np.float32)) for k in range(nev.value)]
    return recs, events, cnt, pool


def _in_burst_cut(events, lo, hi, after=40):
    """a decimated index in [lo, hi) at which some channel is `after` samples into the data of a burst with a good header"""
    for e in sorted(events, key=lambda e: e["dec_index"]):
        if e["kind"] == 2 and e["i"][3] == 0 and lo <= e["dec_index"] + after < hi:
            return int(e["dec_index"]) + after
    raise AssertionError("no burst to cut into")


@pytest.mark.parametrize("os_,fmt", [(10, "u8"), (20, "s16")])
def test_walk_with_restarts_equals_segmented_oracles(rs, os_, fmt):
    bpp = 4 if fmt == "s16" else 2
    rate = 105000 * os_
    ofmt = po.FMT_S16 if fmt == "s16" else po.FMT_U8
    w = os_ * bpp
    streams = []
    for k in range(2):
        iq, offs, _ = synth.traffic_stream(rate, 0.7, 4, 8.0, 24.0, -20.0, 0x52535400 + 16 * k + os_, fmt)
        b = np.ascontiguousarray(iq).view(np.uint8).reshape(-1)
        streams.append((b[:b.size // w * w], offs))
    # segment tunings: the start, a reset (same tuning), then a retune to another centre and other frequencies, fed another
    # stream from then on, and a reset of that
    a, b = streams
    ca, cb = 136500000, 136725000
    tunings = [(ca, [ca + int(o) for o in a[1]])] * 2 + [(cb, [cb + int(o) for o in b[1][::-1]])] * 2
    na, nb = a[0].size // w, b[0].size // w
    whole_a = po.Oracle(rate, os_, ofmt, *tunings[0], trace=True)
    whole_a.process(a[0])
    c1 = _in_burst_cut(whole_a.events(), na // 5, na // 2)
    c2 = c1 + 100                                           # within 160 samples of the previous cut
    whole_b = po.Oracle(rate, os_, ofmt, *tunings[2], trace=True)
    whole_b.process(b[0])
    d3 = _in_burst_cut(whole_b.events(), nb // 3, nb - 3000)
    cuts = [c1, c2, c2 + d3]
    total = c2 + nb
    bounds = [0] + cuts + [total]
    pieces = [a[0][:c1 * w], a[0][c1 * w:c2 * w], b[0][:d3 * w], b[0][d3 * w:]]
    oracles = []
    for k, (cf, fr) in enumerate(tunings):
        o = po.Oracle(rate, os_, ofmt, cf, fr, trace=True, dec_tap=True)
        o.process(pieces[k])
        oracles.append(o)
    dec = np.concatenate([o.dec_samples() for o in oracles])
    assert dec.shape[0] == total
    recs, events, cnt, pool = _walk(rs, dec, np.concatenate([fr for _, fr in tunings]), cuts, rate)

    got = sorted((r["channel"], r["burst_seq"], k, d, r["num_fec_corrections"], r["sync_dec_index"], r["freq"],
                  np.float32(r["frame_pwr"]).view(np.uint32), np.float32(r["ppm_error"]).view(np.uint32))
                 for r in recs for k, (d, _) in enumerate(r["frames"]))
    want, want_ev = [], []
    seq = np.zeros(4, np.int64)
    sync, hdr = np.zeros(4, np.int64), np.zeros(4, np.int64)
    abandoned = 0
    for k, o in enumerate(oracles):
        fr = tunings[k][1]
        for f in o.frames():
            want.append((f.channel, f.burst_seq + int(seq[f.channel]), f.idx, f.data, f.num_fec_corrections,
                         f.sync_dec_index + bounds[k], fr[f.channel], np.float32(f.frame_pwr).view(np.uint32),
                         np.float32(f.ppm_error).view(np.uint32)))
        ev = o.events()
        want_ev += [dict(e, dec_index=e["dec_index"] + bounds[k]) for e in ev]
        oc = o.counters().astype(np.int64)
        seq += oc[:, 2]
        sync += oc[:, 0]
        hdr += oc[:, 1]
        # bursts in progress at the segment's end: a good header and no completion (kind 3) before the cut
        in_progress = sum(1 for e in ev if e["kind"] == 2 and e["i"][3] == 0) - sum(1 for e in ev if e["kind"] == 3)
        if k < len(oracles) - 1:
            abandoned += in_progress
        else:
            held = in_progress
    assert len(want) > 10
    assert got == sorted(want)
    assert len(recs) == sum(sum(1 for e in o.events() if e["kind"] == 3) for o in oracles)
    util.assert_events_equal(events, want_ev, f"restart walk os {os_}")
    assert cnt[:, 0].tolist() == sync.tolist() and cnt[:, 1].tolist() == hdr.tolist()
    n_slots, free, held_now, back = (int(x) for x in pool)
    assert back == abandoned and abandoned >= 2                 # the cuts at c1 and c3 fall inside bursts
    assert held_now == held and free + held_now == n_slots      # every abandoned slot is back in the pool


# ---- refusals that need no device ----
def test_restart_refuses_without_a_context():
    L = vd.load_library()
    fr = np.zeros(4, np.uint32)
    assert L.vdl2gpu_restart_receiver(None, 0, 0, None) == EINVAL
    assert L.vdl2gpu_restart_receiver(None, 0, 136500000, fr.ctypes.data) == EINVAL
    assert "no context" in L.vdl2gpu_last_error().decode()


def _detached(receivers):
    """a Vdl2MixedReceivers with the bookkeeping restart_receiver checks, but no library context behind it"""
    g = vd.Vdl2MixedReceivers.__new__(vd.Vdl2MixedReceivers)
    g.L, g.h = None, None
    g.receivers = [(cf, list(fr)) for cf, fr in receivers]
    g.n_receivers = len(receivers)
    g.freqs = np.ascontiguousarray([f for _, fr in receivers for f in fr], np.uint32)
    g._first = np.concatenate([[0], np.cumsum([len(fr) for _, fr in receivers])]).astype(np.int64)
    return g


def test_python_checks_the_frequency_count_before_the_library():
    g = _detached([(136500000, [136525000, 136550000]), (136900000, [136975000])])
    with pytest.raises(ValueError, match="receiver 0 has 2 channels, 3 frequencies"):
        g.restart_receiver(0, freqs=[1, 2, 3])
    with pytest.raises(ValueError, match="receiver 1 has 1 channels, 0 frequencies"):
        g.restart_receiver(1, centerfreq=136800000, freqs=[])
    with pytest.raises(ValueError, match="receiver 2 of 2"):
        g.restart_receiver(2)
    with pytest.raises(ValueError, match="receiver -1 of 2"):
        g.restart_receiver(-1)
    assert g.receivers == [(136500000, [136525000, 136550000]), (136900000, [136975000])]     # nothing changed
    assert g.freqs.tolist() == [136525000, 136550000, 136975000]
