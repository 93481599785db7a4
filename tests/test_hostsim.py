"""CPU: the device functions of dumpvdl2_b200/csrc/vdl2_core.cuh, compiled for the host (tests/hostsim,
TEST-ONLY), stepped against the oracle: K1 arithmetic (table form of the NCO), the K2 state machine and the K3
burst decoder.  This is how kernel logic is checked without a GPU; the -m gpu tests repeat it on the device."""
import numpy as np
import pytest
from oracle import pyoracle as po
from tests import cases, k3_corpus, util
from tests.hostsim import pyhostsim as hs


def _samples(case):
    b = util.case_bytes(case)
    if case["fmt"] == "s16":
        raw = b[:b.size // 2 * 2].view("<i2")
        return (raw.astype(np.float32) / np.float32(32768.0)).reshape(-1)
    return po.levels_u8()[b]


@pytest.mark.parametrize("use_pre", [5, 4, 3, 2, 1, 0], ids=["ring_nomag", "ring_staged", "ring", "blocked_lut", "blocked", "per_sample"])
@pytest.mark.parametrize("name", ["cfg2", "mixed_s16", "fec", "noisy", "wav", "hdlc_edge", "mirics_os13", "maxlen", "stress"])
def test_device_functions_on_host_match_oracle(name, use_pre):
    c = (cases.ALL_GOLDEN.get(name) or getattr(cases, "case_" + name))()
    o = util.run_oracle(c, trace=True, dec_tap=True)
    odec = o.dec_samples()
    s = _samples(c)
    s = s[:s.size // 2 * 2]
    hdec = hs.k1(s, c["fs"], c["oversample"], c["centerfreq"], c["freqs"])
    assert hdec.shape == odec.shape
    assert np.array_equal(hdec.view(np.uint32), odec.view(np.uint32)), "K1 arithmetic differs from the oracle"
    recs, ev, cnt = hs.k2k3(odec, c["freqs"], c["fs"], use_pre=use_pre)
    got = []
    for r in recs:
        for k, (data, crc) in enumerate(r["frames"]):
            got.append((r["channel"], r["burst_seq"], k, data, r["num_fec_corrections"], r["sync_dec_index"],
                        np.float32(r["frame_pwr"]).view(np.uint32), np.float32(r["mag_nf"]).view(np.uint32),
                        np.float32(r["ppm_error"]).view(np.uint32), crc == 0xF0B8 and len(data) >= 11))
    want = [(f.channel, f.burst_seq, f.idx, f.data, f.num_fec_corrections, f.sync_dec_index,
             np.float32(f.frame_pwr).view(np.uint32), np.float32(f.mag_nf).view(np.uint32),
             np.float32(f.ppm_error).view(np.uint32), f.fcs_ok) for f in o.frames()]
    assert sorted(got) == sorted(want)
    util.assert_events_equal(ev, o.events(), f"hostsim events [{name}]")
    oc = o.counters()
    assert np.array_equal(cnt[:, 0], oc[:, 0]) and np.array_equal(cnt[:, 1], oc[:, 1])
    # burst-level bookkeeping: status and per-block RS results
    ob = {(e["channel"], i): e for i, e in enumerate([e for e in o.events() if e["kind"] == 3])}
    assert len(recs) == len(ob)


def test_max_ppm_veto_in_blocked_walk():
    """A vetoed preamble leaves the sample clock at the sync point (src/demod.c:179,190-192): the blocked walk
    must fall back to the per-sample path there."""
    c = dict(cases.case_mixed_s16()); c["max_ppm"] = 1.0
    o = util.run_oracle(c, trace=True, dec_tap=True)
    for mode in (1, 2, 3, 4, 5):
        _check_veto(c, o, mode)


def _check_veto(c, o, mode):
    recs, ev, cnt = hs.k2k3(o.dec_samples(), c["freqs"], c["fs"], max_ppm=1.0, use_pre=mode)
    got = sorted((r["channel"], r["burst_seq"], k, d, r["sync_dec_index"]) for r in recs for k, (d, _) in enumerate(r["frames"]))
    want = sorted((f.channel, f.burst_seq, f.idx, f.data, f.sync_dec_index) for f in o.frames())
    assert got == want and len(want) < 14
    util.assert_events_equal(ev, o.events(), "hostsim max_ppm events")
    assert any(e["kind"] == 1 and e["i"][3] == 0 for e in ev)


def test_rs_decoder_matches_oracle_beyond_capacity():
    """Same result as the oracle (== Karn's decoder) for 0..7 errors incl. failures and miscorrections."""
    import ctypes as C
    rng = np.random.default_rng(7)
    L = hs.lib()
    for trial in range(3000):
        nfec = [6, 6, 6, 4, 2][trial % 5]
        msg = np.zeros(249, np.uint8)
        k = 249 if nfec == 6 else int(rng.integers(3, 68))
        msg[:k] = rng.integers(0, 256, k, dtype=np.uint8)
        cw = po.rs_encode(msg)
        cw[249 + nfec:] = 0
        for _ in range(int(rng.integers(0, 8))):
            cw[int(rng.integers(0, 249 + nfec))] ^= int(rng.integers(1, 256))
        want_ret, want = po.rs_verify(cw, nfec)
        mine = cw.copy()
        got_ret = L.hostsim_rs_verify(mine.ctypes.data, nfec)
        assert got_ret == want_ret and np.array_equal(mine, want), (trial, nfec, got_ret, want_ret)
        lanes = cw.copy()          # the warp-cooperative form of K3 (lane-partial syndromes, lane-strided Chien search)
        got_ret = L.hostsim_rs_verify_lanes(lanes.ctypes.data, nfec)
        assert got_ret == want_ret and np.array_equal(lanes, want), ("lanes", trial, nfec, got_ret, want_ret)


def test_header_code_and_crc_match_oracle():
    import ctypes as C
    L, O = hs.lib(), po.lib()
    rng = np.random.default_rng(11)
    words = list(rng.integers(0, 1 << 22, 20000)) + [O.vo_header_encode(int(n)) ^ (1 << int(b)) for n in range(0, 0x4000, 97) for b in range(25)]
    for w in words:
        w = int(w) & 0x3FFFFF
        s = C.c_uint32(0)
        fixed = L.hostsim_header_fix(w, C.byref(s))
        ow = C.c_uint32(w)
        os_ = O.vo_header_decode(C.byref(ow))
        assert (fixed, s.value) == (ow.value, os_)
        assert L.hostsim_synd_weight(s.value) == O.vo_synd_weight(os_)
    for n in (0, 1, 2, 11, 300):
        d = rng.integers(0, 256, n, dtype=np.uint8)
        assert L.hostsim_crc16(d.ctypes.data if n else None, n) == po.crc16(d.tobytes())


def test_library_tables_match_oracle():
    import ctypes as C
    for rate in (1050000, 2100000, 1365000):
        lv = np.zeros(256, np.float32); s = np.zeros(257, np.float32); c = np.zeros(257, np.float32)
        A = np.zeros(3, np.float32); B = np.zeros(3, np.float32); X = np.zeros(16, np.float32); d = np.zeros(1, np.float32); P = np.zeros(16, np.float32)
        hs.lib().hostsim_tables(C.c_uint32(rate), *[C.c_void_p(a.ctypes.data) for a in (lv, s, c, A, B, X, d, P)])
        os_, oc = po.sincos_lut(); oa, ob = po.lpf_design(rate); ox, od, op = po.sync_consts()
        for got, want in ((lv, po.levels_u8()), (s, os_), (c, oc), (A, oa), (B, ob), (X, ox), (P, op)):
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        assert d[0] == od
        # the pipelined K1 relies on nothing about A; but document the structure the strict design has
        assert A[1] == 2 * A[0] and A[2] == A[0]


def test_fp32_unwrap_update_equals_the_double_arithmetic_of_the_reference():
    """src/demod.c:137-141 updates `unwrap` in double and narrows; the kernels use an FP32-only TwoSum form.
    Enumerate every value `unwrap` can take (<= 15 steps of +-2pi from 0) and check all transitions."""
    import ctypes as C
    L = hs.lib()
    L.hostsim_unwrap_step.restype = C.c_float
    L.hostsim_unwrap_step.argtypes = [C.c_float, C.c_float]
    two_pi = np.float64(2.0) * np.float64(np.pi)
    frontier, seen, n = {np.float32(0).tobytes()}, {np.float32(0).tobytes()}, 0
    for depth in range(15):
        nxt = set()
        for b in frontier:
            u = np.frombuffer(b, np.float32)[0]
            assert L.hostsim_unwrap_step(u, np.float32(0.5)) == u          # no jump: unchanged
            for step, sign in ((np.float32(3.2), -1.0), (np.float32(-3.2), 1.0)):   # step > pi: -2pi ; step < -pi: +2pi
                want = np.float32(np.float64(u) + sign * two_pi)
                got = np.float32(L.hostsim_unwrap_step(u, step))
                assert got.tobytes() == want.tobytes(), (u, sign, got, want)
                nxt.add(want.tobytes()); n += 1
        frontier = nxt - seen
        seen |= nxt
    assert len(seen) == 77 and n == 138
    # the jump thresholds: `errdiff > M_PI` with errdiff float, M_PI double
    for x in (np.float32(np.pi), np.nextafter(np.float32(np.pi), np.float32(0)), np.nextafter(np.float32(np.pi), np.float32(4))):
        jumped = L.hostsim_unwrap_step(np.float32(0), x) != 0
        assert jumped == (np.float64(x) > np.pi)
        jumped = L.hostsim_unwrap_step(np.float32(0), -x) != 0
        assert jumped == (np.float64(-x) < -np.pi)


def test_unwrap_transition_table_equals_the_double_arithmetic_of_the_reference():
    """The K2 walk replaces the arithmetic by a 77-state transition table built at start-up (vdl2_tables_host.h):
    every row must hold exactly fl32((double)u -/+ 2pi) for its state, and walking the table along random step
    sequences must give the same values as the arithmetic form."""
    import ctypes as C
    L = hs.lib()
    lut = np.zeros(80 * 6, np.uint32)
    n = L.hostsim_unwrap_lut(lut.ctypes.data_as(C.c_void_p))
    assert n == 77
    two_pi = np.float64(2.0) * np.float64(np.pi)
    rows = lut.reshape(80, 3, 2)
    vals = {}                                  # state -> value, from the rows pointing at it
    assert rows[0, 0, 0] == 0 and rows[0, 0, 1] == 0
    vals[0] = np.float32(0)
    depth = {0: 0}
    order = [0]
    for s in order:                            # breadth first, like the builder
        u = vals[s]
        assert rows[s, 0, 0] == s * 24 and rows[s, 0, 1:].view(np.float32)[0].tobytes() == u.tobytes()
        if depth[s] >= 15:
            continue
        for j, sign in ((1, -1.0), (2, 1.0)):
            want = np.float32(np.float64(u) + sign * two_pi)
            nxt = int(rows[s, j, 0]) // 24
            assert rows[s, j, 0] % 24 == 0 and nxt < n
            assert rows[s, j, 1:].view(np.float32)[0].tobytes() == want.tobytes(), (s, j)
            if nxt not in vals:
                vals[nxt] = want; depth[nxt] = depth[s] + 1; order.append(nxt)
            assert vals[nxt].tobytes() == want.tobytes()
    assert len(vals) == 77
    L.hostsim_unwrap_step.restype = C.c_float
    L.hostsim_unwrap_step.argtypes = [C.c_float, C.c_float]
    L.hostsim_unwrap_lut_step.restype = C.c_float
    L.hostsim_unwrap_lut_step.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.c_float]
    rng = np.random.default_rng(77)
    for trial in range(300):
        row, u = C.c_uint32(0), np.float32(0)
        for step in rng.uniform(-6.2, 6.2, 15).astype(np.float32):
            u = np.float32(L.hostsim_unwrap_step(u, step))
            got = np.float32(L.hostsim_unwrap_lut_step(lut.ctypes.data_as(C.c_void_p), C.byref(row), step))
            assert got.tobytes() == u.tobytes()


def _check_k3(it):
    """the host form of K3 on one corpus item equals the oracle's answer, FCS residues included"""
    st, fr, corr, rs, crcs = hs.k3(it["bits"], it["datalen_bits"])
    w = it["want"]
    assert (st, fr, corr) == (w["status"], w["frames"], w["corr"]), (it["kind"], st, w["status"], len(fr), len(w["frames"]))
    assert [int(r) for r in rs] == w["rs"], (it["kind"], list(rs), w["rs"])
    assert [int(c) for c in crcs] == [po.crc16(f) for f in fr]


def _items(kind):
    return [it for it in k3_corpus.corpus() if it["kind"] == kind]


@pytest.mark.parametrize("trial", range(40))
def test_burst_decoder_matches_oracle_on_hdlc_edge_cases(trial):
    """K3 device functions (de-interleave, RS, HDLC unstuff, FCS) against the oracle's restatement of
    src/decode.c:259-380 + src/bitstream.c:109-150 on crafted payloads (k3_corpus.hdlc_edge_payload): repeated / missing
    flags, aborts (seven ones), frames that are not whole octets, back-to-back flags, length cuts, multi-block and
    short-block bursts, RS errors within and beyond capacity."""
    mine = [it for it in _items("hdlc_edge") if it["trial"] == trial]
    if not mine:
        pytest.skip("payload too short for FEC")
    _check_k3(mine[0])


@pytest.mark.parametrize("n_octets", k3_corpus.GEOMETRY_LENGTHS)
def test_burst_decoder_block_geometry_edges(n_octets):
    """Block geometry corners of src/decode.c:124-133,222-297: last-block lengths around the FEC-octet thresholds
    (2|3, 30|31, 67|68), exact multiples of 249, and the maximum transmission length (9 blocks, 2047 octets),
    each with a couple of corrupted octets in the first and the last block."""
    mine = [it for it in _items("geometry") if it["datalen_bits"] == 8 * n_octets]
    if not mine:
        pytest.skip("no FEC octets for this length")
    nblk = -(-n_octets // 249)
    for it in mine:
        _check_k3(it)
        assert sum(r != -128 for r in it["want"]["rs"]) == nblk


def test_burst_decoder_fuzz_random_payloads():
    """Random transmissions (any bit length 17..16383, random content with a sprinkling of flags, 0..8 corrupted octets
    anywhere in the code words): K3's device functions must return exactly the oracle's status, frames, correction
    count, per-block RS results and FCS residues."""
    mine = _items("fuzz")
    for it in mine:
        _check_k3(it)
    assert len(mine) > 200


def test_burst_corpus_matches_oracle_and_covers_every_rs_outcome():
    """The rest of the burst corpus the GPU burst-decoder tests decode (tests/k3_corpus.py) through the host form of K3:
    RS blocks past capacity, geometry lengths of 5-9 blocks, bursts of hundreds of frames, truncated bursts and the
    one-block volume.  The corpus must hold every RS outcome, judged from the oracle's answers: correct decodes,
    failures (deg(lambda) != number of roots), miscorrections, a failure in the first and in a middle block, a
    miscorrected shortened last block; and more bursts than two grid-strides of K3."""
    items = k3_corpus.corpus()
    for it in items:
        if it["kind"] not in ("hdlc_edge", "fuzz") and not (it["kind"] == "geometry" and it["datalen_bits"] // 8 in k3_corpus.GEOMETRY_LENGTHS):
            _check_k3(it)
    assert len(items) >= 2 * k3_corpus.K3_GRID
    blocks = [b for it in items if it["kind"] == "rs" for b in it["blocks"]]
    kinds = {k for k, _, _ in blocks}
    assert {"ok", "fail", "miscorrect"} <= kinds
    assert any(k == "miscorrect" and last and nfec == 2 for k, nfec, last in blocks)
    assert any(k == "miscorrect" and last and nfec == 4 for k, nfec, last in blocks)
    first = middle = 0
    for it in items:
        r, nblk = it["want"]["rs"], -(-it["datalen_bits"] // (8 * 249))
        if it["kind"] != "rs" or nblk < 3 or -1 not in r:
            continue
        q = r.index(-1)
        assert all(x == -128 for x in r[q + 1:])                # blocks after the failure are not run
        first += q == 0
        middle += 0 < q < nblk - 1
    assert first and middle
    status = {it["want"]["status"] for it in items}
    assert {0, k3_corpus.ERR_FEC_BAD, k3_corpus.ERR_DATA_TRUNCATED, k3_corpus.ERR_FEC_TRUNCATED} <= status
    assert max(len(it["want"]["frames"]) for it in items) > 128
    assert any(it["datalen_bits"] == 8 * 2047 for it in items)
