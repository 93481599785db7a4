"""-m gpu: the burst decoder kernel (k3_burst_fec) burst by burst against the oracle.

The bursts of tests/k3_corpus.py (RS blocks past capacity, every block geometry, HDLC edge cases and fuzz, bursts of
hundreds of frames, truncated bursts, a volume of one-block bursts) are queued in a stage exactly as K2 hands them over
(vdl2gpu_stage_queue_bursts) and decoded by the real kernel: the warp-cooperative RS decoder, the cooperative table
builds, the second RS block per warp, the grid-stride loop over the ready list, record packing and overflow, the
per-channel counters and the return of burst-pool slots.  Every record must equal the oracle's answer field for field.
Also: the serial RS stub past capacity, and the fuzz stream through the whole pipeline."""
import ctypes as C
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import api
from oracle import pyoracle as po
from tests import cases, k3_corpus, util
from tests.hostsim import pyhostsim as hs

pytestmark = pytest.mark.gpu

HDR = 32                                  # vdl2_out_header
MAX_BITS = 25 + 8 * (2048 + 54) + 2       # VDL2_MAX_BURST_BITS
EINVAL, ETOOBIG = -1, -5


class Stage:
    """a vdl2gpu_stage of n_ch channels (max(256, 3 n_ch) burst-pool slots) on torch-allocated device memory"""

    def __init__(self, n_ch=k3_corpus.N_CHANNELS):
        import torch
        self.L = vd.load_library()
        freqs = [136000000 + 8333 * k for k in range(n_ch)]
        self.cfg, self._fr = api.make_config(2100000, 20, vd.FMT_U8, 136500000, freqs)
        self.n_ch, self.n_slots = n_ch, max(256, 3 * n_ch)
        nbytes = self.L.vdl2gpu_stage_device_bytes(n_ch, 16, 0)
        self.mem = torch.zeros(nbytes + 256, dtype=torch.uint8, device="cuda")
        self.h = C.c_void_p()
        rc = self.L.vdl2gpu_stage_create(C.byref(self.cfg), 16, C.c_void_p((self.mem.data_ptr() + 255) & ~255), nbytes, C.byref(self.h))
        assert rc == 0, self.L.vdl2gpu_last_error()

    def queue(self, items):
        arr = (api._Burst * max(1, len(items)))()
        keep = []
        for k, it in enumerate(items):
            w = _words(it["bits"])
            keep.append(w)
            b = arr[k]
            b.channel, b.datalen_bits, b.nbits, b.syndrome = it["channel"], it["datalen_bits"], it["nbits"], it["syndrome"]
            b.frame_pwr, b.mag_nf, b.ppm_error, b.freq = it["frame_pwr"], it["mag_nf"], it["ppm_error"], it["freq"]
            b.sync_dec_index = it["sync_dec_index"]
            b.words = w.ctypes.data_as(C.POINTER(C.c_uint32))
        return self.L.vdl2gpu_stage_queue_bursts(self.h, arr, len(items))

    def decode(self, region_bytes):
        """one vdl2gpu_launch_burst_fec into a region of region_bytes -> (header fields, records)"""
        import torch
        region = torch.full((region_bytes + 16,), 0xA5, dtype=torch.uint8, device="cuda")
        assert self.L.vdl2gpu_launch_burst_fec(self.h, region.data_ptr(), region_bytes, None) == 0
        torch.cuda.synchronize()
        buf = region.cpu().numpy()
        assert (buf[region_bytes:] == 0xA5).all(), "K3 wrote past the end of the region"
        h = buf[:HDR].view(np.uint32)
        head = dict(bytes_used=int(h[0]), n_records=int(h[1]), pool_overflows=int(h[2]), out_overflows=int(h[3]))
        body = buf[HDR:region_bytes]
        off = 0
        for _ in range(head["n_records"]):                  # records lie back to back from offset 0
            rec = int(body[off:off + 4].view(np.uint32)[0])
            assert rec >= 80 and rec % 16 == 0, f"bad record size {rec} at {off}"
            off += rec
        assert off <= region_bytes - HDR, "a record crosses the end of the region"
        return head, hs.parse_records(body, off), off

    def counters(self):
        out = np.zeros((self.n_ch, po.NUM_COUNTERS), np.uint64)
        assert self.L.vdl2gpu_stage_read_counters(self.h, out.ctypes.data) == 0
        return out

    def close(self):
        self.L.vdl2gpu_stage_destroy(self.h)


def _words(bits):
    """bit i at words[i / 32] >> (31 - i % 32), the last partial word zero-filled (vdl2_burst_slot.words)"""
    b = np.zeros(-(-len(bits) // 32) * 32, np.uint8)
    b[:len(bits)] = bits
    return np.ascontiguousarray(np.packbits(b).view(">u4").astype(np.uint32))


def _rec_bytes(it):
    fr = it["want"]["frames"]
    return (80 + 4 * len(fr) + sum(len(f) for f in fr) + 15) & ~15


def _check_records(recs, items, what, all_present=True):
    """every record is the oracle's answer for the burst it names (burst_seq = position in the queue call)"""
    seen = set()
    for r in recs:
        k = r["burst_seq"]
        assert k < len(items) and k not in seen, f"{what}: unexpected record burst_seq {k}"
        seen.add(k)
        it, w = items[k], items[k]["want"]
        ctx = f"{what}: burst {k} ({it['kind']}, datalen {it['datalen_bits']}, nbits {it['nbits']})"
        assert r["status"] == w["status"], f"{ctx}: status {r['status']} != {w['status']}"
        assert [f for f, _ in r["frames"]] == w["frames"], f"{ctx}: frames differ ({len(r['frames'])} vs {len(w['frames'])})"
        assert [c for _, c in r["frames"]] == [po.crc16(f) for f in w["frames"]], f"{ctx}: FCS residues differ"
        assert r["num_fec_corrections"] == w["corr"], f"{ctx}: corrections {r['num_fec_corrections']} != {w['corr']}"
        nblk = -(-it["datalen_bits"] // (8 * 249))
        assert r["num_blocks"] == nblk and r["rs_ret"] == w["rs"], f"{ctx}: rs {r['rs_ret']} != {w['rs']}"
        assert (r["channel"], r["datalen_bits"], r["syndrome"], r["freq"], r["sync_dec_index"]) == \
            (it["channel"], it["datalen_bits"], it["syndrome"], it["freq"], it["sync_dec_index"]), f"{ctx}: metadata"
        for fld in ("frame_pwr", "mag_nf", "ppm_error"):
            assert np.float32(r[fld]).view(np.uint32) == np.float32(it[fld]).view(np.uint32), f"{ctx}: {fld}"
    if all_present:
        assert len(seen) == len(items), f"{what}: {len(seen)} records for {len(items)} bursts"
    return seen


def _decode_all(st, items, what, slack=0):
    assert st.queue(items) == 0, st.L.vdl2gpu_last_error()
    total = sum(_rec_bytes(it) for it in items)
    head, recs, used = st.decode(HDR + max(total + slack, 256))
    _check_records(recs, items, what)
    assert head["n_records"] == len(items) and head["bytes_used"] == total == used
    return head


@pytest.fixture(scope="module")
def corpus():
    return k3_corpus.corpus()


def test_whole_corpus_in_one_launch(corpus):
    """~6000 bursts over 2048 channels in one launch (three grid-strides of K3): every record and every per-channel
    counter equal to the oracle's"""
    st = Stage()
    assert len(corpus) > 2 * k3_corpus.K3_GRID and len(corpus) <= st.n_slots
    before = st.counters()
    assert not before.any()
    head = _decode_all(st, corpus, "corpus", slack=4096)
    assert head["pool_overflows"] == 0 and head["out_overflows"] == 0
    assert np.array_equal(st.counters(), k3_corpus.burst_counters(corpus))
    st.close()


def test_slots_come_back_and_stale_words_are_never_read(corpus):
    """Round 1 fills every slot with bursts of the longest nbits whose bits past the burst are all ones; round 2 queues
    the corpus, whose bursts land in the same slots (the free list is a stack) on top of those stale words, and must
    still decode exactly; then the whole pool can be queued again."""
    st = Stage()
    base = [it for it in corpus if it["kind"] == "volume"][:st.n_slots]
    long_ = []
    for it in (base * (st.n_slots // len(base) + 1))[:st.n_slots]:
        n = MAX_BITS - MAX_BITS % 3
        bits = np.ones(n, np.uint8)
        bits[:it["nbits"]] = it["bits"]
        long_.append(dict(it, bits=bits, nbits=n))
    _decode_all(st, long_, "round 1 (long, ones)", slack=4096)
    assert st.queue(long_[:1]) == 0 and st.queue(long_[:1]) == EINVAL       # a queue is pending
    st.decode(1 << 16)
    _decode_all(st, corpus, "round 2 (corpus on stale slots)", slack=4096)
    assert st.queue(long_ + long_[:1]) == ETOOBIG        # one more than the pool
    _decode_all(st, long_, "round 3 (the whole pool again)", slack=4096)
    st.close()



def test_small_launches_and_the_grid_stride_edge(corpus):
    """an empty queue, one burst, exactly K3_GRID bursts and K3_GRID + 1 on one stage; refusals of the queue stub"""
    st = Stage()
    head, recs, used = st.decode(HDR + 4096)
    assert head == dict(bytes_used=0, n_records=0, pool_overflows=0, out_overflows=0) and recs == [] and used == 0
    assert not st.counters().any()
    bad = dict(corpus[0], channel=st.n_ch)
    assert st.queue([bad]) == EINVAL
    assert st.queue([dict(corpus[0], nbits=MAX_BITS + 1, bits=np.zeros(MAX_BITS + 1, np.uint8))]) == EINVAL
    done = []
    for n in (1, k3_corpus.K3_GRID, k3_corpus.K3_GRID + 1):
        items = corpus[len(done):len(done) + n]
        _decode_all(st, items, f"{n} bursts")
        done += items
    assert np.array_equal(st.counters(), k3_corpus.burst_counters(done))
    st.close()


def test_output_region_overflow(corpus):
    """a region one byte short of the records: at least one record is missing, out_overflows counts every missing one,
    every record present is whole and correct, none crosses the end (which ones drop depends on the order of the
    atomicAdds, so that is not asserted)"""
    st = Stage()
    items = corpus[:3000]
    assert st.queue(items) == 0
    total = sum(_rec_bytes(it) for it in items)
    head, recs, used = st.decode(HDR + total - 1)
    assert 0 < head["n_records"] < len(items) and len(recs) == head["n_records"]
    assert head["out_overflows"] == len(items) - head["n_records"]
    assert used <= total - 1
    _check_records(recs, items, "overflow", all_present=False)
    _decode_all(st, items, "after the overflow")                                  # the slots came back
    st.close()


def test_rs_stub_past_capacity():
    """the serial device decoder (vdl2gpu_launch_rs_verify) on 5-8 errors in full blocks and past capacity in shortened
    blocks (2 and 4 FEC octets): return value and corrected block equal to the oracle's, failures and miscorrections
    included"""
    import torch
    L = vd.load_library()
    rng = np.random.default_rng(0x5253)
    n = 3000
    blocks = np.zeros((n, 255), np.uint8); fec = np.zeros(n, np.int32); want_ret = np.zeros(n, np.int32); want = np.zeros_like(blocks)
    for i in range(n):
        nf = (6, 6, 4, 2)[i % 4]
        msg = np.zeros(249, np.uint8)
        k = 249 if nf == 6 else int(rng.integers(3, 68))
        msg[:k] = rng.integers(0, 256, k, dtype=np.uint8)
        b = po.rs_encode(msg)
        b[249 + nf:] = 0
        cols = list(range(k)) + list(range(249, 249 + nf))
        n_err = int(rng.integers(5, 9)) if nf == 6 else int(rng.integers(nf // 2 + 1, 9))
        for c in rng.choice(len(cols), size=min(n_err, len(cols)), replace=False):
            b[cols[int(c)]] ^= int(rng.integers(1, 256))
        blocks[i] = b; fec[i] = nf
        want_ret[i], want[i] = po.rs_verify(b, nf)
    d_b = torch.from_numpy(blocks).cuda(); d_f = torch.from_numpy(fec).cuda(); d_r = torch.zeros(n, dtype=torch.int32, device="cuda")
    assert L.vdl2gpu_launch_rs_verify(d_b.data_ptr(), d_f.data_ptr(), n, d_r.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert np.array_equal(d_r.cpu().numpy(), want_ret)
    assert np.array_equal(d_b.cpu().numpy(), want)
    for nf in (6, 4, 2):
        sel = fec == nf
        assert (want_ret[sel] < 0).any() and (want_ret[sel] >= 0).any(), f"{nf} FEC octets: failures and decodes expected"


@pytest.mark.parametrize("flags", [0, vd.FLAG_NO_GRAPH], ids=["graphs", "no_graph"])
def test_fuzz_stream_through_the_pipeline(flags):
    """cases.case_fuzz (random-length, cut and corrupted transmissions on two channels) through Vdl2Channels: frames, trace
    events and per-channel counters equal to the oracle's; this covers K2's packing of such bursts into slots"""
    c = cases.case_fuzz()
    o = util.run_oracle(c, trace=True)
    g = vd.Vdl2Channels(c["fs"], c["oversample"], util.fmt_code(c), c["centerfreq"], c["freqs"], max_ppm=c.get("max_ppm", 0.0),
                        max_chunk_bytes=max(c["chunk"], 1 << 16), flags=flags | vd.FLAG_TRACE)
    g.process_chunked(util.case_bytes(c), c["chunk"])
    frames = g.flush()
    st = g.stats()
    assert st["pool_overflows"] == 0 and st["out_overflows"] == 0
    util.assert_frames_equal(frames, o.frames(), f"fuzz stream [{flags}]")
    util.assert_events_equal(g.read_events(), o.events(), f"fuzz stream events [{flags}]")
    assert np.array_equal(g.channel_counters(), o.counters())
    assert st["bursts"] >= 12
    g.close()
