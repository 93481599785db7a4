"""CPU: the K2 corpus (tests/k2_corpus.py) covers every position of the sync walk it is built to reach, and the host
build of the device functions (tests/hostsim), fed on the corpus's launch schedule so that every launch ends in its
own walk tail, equals the oracle on it under every walk form: sync and header events bit for bit, frames with their
metadata, counters."""
import numpy as np
import pytest
from tests import k2_corpus as kc, util
from tests.hostsim import pyhostsim as hs


def frame_rows_hostsim(recs):
    return sorted((r["channel"], r["burst_seq"], k, data, r["num_fec_corrections"], r["sync_dec_index"],
                   np.float32(r["frame_pwr"]).view(np.uint32), np.float32(r["mag_nf"]).view(np.uint32),
                   np.float32(r["ppm_error"]).view(np.uint32), crc == 0xF0B8 and len(data) >= 11)
                  for r in recs for k, (data, crc) in enumerate(r["frames"]))


def frame_rows_oracle(frames):
    return sorted((f.channel, f.burst_seq, f.idx, f.data, f.num_fec_corrections, f.sync_dec_index,
                   np.float32(f.frame_pwr).view(np.uint32), np.float32(f.mag_nf).view(np.uint32),
                   np.float32(f.ppm_error).view(np.uint32), f.fcs_ok) for f in frames)


@pytest.mark.parametrize("name", list(kc.STAGES))
def test_k2_corpus_covers_every_walk_position(name):
    """Every cell of the walk the corpus is built to reach is hit at least once in the oracle's run: the ring position
    and attempt offset of a searching block (where the 60 reads and the 12 writes wrap), nfcnt reaching 1000 on each
    of a block's four attempts and in the tail, every symbol phase at the entry of a locked block; sync, header and
    burst end at every block offset, every tail position and just after a launch start; syncs 150..320 samples after a
    reset, syncs whose preamble spans three launches, a metric just below the threshold; headers announcing no FEC or
    too long a transmission; zeros, subnormals, extreme magnitudes, clipping, long silence; max_ppm on both sides; the
    longest transmission."""
    cells = kc.coverage(name)
    for cell in sorted(cells, key=str):
        print(name, cell, cells[cell])
    empty = [c for c in kc.required_cells(name) if not cells.get(c)]
    assert not empty, f"{name}: cells not hit: {empty}"


@pytest.mark.parametrize("use_pre", [5, 4, 3, 2, 1, 0], ids=["ring_nomag", "ring_staged", "ring", "blocked_lut", "blocked", "per_sample"])
@pytest.mark.parametrize("name", list(kc.STAGES))
def test_k2_corpus_device_functions_on_host_match_oracle(name, use_pre):
    s, o = kc.stage(name), kc.oracle(name)
    recs, ev, cnt = hs.k2k3(s["dec"], s["freqs"], 2100000, max_ppm=s["max_ppm"], use_pre=use_pre,
                            launches=kc.LAUNCHES, event_cap=1 << 20)
    util.assert_events_equal(ev, o.events(), f"hostsim events [{name}]")
    assert frame_rows_hostsim(recs) == frame_rows_oracle(o.frames())
    oc = o.counters()
    assert np.array_equal(cnt[:, 0], oc[:, 0]) and np.array_equal(cnt[:, 1], oc[:, 1])
    assert len(recs) == sum(1 for e in o.events() if e["kind"] == 3)


@pytest.mark.parametrize("name", list(kc.STAGES))
def test_oracle_on_decimated_samples_matches_the_reference_demod(name):
    """Oracle.process_dec against the reference's own demod() fed the same decimated samples (its strict build, stored
    by tests/golden/make_golden.py): per channel the same frames with the same metadata, in the same order, on every
    channel where the reference's behaviour is defined."""
    import hashlib
    from oracle import pyoracle as po
    gold = util.load_golden("k2_corpus_reference")[name]
    s = kc.stage(name)
    assert hashlib.sha256(s["dec"].tobytes()).hexdigest() == gold["dec_sha256"], "corpus regenerated differently"
    per, ok = {}, set(kc.reference_defined(name))
    for f in sorted(kc.oracle(name).frames(), key=lambda f: f.key()):
        if f.channel in ok:
            per.setdefault(f.channel, []).append(po.frame_line(f))
    got = {str(c): [len(v), hashlib.sha256("\n".join(v).encode()).hexdigest()[:16]] for c, v in sorted(per.items())}
    assert sum(n for n, _ in got.values()) == gold["n_frames"] > 0
    assert got == gold["channels"]


def test_ragged_span_plan_puts_events_in_every_tail_position():
    """The span counts of the ragged fleet (k2_corpus.ragged_spans) hold every residue mod 12 and the counts 1..11 and
    149..161, and put syncs, headers and burst ends at every tail position; test_gpu_k2_corpus.py feeds them to the device."""
    oracles = kc.ragged_oracles()
    spans = kc.ragged_spans(oracles, [kc.ragged_n_dec(x) for x in kc.ragged_fleet()])
    assert max(max(s) for s in spans) <= kc.RAGGED_W
    cells, lengths = kc.ragged_tail_cells(spans, oracles)
    for cell in sorted(cells):
        print("ragged", cell, cells[cell])
    assert {n % kc.BLOCK for n in lengths} == set(range(kc.BLOCK))
    assert set(range(1, 12)) | set(range(149, 162)) <= lengths
    empty = [(k, t) for k in ("sync", "header", "end") for t in range(kc.BLOCK - 1) if not cells.get((k, t))]
    assert not empty, f"tail cells not hit: {empty}"
