"""-m gpu: the default K2 walk, which slices a burst's data symbols after its block loop (vdl2_defer), on launch schedules
that reach that path's own cases: one launch holding a whole corpus stage (more bursts per channel than the one-burst
queue holds) and runs of one-sample launches inside bursts.  Events, frames with their metadata and counters equal the
oracle's, whatever the schedule.  The ragged walk runs a fleet whose spans are planned around burst ends
(k2_corpus.defer_spans), with and without restarts at span boundaries."""
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from tests import k2_corpus as kc, util
from tests import test_gpu_k2_corpus as g
from tests import test_gpu_restart_receivers as rr

pytestmark = pytest.mark.gpu

_bounds = kc.launch_bounds


@pytest.mark.parametrize("name,schedule", [("main", "one_launch"), ("long", "one_launch"), ("main", "one_sample_launches")])
def test_deferred_symbols_on_the_device_match_the_oracle(name, schedule, monkeypatch):
    launches = (kc.stage(name)["dec"].shape[0],) if schedule == "one_launch" else (1,) * 30 + (37,)
    monkeypatch.setattr(kc, "LAUNCHES", launches)
    monkeypatch.setattr(kc, "launch_bounds", lambda n_dec: _bounds(n_dec, launches))
    o = kc.oracle(name)
    frames, cnt, events = g._run_stage(name, vd.FLAG_TRACE)
    util.assert_events_equal(events, o.events(), f"K2 corpus events [{name} {schedule}]")
    util.assert_frames_equal(frames, o.frames(), f"K2 corpus frames [{name} {schedule}]")
    assert np.array_equal(cnt, o.counters()), f"{name} {schedule}: counters differ"



def _defer_fleet_plan():
    oracles = kc.defer_oracles()
    rxs = kc.defer_fleet()
    n_dec = [kc.ragged_n_dec(x) for x in rxs]
    return rxs, oracles, kc.defer_spans(oracles, n_dec), n_dec


@pytest.mark.parametrize("flags", [vd.FLAG_TRACE, 0], ids=["trace", "plain"])
def test_deferral_plan_ragged_spans_match_the_oracle_per_receiver(flags):
    """k2_sync_slice_ragged on k2_corpus.defer_spans (64 one-channel receivers, spans that end on, one before and one after a
    burst's last symbol, empty and one-sample spans inside a burst, spans holding two and three burst ends): each
    receiver's frames, counters and, with the trace on, events equal its oracle's on its whole stream"""
    rxs, oracles, spans, n_dec = _defer_fleet_plan()
    res, pos = rr._run(rxs, [x["buf"] for x in rxs], spans, {}, flags)
    assert res["stats"]["pool_overflows"] == 0 and res["stats"]["out_overflows"] == 0
    assert res["positions"].tolist() == n_dec == pos
    n_frames = 0
    for r, o in enumerate(oracles):
        mine = [f for f in res["frames"] if f.channel == r]
        for f in mine:
            f.channel = 0
        util.assert_frames_equal(mine, o.frames(), f"deferral fleet receiver {r}")
        assert np.array_equal(res["cnt"][r:r + 1], o.counters()), f"deferral fleet receiver {r}: counters"
        if res["events"] is not None:
            util.assert_events_equal([dict(e, channel=0) for e in res["events"] if e["channel"] == r], o.events(),
                                     f"deferral fleet receiver {r}")
        n_frames += len(mine)
    assert n_frames == sum(len(o.frames()) for o in oracles) > 1000


def test_deferral_plan_restarts_at_a_span_boundary_inside_and_just_after_a_burst():
    """the deferral fleet with two restarts (vdl2gpu_restart_receiver) at span boundaries: one receiver while its burst is
    open (header decoded, last symbol still to come), another whose burst ended on the previous span's last sample.  Both
    decode what the segmented oracles decode; every other receiver what it decodes without a restart."""
    rxs, oracles, spans, n_dec = _defer_fleet_plan()
    cum = np.cumsum([[0] * len(rxs)] + spans, axis=0)            # cum[k][r]: receiver r's samples before span k
    picks = {}
    for r, o in enumerate(oracles):
        ev = sorted(o.events(), key=lambda e: e["dec_index"])
        ends = {int(e["dec_index"]) for e in ev if e["kind"] == 3}
        opened = [(int(h["dec_index"]), min(x for x in ends if x > h["dec_index"])) for h in ev
                  if h["kind"] == 2 and h["i"][3] == 0 and any(x > h["dec_index"] for x in ends)]
        for k in range(2, len(spans) - 2):
            b = int(cum[k][r])
            if "open" not in picks and r % 2 == 0 and spans[k][r] > 0 and any(h < b <= e for h, e in opened):
                picks["open"] = (r, k, b)
            if "ended" not in picks and r % 2 == 1 and spans[k][r] > 0 and b - 1 in ends:
                picks["ended"] = (r, k, b)
    assert picks.keys() == {"open", "ended"}, picks
    restarts, segs = {}, {}
    for r, k, b in picks.values():
        restarts.setdefault(k, []).append((r, None, None))
        x = rxs[r]
        segs[r] = rr._segments(x, x["buf"][:n_dec[r] * x["os"] * (4 if x["fmt"] == "s16" else 2)], [b],
                               [(x["centre"], x["freqs"])] * 2)
    res, pos = rr._run(rxs, [x["buf"] for x in rxs], spans, restarts, vd.FLAG_TRACE)
    assert res["stats"]["pool_overflows"] == 0 and res["stats"]["out_overflows"] == 0
    last = [c for c in spans if max(c) > 0][-1]
    for r, o in enumerate(oracles):
        mine = [f for f in res["frames"] if f.channel == r]
        for f in mine:
            f.channel = 0
        cnt = res["cnt"][r:r + 1]
        ev = [dict(e, channel=0) for e in res["events"] if e["channel"] == r]
        what = f"deferral fleet receiver {r}"
        if r in segs:
            rr._check_restarted(mine, cnt, res["dec"][:, r:r + 1], ev, *segs[r], last[r], what + " restarted")
        else:
            util.assert_frames_equal(mine, o.frames(), what)
            assert np.array_equal(cnt, o.counters()), f"{what}: counters"
            util.assert_events_equal(ev, o.events(), what)
