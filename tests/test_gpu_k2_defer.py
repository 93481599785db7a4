"""-m gpu: the default K2 walk, which slices a burst's data symbols after its block loop (vdl2_defer), on launch schedules
that reach that path's own cases: one launch holding a whole corpus stage (more bursts per channel than the one-burst
queue holds) and runs of one-sample launches inside bursts.  Events, frames with their metadata and counters equal the
oracle's, whatever the schedule."""
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from tests import k2_corpus as kc, util
from tests import test_gpu_k2_corpus as g

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

