"""-m gpu: the K2 corpus (tests/k2_corpus.py) through the device's sync walk and burst decoder, launch by launch on the
corpus's schedule (launches of 1..2399 decimated samples, so that every event also lands in a walk tail, just after
a launch start, and in phase history carried over several short launches), against the oracle: sync and header events
bit for bit, frames with their metadata, per-channel counters.  Repeated with the trace off (the production path) and
under every walk form the library keeps."""
import ctypes as C
import os
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import api
from tests import k2_corpus as kc, util

pytestmark = pytest.mark.gpu


def _run_stage(name, flags, env=None):
    """(frames, counters, events) of one corpus stage through vdl2gpu_launch_sync_slice + vdl2gpu_launch_burst_fec"""
    import torch
    s = kc.stage(name)
    L = vd.load_library()
    dec = s["dec"]
    n_total, n_ch = dec.shape[:2]
    max_dec = max(kc.LAUNCHES)
    cfg, _keep = api.make_config(kc.DEC_RATE, 1, vd.FMT_U8, kc.CENTER, s["freqs"], max_ppm=s["max_ppm"], flags=flags)
    stride = L.vdl2gpu_stage_row_stride(n_ch)
    nbytes = L.vdl2gpu_stage_device_bytes(n_ch, max_dec, flags)
    mem = torch.zeros(nbytes + 256, dtype=torch.uint8, device="cuda")
    h = C.c_void_p()
    old = {k: os.environ.get(k) for k in (env or {})}
    try:
        for k, v in (env or {}).items():        # the walk form is chosen when the stage is created
            os.environ[k] = str(v)
        rc = L.vdl2gpu_stage_create(C.byref(cfg), max_dec, C.c_void_p((mem.data_ptr() + 255) & ~255), nbytes, C.byref(h))
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    assert rc == 0, L.vdl2gpu_last_error()
    padded = np.zeros((n_total, stride, 2), np.float32)
    padded[:, :n_ch] = dec
    d_dec = torch.from_numpy(padded).cuda()
    region = torch.zeros(2 << 20, dtype=torch.uint8, device="cuda")
    frames = []
    for a, n in kc.launch_bounds(n_total):
        assert L.vdl2gpu_launch_sync_slice(h, d_dec[a:a + n].data_ptr(), n, None) == 0
        assert L.vdl2gpu_launch_burst_fec(h, region.data_ptr(), region.numel(), None) == 0
        torch.cuda.synchronize()
        frames += api.parse_records(region.cpu().numpy().tobytes(), kc.DEC_RATE)
    cnt = np.zeros((n_ch, 9), np.uint64)
    assert L.vdl2gpu_stage_read_counters(h, cnt.ctypes.data) == 0
    events = []
    if flags & vd.FLAG_TRACE:
        cap = 1 << 18
        ev = (api._Event * cap)()
        k = L.vdl2gpu_stage_read_events(h, C.cast(ev, C.c_void_p), cap)
        assert 0 <= k < cap, "event buffer full"
        events = [dict(channel=ev[i].channel, kind=ev[i].kind, dec_index=ev[i].dec_index, i=list(ev[i].i),
                       f=np.array(list(ev[i].f), np.float32)) for i in range(k)]
    L.vdl2gpu_stage_destroy(h)
    return frames, cnt, events


def _same_frames(a, b):
    key = lambda f: f.key()
    return [util.frame_tuple(f) + (f.sync_dec_index, np.float32(f.frame_pwr).tobytes(), np.float32(f.ppm_error).tobytes(),
                                   np.float32(f.mag_nf).tobytes()) for f in sorted(a, key=key)] == \
           [util.frame_tuple(f) + (f.sync_dec_index, np.float32(f.frame_pwr).tobytes(), np.float32(f.ppm_error).tobytes(),
                                   np.float32(f.mag_nf).tobytes()) for f in sorted(b, key=key)]


@pytest.mark.parametrize("name", list(kc.STAGES))
def test_k2_corpus_on_the_device_matches_the_oracle(name):
    """trace on: events, frames, metadata and counters equal the oracle's; trace off: the same frames and counters"""
    o = kc.oracle(name)
    frames, cnt, events = _run_stage(name, vd.FLAG_TRACE)
    util.assert_events_equal(events, o.events(), f"K2 corpus events [{name}]")
    util.assert_frames_equal(frames, o.frames(), f"K2 corpus frames [{name}]")
    assert np.array_equal(cnt, o.counters()), f"{name}: counters differ"
    plain, cnt_plain, _ = _run_stage(name, 0)
    assert _same_frames(plain, frames) and np.array_equal(cnt_plain, cnt), f"{name}: trace off differs from trace on"


@pytest.mark.parametrize("env", [dict(VDL2GPU_K2_VARIANT=0), dict(VDL2GPU_K2_VARIANT=1), dict(VDL2GPU_K2_VARIANT=3),
                                 dict(VDL2GPU_K2_VARIANT=4), dict(VDL2GPU_K2_VARIANT=5), dict(VDL2GPU_K2A=0)],
                         ids=["k2_0", "k2_1", "k2_3", "k2_4", "k2_5", "k2a_0"])
@pytest.mark.parametrize("name", ["main", "ppm"])
def test_k2_corpus_under_every_walk_form(name, env):
    o = kc.oracle(name)
    frames, cnt, events = _run_stage(name, vd.FLAG_TRACE, env)
    util.assert_events_equal(events, o.events(), f"K2 corpus events [{name} {env}]")
    util.assert_frames_equal(frames, o.frames(), f"K2 corpus frames [{name} {env}]")
    assert np.array_equal(cnt, o.counters()), f"{name} {env}: counters differ"


def test_k2_corpus_ragged_spans_match_the_oracle_per_receiver():
    """k2_sync_slice_ragged: a ragged mixed-receivers context (48 one-channel receivers, cu8 at oversample 10 and cs16 at
    20) fed IQ in spans whose per-receiver counts put syncs, headers and burst ends at every tail position of the walk
    (k2_corpus.ragged_spans); each receiver's frames, counters and trace events equal the oracle's on its whole stream."""
    rxs = kc.ragged_fleet()
    oracles = kc.ragged_oracles()
    n_dec = [kc.ragged_n_dec(x) for x in rxs]
    spans = kc.ragged_spans(oracles, n_dec)
    g = vd.Vdl2MixedReceivers([(x["centre"], x["freqs"], x["os"], vd.FMT_S16 if x["fmt"] == "s16" else vd.FMT_U8) for x in rxs],
                              max_chunk_bytes=kc.RAGGED_W * 80, flags=vd.FLAG_TRACE, ragged=True)
    g.process_ragged([x["buf"] for x in rxs], spans)
    frames = g.flush()
    events = g.read_events(1 << 20)
    cnt, st, positions = g.channel_counters(), g.stats(), g.receiver_positions()
    g.close()
    assert st["pool_overflows"] == 0 and st["out_overflows"] == 0
    assert positions.tolist() == n_dec
    n_frames = 0
    for r, o in enumerate(oracles):
        mine = [f for f in frames if f.channel == r]
        for f in mine:
            f.channel = 0
        util.assert_frames_equal(mine, o.frames(), f"ragged receiver {r}")
        assert np.array_equal(cnt[r:r + 1], o.counters()), f"ragged receiver {r}: counters"
        util.assert_events_equal([dict(e, channel=0) for e in events if e["channel"] == r], o.events(), f"ragged receiver {r}")
        n_frames += len(mine)
    assert n_frames > 400
