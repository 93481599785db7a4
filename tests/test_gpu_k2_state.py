"""-m gpu: the state every K2 launch leaves on the device, against the host reference of test_k2_state.py.

A stage (vdl2gpu_stage_create) lives in one block of device memory that the test owns, laid out as the host helper
restates it (pinned on the CPU against vdl2gpu_stage_device_bytes).  So the test reads the K2 plane, the ring, the phase
plane, the pool, the free list, the ready list and the queue counters straight from that memory.  It checks them right
after create, then after every vdl2gpu_launch_sync_slice, before vdl2gpu_launch_burst_fec, against the plain per-sample
walk on the host:
- every K2_* field bit for bit, K2_SLOT only by sign (slot numbers follow the order of the device's atomics);
- the ring bit for bit;
- the phase plane's 160 history rows and the launch's own rows (vdl2_launch_copy_hist, launches below 160 included);
- the ready bursts as a multiset of header and words, and an open burst's words written so far, through the device's
  slot index;
- the pool counters, and after K3 a free list that holds every slot no open burst holds.
An error in a field that only picks a code path (pure_run), or that the walk overwrites before it next reads it (pherr0;
dphi and syndrome while searching), changes no output; here it fails the launch that makes it.  Run for every walk form
the library keeps, with the trace on and off, on schedules from one launch per stage to one-sample launches.  A second set of runs drains the burst pool before every launch, so that
headers inside the deferred walk meet an empty pool."""
import ctypes as C
import os
import numpy as np
import pytest
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import api
from tests import k2_corpus as kc
from tests import test_gpu_k2_corpus as gk
from tests import test_k2_state as ks

pytestmark = pytest.mark.gpu

K2 = ks.K2
ONE_SAMPLE = (1,) * 30 + (37,)
SHORT = (9, 10, 11, 12, 13, 19, 20, 21, 24, 25)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return ks.build(tmp_path_factory.mktemp("k2state"))


class DeviceStage:
    """a stage in device memory the test owns, and views of its planes"""

    def __init__(self, L, dec, freqs, max_ppm, flags, max_dec, env=None):
        import torch
        self.V = V = vd.load_library()
        self.n_dec, self.n_ch = dec.shape[:2]
        self.max_dec = max_dec
        self.off, self.total, self.n_slots = ks.stage_layout(L, self.n_ch, max_dec, flags)
        self.n_chp = V.vdl2gpu_stage_row_stride(self.n_ch)
        assert self.total == V.vdl2gpu_stage_device_bytes(self.n_ch, max_dec, flags)
        self.slot_words, self.H = L.slot_words, L.slot_header_words
        cfg, self._keep = api.make_config(kc.DEC_RATE, 1, vd.FMT_U8, kc.CENTER, freqs, max_ppm=max_ppm, flags=flags)
        self.mem = torch.zeros(self.total + 256, dtype=torch.uint8, device="cuda")
        base = (self.mem.data_ptr() + 255) & ~255
        self.buf = self.mem[base - self.mem.data_ptr():][:self.total]
        self.h = C.c_void_p()
        old = {k: os.environ.get(k) for k in (env or {})}
        try:
            for k, v in (env or {}).items():          # the walk form is chosen when the stage is created
                os.environ[k] = str(v)
            rc = V.vdl2gpu_stage_create(C.byref(cfg), max_dec, C.c_void_p(base), self.total, C.byref(self.h))
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        assert rc == 0, V.vdl2gpu_last_error()
        padded = np.zeros((self.n_dec, self.n_chp, 2), np.float32)
        padded[:, :self.n_ch] = dec
        self.d_dec = torch.from_numpy(padded).cuda()
        self.region = torch.zeros(4 << 20, dtype=torch.uint8, device="cuda")

    def _part(self, name, nbytes):
        import torch
        o = self.off[name]
        return self.buf[o:o + nbytes].view(torch.int32)

    def plane(self, name, rows):
        """[rows][n_ch] of a plane with the stage's row stride, as uint32"""
        return self._part(name, rows * self.n_chp * 4).reshape(rows, self.n_chp)[:, :self.n_ch].cpu().numpy().view(np.uint32)

    def ctl(self):
        return dict(zip(ks.CTL, (int(x) for x in self._part("ctl", 4 * len(ks.CTL)).cpu().numpy().view(np.uint32))))

    def free_list(self, n):
        return self._part("free_list", 4 * n).cpu().numpy() if n > 0 else np.zeros(0, np.int32)

    def ready_slots(self, n):
        return self._part("ready", 4 * n).cpu().numpy().view(np.uint32) if n else np.zeros(0, np.uint32)

    def slots(self, idx):
        """[len(idx)][slot words] of pool slots idx"""
        import torch
        pool = self._part("pool", self.n_slots * self.slot_words * 4).reshape(self.n_slots, self.slot_words)
        if len(idx) == 0:
            return np.zeros((0, self.slot_words), np.uint32)
        return pool[torch.as_tensor(np.asarray(idx, np.int64), device="cuda")].cpu().numpy().view(np.uint32)

    def sync_slice(self, a, n):
        import torch
        assert self.V.vdl2gpu_launch_sync_slice(self.h, self.d_dec[a:a + n].data_ptr(), n, None) == 0
        torch.cuda.synchronize()

    def burst_fec(self):
        """K3; -> (frames, [(channel, burst_seq)] of every record)"""
        import torch
        assert self.V.vdl2gpu_launch_burst_fec(self.h, self.region.data_ptr(), self.region.numel(), None) == 0
        torch.cuda.synchronize()
        raw = self.region.cpu().numpy().tobytes()
        hdr = np.frombuffer(raw[:32], np.uint32)
        keys, at = [], 32
        for _ in range(int(hdr[1])):
            rec = np.frombuffer(raw[at:at + 12], np.uint32)
            keys.append((int(rec[1]), int(rec[2])))
            at += int(rec[0])
        frames = []
        cb = api._FRAME_CB(lambda fp, _u: frames.append(api.frame_from_c(fp.contents)))
        buf = np.frombuffer(raw, np.uint8)
        rc = self.V.vdl2gpu_parse_records(buf.ctypes.data, buf.size, kc.DEC_RATE, cb, None)
        assert rc >= 0 or (rc == -6 and hdr[2] > 0), rc          # VDL2GPU_EOVERFLOW: the pool ran out in this launch
        return frames, keys

    def queue_dummies(self, channel, n):
        bursts = (api._Burst * max(n, 1))()
        for b in bursts:
            b.channel = channel
        assert self.V.vdl2gpu_stage_queue_bursts(self.h, bursts, n) == 0

    def close(self):
        self.V.vdl2gpu_stage_destroy(self.h)


def check_fresh(dev, host):
    """right after create: every channel as vdl2_chan_init leaves it, zero ring and phase plane, a full free list"""
    want = host.read()
    assert np.array_equal(dev.plane("k2", len(K2)), want["k2"]), "K2 plane after create"
    assert not dev.plane("ring", kc.RING).any() and not dev.plane("phase", kc.RING + dev.max_dec).any()
    c = dev.ctl()
    assert c["free_top"] == dev.n_slots and c["n_ready"] == 0 and c["pool_overflows"] == 0
    assert np.array_equal(dev.free_list(dev.n_slots), np.arange(dev.n_slots))


def check_launch(dev, host, a, n, what, full_pool=True, dummy_channel=None):
    """the device after one launch against the host's per-sample walk; -> the device's K2_SLOT of every channel"""
    want = host.read()
    k2 = dev.plane("k2", len(K2))
    keep = np.ones(len(K2), bool)
    keep[K2["SLOT"]] = False
    bad = np.argwhere(k2[keep] != want["k2"][keep])
    if bad.size:
        f, ch = bad[0]
        name = [k for k, v in K2.items() if v == np.flatnonzero(keep)[f]][0]
        raise AssertionError(f"{what}: K2_{name} of channel {ch} after the launch at {a}+{n}: "
                             f"{k2[np.flatnonzero(keep)[f], ch]:#x}, host {want['k2'][np.flatnonzero(keep)[f], ch]:#x}")
    dslot, hslot = k2[K2["SLOT"]].view(np.int32), want["k2"][K2["SLOT"]].view(np.int32)
    if full_pool:
        assert np.array_equal(dslot >= 0, hslot >= 0), f"{what}: K2_SLOT sign at {a}+{n}"
    else:                                   # a channel may have found the pool empty
        assert np.all(hslot[dslot >= 0] >= 0), f"{what}: a slot the host did not take at {a}+{n}"
    ring = dev.plane("ring", kc.RING)
    assert ring.tobytes() == want["ring"].view(np.uint32).tobytes(), \
        f"{what}: ring of channel {np.argwhere(ring != want['ring'].view(np.uint32))[0][1]} at {a}+{n}"
    ph = dev.plane("phase", kc.RING + n)
    assert ph[:kc.RING].tobytes() == want["hist"].view(np.uint32).tobytes(), f"{what}: phase history rows at {a}+{n}"
    assert ph[kc.RING:].tobytes() == host.phase_rows(kc.RING + a, n).view(np.uint32).tobytes(), f"{what}: phase rows at {a}+{n}"
    # open bursts: the words written so far, through each side's own slot index
    both = np.flatnonzero((dslot >= 0) & (hslot >= 0))
    got = dev.slots(dslot[both])
    H = dev.H
    for i, ch in enumerate(both):
        w = ks.slot_words_used(k2[K2["NBITS"], ch], False)
        assert np.array_equal(got[i, H:H + w], host.slot(hslot[ch])[H:H + w]), f"{what}: open burst words, channel {ch} at {a}+{n}"
    c, hc = dev.ctl(), want["ctl"]
    ready = dev.slots(dev.ready_slots(c["n_ready"]))
    mine = sorted(ks.ready_key(host.L, s) for s in ready if dummy_channel is None or s[0] != dummy_channel)
    theirs = sorted(ks.ready_key(host.L, s) for s in host.ready())
    if full_pool:
        assert c["n_ready"] == hc["n_ready"] and c["free_top"] == hc["free_top"], f"{what}: {c} != host {hc}"
        assert c["pool_overflows"] == hc["pool_overflows"] == 0, what
        assert mine == theirs, f"{what}: ready bursts at {a}+{n}"
    else:
        left = list(theirs)
        for k in mine:
            assert k in left, f"{what}: a ready burst the host does not have at {a}+{n}"
            left.remove(k)
    return dslot


def check_no_leak(dev, dslot, what):
    """after K3: the free list holds every slot no open burst holds"""
    c = dev.ctl()
    held = dslot[dslot >= 0]
    assert c["n_ready"] == 0 and c["free_top"] + held.size == dev.n_slots, f"{what}: {c}, {held.size} slots held"
    assert np.array_equal(np.sort(np.concatenate([dev.free_list(c["free_top"]), held])), np.arange(dev.n_slots)), \
        f"{what}: free list"


def _stage_input(name, n_ch=None, silent=False):
    s = kc.stage(name)
    dec, freqs = s["dec"], list(s["freqs"])
    if n_ch is not None:
        dec, freqs = dec[:, :n_ch], freqs[:n_ch]
    if silent:                                   # one channel of digital silence after the corpus channels
        dec = np.concatenate([dec, np.zeros((dec.shape[0], 1, 2), np.float32)], axis=1)
        freqs = freqs + [kc.CENTER]
    return np.ascontiguousarray(dec), freqs, s["max_ppm"]


def run_state(lib, name, launches, flags, env=None, n_ch=None):
    dec, freqs, max_ppm = _stage_input(name, n_ch)
    bounds = kc.launch_bounds(dec.shape[0], launches)
    max_dec = max(n for _, n in bounds)
    dev = DeviceStage(lib, dec, freqs, max_ppm, flags, max_dec, env)
    host = ks.HostStage(lib, dec, freqs, max_ppm, dev.n_slots, ks.PER_SAMPLE, trace=bool(flags & vd.FLAG_TRACE))
    what = f"{name} {env or 'default'} flags={flags}"
    n_frames = 0
    try:
        check_fresh(dev, host)
        for a, n in bounds:
            dev.sync_slice(a, n)
            host.step(n)
            dslot = check_launch(dev, host, a, n, what)
            frames, _ = dev.burst_fec()
            n_frames += len(frames)
            check_no_leak(dev, dslot, what)
    finally:
        host.close()
        dev.close()
    return n_frames


FORMS = [dict(VDL2GPU_K2_VARIANT=v) for v in (0, 1, 2, 3, 4, 258, 261)] + [dict(VDL2GPU_K2A=0)]


@pytest.mark.parametrize("trace", [vd.FLAG_TRACE, 0], ids=["trace", "plain"])
@pytest.mark.parametrize("name", list(kc.STAGES))
def test_default_walk_leaves_the_host_state_after_every_launch(lib, name, trace):
    assert run_state(lib, name, kc.LAUNCHES, trace) > 0


@pytest.mark.parametrize("env", FORMS, ids=lambda e: "_".join(f"{k[8:].lower()}{v}" for k, v in e.items()))
def test_every_walk_form_leaves_the_host_state_after_every_launch(lib, env):
    assert run_state(lib, "main", kc.LAUNCHES, vd.FLAG_TRACE, env) > 0


@pytest.mark.parametrize("trace", [vd.FLAG_TRACE, 0], ids=["trace", "plain"])
@pytest.mark.parametrize("schedule", ["one_launch", "one_sample", "short"])
def test_default_walk_state_on_every_schedule(lib, schedule, trace):
    n_ch = 128 if schedule == "one_sample" else None
    launches = {"one_launch": (kc.stage("main")["dec"].shape[0],), "one_sample": ONE_SAMPLE, "short": SHORT}[schedule]
    run_state(lib, "main", launches, trace, n_ch=n_ch)


@pytest.mark.parametrize("left", [0, 1, 8])
def test_headers_meet_an_empty_pool_in_the_deferred_walk(lib, left):
    """Before every launch the free list is drained down to `left` slots by dummy bursts (nbits = 0) queued on a silent
    channel, so that headers meet an empty pool inside the walk; which channels get a slot then depends on timing.
    What does not: the state (against a host run with a full pool, slots aside), every record equal to the oracle's
    burst with the same (channel, burst_seq), the bursts without a record equal to pool_overflows, no slot leaked."""
    dec, freqs, max_ppm = _stage_input("main", silent=True)
    silent = dec.shape[1] - 1
    bounds = kc.launch_bounds(dec.shape[0])
    max_dec = max(n for _, n in bounds)
    dev = DeviceStage(lib, dec, freqs, max_ppm, vd.FLAG_TRACE, max_dec)
    host = ks.HostStage(lib, dec, freqs, max_ppm, dev.n_slots, ks.PER_SAMPLE)
    what = f"empty pool, {left} left"
    frames, records = [], []
    try:
        check_fresh(dev, host)
        for a, n in bounds:
            dev.queue_dummies(silent, dev.ctl()["free_top"] - left)
            dev.sync_slice(a, n)
            host.step(n)
            dslot = check_launch(dev, host, a, n, what, full_pool=False, dummy_channel=silent)
            f, keys = dev.burst_fec()
            frames += [x for x in f if x.channel != silent]
            records += [k for k in keys if k[0] != silent]
            check_no_leak(dev, dslot, what)
        overflows = dev.ctl()["pool_overflows"]
    finally:
        host.close()
        dev.close()
    o = kc.oracle("main")
    assert len(set(records)) == len(records)
    want = {}
    for x in o.frames():
        want.setdefault((x.channel, x.burst_seq), []).append(x)
    got = {}
    for x in frames:
        got.setdefault((x.channel, x.burst_seq), []).append(x)
    assert set(got) <= set(records)
    for k in records:
        assert gk._same_frames(got.get(k, []), want.get(k, [])), f"{what}: burst {k} differs from the oracle's"
    # every header that takes a slot (status 0) ends as a record, an overflow, or a burst still open at the end
    headers = sum(1 for e in o.events() if e["kind"] == 2 and e["i"][3] == 0)
    open_at_end = int(np.sum(dslot >= 0))
    assert overflows > 0, f"{what}: no header met the empty pool"
    assert len(records) + overflows + open_at_end == headers, (len(records), overflows, open_at_end, headers)
    assert (len(records) > 0) == (left > 0)
