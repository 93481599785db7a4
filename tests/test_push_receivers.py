"""CPU: pushed input on a ragged mixed-receivers context (vdl2gpu_push, vdl2gpu_submit_pushed) without a GPU - the ring
arithmetic of vdl2_core.cuh compiled for the host (tests/hostsim/push_rings.cpp, TEST-ONLY): ring layout and alignment,
writes and reads across the wrap, free room with spans in flight and the no-deadlock guarantee after a drain, the drain
loop of submit_pushed, the timestamp anchor - and the refusals that need no device."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
import dumpvdl2_b200 as vd

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "dumpvdl2_b200", "csrc")
EINVAL = -1
MIX = [(10, 0), (20, 1), (13, 0), (20, 0), (10, 1)]          # (oversample, format): every rate/format kind, odd groups at 13


@pytest.fixture(scope="module")
def lay(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("push_rings") / "libpush.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I", CSRC, "-o", so, os.path.join(HERE, "hostsim", "push_rings.cpp")])
    L = C.CDLL(so)
    L.push_ring_layout.restype = C.c_uint64
    L.push_ring_layout.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    L.push_room.restype = C.c_uint64
    L.push_room.argtypes = [C.c_uint64] * 3
    L.push_segments.argtypes = [C.c_uint64] * 3 + [C.c_void_p]
    L.push_take.restype = C.c_uint32
    L.push_take.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32]
    L.push_realign.restype = C.c_uint64
    L.push_realign.argtypes = [C.c_uint64, C.c_uint32]
    L.push_span_table.argtypes = [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 5
    L.push_sync_end.restype = C.c_uint64
    L.push_sync_end.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32]
    L.push_back_seconds.restype = C.c_double
    L.push_back_seconds.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32]
    return L


def _layout(lay, mix, max_chunk, max_span):
    os_ = np.array([m[0] for m in mix], np.uint32)
    fmt = np.array([m[1] for m in mix], np.uint32)
    base, cap = np.zeros(len(mix), np.uint64), np.zeros(len(mix), np.uint64)
    total = lay.push_ring_layout(os_.ctypes.data, fmt.ctypes.data, len(mix), max_chunk, max_span, base.ctypes.data, cap.ctypes.data)
    return total, base, cap


def _gb(m):
    return m[0] * (4 if m[1] else 2)


def _segs(lay, cap, pos, n):
    out = np.zeros(4, np.uint64)
    lay.push_segments(cap, pos, n, out.ctypes.data)
    return [int(v) for v in out]


def test_ring_layout_and_alignment(lay):
    max_chunk = 1 << 20
    max_span = max_chunk // 80
    total, base, cap = _layout(lay, MIX, max_chunk, max_span)
    for r, m in enumerate(MIX):
        need = max_chunk + (max_span + 1) * _gb(m)
        assert need <= int(cap[r]) < need + 16 and int(cap[r]) % 16 == 0
        assert int(base[r]) % 16 == 0
        assert int(base[r]) == int(cap[:r].sum())
    assert total == int(cap.sum())
    # a cs16 receiver at oversample 20 at the default 1 MiB: about 2 MiB
    assert int(cap[1]) == (max_chunk + (max_span + 1) * 80 + 15) // 16 * 16 and abs(int(cap[1]) - (2 << 20)) < 1024


def test_ring_offsets_pass_4_gib(lay):
    n = 65535
    max_chunk = 1 << 20
    total, base, cap = _layout(lay, [(20, 1)] * n, max_chunk, max_chunk // 80)
    assert total > 1 << 37 and int(base[-1]) > 1 << 32 and total == int(base[-1]) + int(cap[-1])
    assert np.all(base.astype(object) % 16 == 0)
    assert np.all(np.diff(base.astype(np.int64)) == int(cap[0]))


@pytest.mark.parametrize("pos,n", [(0, 100), (900, 100), (950, 100), (1000, 24), (999, 1), (1023, 1024 - 0), (5 * 1024 + 7, 1017),
                                   (5 * 1024 + 7, 1), (1024 * 3 - 4, 4)])
def test_writes_and_reads_across_the_wrap(lay, pos, n):
    cap = 1024
    o0, l0, o1, l1 = _segs(lay, cap, pos, n)
    assert o0 == pos % cap and l0 + l1 == n and o1 == 0
    assert l0 == min(n, cap - pos % cap)
    assert (l1 > 0) == (pos % cap + n > cap)                  # an exact fit to the end is one piece
    ring = np.zeros(cap, np.int64)
    data = np.arange(pos, pos + n)
    ring[o0:o0 + l0] = data[:l0]
    ring[o1:o1 + l1] = data[l0:]
    assert all(ring[p % cap] == p for p in range(pos, pos + n))


class Model:
    """the library's per-receiver queue bookkeeping (vdl2gpu_push / vdl2gpu_submit_pushed / restart), stepped with the
    functions of vdl2_core.cuh; spans in flight complete when complete() is called"""

    def __init__(self, lay, mix, max_chunk, n_inflight=4):
        self.lay, self.mix = lay, mix
        self.max_chunk = max_chunk
        self.max_span = max_chunk // max(_gb(m) for m in mix)
        _, _, self.cap = _layout(lay, mix, max_chunk, self.max_span)
        n = len(mix)
        self.head, self.tail, self.freed = [0] * n, [0] * n, [0] * n
        self.fences = [[] for _ in range(n)]                   # [(span number, pos)]
        self.done = -1                                          # spans up to this one have completed K0
        self.spans = 0
        self.n_inflight = n_inflight
        self.pos = np.zeros(n, np.uint64)
        self.prev = np.zeros(n, np.uint32)
        self.tables = []

    def room(self, r):
        while self.fences[r] and self.fences[r][0][0] <= self.done:
            self.freed[r] = self.fences[r].pop(0)[1]
        return self.lay.push_room(int(self.cap[r]), self.head[r], self.freed[r])

    def push(self, r, n):
        """True if the push fits now; False if it would have to wait"""
        if self.room(r) < n:
            return False
        self.head[r] += n
        return True

    def submit_pushed(self, during=None):
        """during(): pushes made while the call runs, after each span; they wait for the next call"""
        k = 0
        limit = list(self.head)                                 # the heads read once, at entry
        while True:
            take = [self.lay.push_take(limit[r], self.tail[r], _gb(m), self.max_span) for r, m in enumerate(self.mix)]
            if max(take) == 0:
                return k
            if self.spans - self.done > self.n_inflight:        # acquire_slot: the oldest span has finished
                self.done = self.spans - self.n_inflight - 1
            tail = np.array(self.tail, np.uint64)
            out = np.zeros((len(self.mix), 4), np.uint64)
            n = np.array(take, np.uint32)
            os_ = np.array([m[0] for m in self.mix], np.uint32)
            fmt = np.array([m[1] for m in self.mix], np.uint32)
            self.lay.push_span_table(os_.ctypes.data, fmt.ctypes.data, self.cap.ctypes.data, len(self.mix), n.ctypes.data,
                                     tail.ctypes.data, self.pos.ctypes.data, self.prev.ctypes.data, out.ctypes.data)
            self.tables.append((list(self.tail), take, out))
            for r in range(len(self.mix)):
                if take[r]:
                    self.tail[r] = int(tail[r])
                    self.fences[r].append((self.spans, self.tail[r]))
            self.spans += 1
            k += 1
            if during:
                during()

    def complete(self):
        self.done = self.spans - 1

    def restart(self, r):
        if self.head[r] != self.tail[r]:
            self.head[r] = self.tail[r] = self.lay.push_realign(self.head[r], 4 if self.mix[r][1] else 2)
            self.fences[r].append((self.spans - 1, self.head[r]))     # (the dropped bytes' copies: done with the last span)


def test_drain_leaves_less_than_a_group_and_tables_follow_the_rings(lay):
    m = Model(lay, MIX, 3001 * 80)
    rng = np.random.default_rng(3)
    for step in range(300):
        r = int(rng.integers(len(MIX)))
        n = int(rng.choice([1, 3, 7, _gb(MIX[r]) - 1, int(rng.integers(1, m.max_chunk + 1)), m.max_chunk]))
        while not m.push(r, n):
            m.submit_pushed()
            if not m.push(r, n):
                m.complete()
        if rng.random() < 0.2:
            k = m.submit_pushed()
            for q, mm in enumerate(MIX):
                assert m.head[q] - m.tail[q] < _gb(mm)         # fewer than one whole group left per receiver
            assert k >= 0
    # every table: off = the tail's ring offset, n = the take, dec_base = the position; spans never wrap over a sample
    pos = [0] * len(MIX)
    for tails, take, out in m.tables:
        for r, mm in enumerate(MIX):
            assert int(out[r, 0]) == tails[r] % int(m.cap[r]) and int(out[r, 1]) == take[r] and int(out[r, 3]) == pos[r]
            assert int(out[r, 0]) % (4 if mm[1] else 2) == 0
            assert take[r] <= m.max_span
            pos[r] += take[r]
    assert m.pos.tolist() == pos


def test_a_far_behind_receiver_catches_up_over_several_spans(lay):
    m = Model(lay, MIX[:2], 100 * 80)
    for _ in range(5):
        assert m.push(0, m.max_chunk)                          # 5 x 8000 bytes of a 20-byte-group receiver: 2000 groups
        if m.room(0) < m.max_chunk:
            m.submit_pushed()
        m.complete()
    m.push(1, 80 * 3)
    k = m.submit_pushed()
    assert k >= 1
    takes = [t[1] for t in m.tables]
    assert all(t[0] <= m.max_span for t in takes) and sum(t[0] for t in takes) == 5 * m.max_chunk // 20
    assert sum(t[1] for t in takes) == 3


def test_room_with_spans_in_flight_and_no_deadlock_after_a_drain(lay):
    """after submit_pushed, a push of max_chunk_bytes fits once the spans in flight have completed, whatever was queued
    and in flight before - i.e. it waits for the GPU, never for the caller"""
    rng = np.random.default_rng(11)
    for trial in range(50):
        m = Model(lay, MIX, int(rng.integers(200, 4000)) * 80)
        for _ in range(40):
            r = int(rng.integers(len(MIX)))
            n = int(rng.integers(1, m.max_chunk + 1))
            if not m.push(r, n):
                m.submit_pushed()
                if not m.push(r, n):                            # only spans in flight hold the room: completing frees it
                    assert m.fences[r]
                    m.complete()
                    assert m.push(r, n)
            if rng.random() < 0.1:
                m.restart(r)
        m.submit_pushed()
        in_flight = [m.head[r] - m.freed[r] for r in range(len(MIX))]
        for r in range(len(MIX)):
            assert m.room(r) == int(m.cap[r]) - (m.head[r] - m.freed[r])
        m.complete()
        for r, mm in enumerate(MIX):
            assert m.room(r) >= m.max_chunk + m.max_span * _gb(mm), (trial, r, in_flight[r])


def test_restart_realigns_to_the_sample_size(lay):
    for pos, bpp, want in [(0, 2, 0), (1, 2, 2), (7, 4, 8), (8, 4, 8), (2 ** 33 + 3, 4, 2 ** 33 + 4), (13 * 2 + 1, 2, 28)]:
        assert lay.push_realign(pos, bpp) == want


def test_timestamp_anchor(lay):
    # a span took groups [1000, 1000 + 50) of a cs16 receiver at oversample 13 (52 bytes a group) from stream position 7004
    gb, bpp, rate = 52, 4, 105000 * 13
    end = lay.push_sync_end(1010, 1000, 7004, gb)
    assert end == 7004 + 11 * gb
    # the push that carried the group's last sample ended 26 samples later: 26 / rate seconds before its arrival
    assert lay.push_back_seconds(end, end + 26 * bpp, bpp, rate) == pytest.approx(26 / rate, rel=0, abs=1e-15)
    assert lay.push_back_seconds(end, end, bpp, rate) == 0.0
    # a push that ends inside a sample: only whole samples after the group's last sample count
    assert lay.push_back_seconds(end, end + 26 * bpp + 3, bpp, rate) == pytest.approx(26 / rate, abs=1e-15)
    assert lay.push_sync_end(2 ** 40, 2 ** 40, 2 ** 42, 80) == 2 ** 42 + 80


def test_refusals_without_a_context():
    L = vd.load_library()
    buf = np.zeros(16, np.uint8)
    assert L.vdl2gpu_push(None, 0, buf.ctypes.data, 16) == EINVAL
    assert "no context" in L.vdl2gpu_last_error().decode()
    assert L.vdl2gpu_push(None, 0, None, 0) == EINVAL
    assert L.vdl2gpu_submit_pushed(None) == EINVAL


def test_python_refuses_a_buffer_the_32_bit_length_cannot_hold():
    g = vd.Vdl2MixedReceivers.__new__(vd.Vdl2MixedReceivers)
    g.L, g.h = None, None
    big = np.empty((1 << 32) + 5, np.uint8)                  # never touched: no memory is committed
    with pytest.raises(vd.Vdl2GpuError, match="4294967301 bytes"):
        g.push(0, big)


def test_submit_pushed_stops_at_the_heads_it_read_at_entry(lay):
    """pushes that arrive while submit_pushed runs are not taken by that call: it returns after draining what was queued
    at entry, however fast the pushes keep coming, and the next call takes them"""
    m = Model(lay, MIX[:2], 100 * 80)
    m.push(0, 100 * 20 * 2 + 7)                                # two spans of receiver 0 and a split group
    late = []

    def during():                                             # another thread pushes a span's worth after every span
        m.complete()
        if m.push(0, 100 * 20):
            late.append(100 * 20)
    assert m.submit_pushed(during) == 2
    assert m.head[0] - m.tail[0] == 7 + sum(late) and len(late) == 2
    assert m.submit_pushed() == 2
    assert m.head[0] - m.tail[0] == 7
