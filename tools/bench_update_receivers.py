#!/usr/bin/env python
"""tools/bench_update_receivers.py — receivers joining and leaving a ragged context (Vdl2MixedReceivers.update_receivers).
The fleet of bench_ragged_receivers.py: R receivers x C channels (default 2048 x 8), the first half cu8 at oversample 10,
the second half cs16 at oversample 20, full spans of 13107 decimated samples through submit_ragged_device; receivers that
join are of the second kind and are appended.  One process reports, with the GPU name, SM clock and power limit read in
the same run:
  - pipelined ms per span (graphs) on the fleet, alternating: R receivers, R + 1 after an update adds one, R again after
    an update removes it, ... (--repeats rounds);
  - the wall time of vdl2gpu_update_receivers for adding 1 receiver, adding 64 and removing 1, each followed by the wall
    time of the first span after it (graph capture) and of a steady span, both from submit to flush.

    python tools/bench_update_receivers.py [--receivers 2048] [--channels 8] [--spans 16] > update.json
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import bench
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth

N_DISTINCT = 2
DEC_RATE = 105000
KINDS = [(10, vd.FMT_U8, 2), (20, vd.FMT_S16, 4)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--receivers", type=int, default=2048, help="even: half of each rate")
    ap.add_argument("--channels", type=int, default=8)
    ap.add_argument("--n-dec", type=int, default=13107)
    ap.add_argument("--spans", type=int, default=16, help="timed spans per measurement")
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_update_receivers.py needs a CUDA device: the demodulator path has no CPU fallback")
    R, C, D, X = a.receivers, a.channels, a.n_dec, 64
    H = R // 2
    seconds = N_DISTINCT * D / DEC_RATE + 0.05
    cls = []
    for k, (os_, fmt, bpp) in enumerate(KINDS):
        iq, offs, _ = synth.traffic_stream(DEC_RATE * os_, seconds, 32 if os_ == 10 else 64, 4.0, 22.0, -20.0, 0x55504800 + k,
                                           "s16" if fmt else "u8")
        w = os_ * bpp
        host = np.ascontiguousarray(iq).view(np.uint8).reshape(-1)
        L = host.size // w
        cls.append(dict(os=os_, fmt=fmt, w=w, offs=offs, L=L, dev=torch.from_numpy(host[:L * w].reshape(L, w)).cuda()))
    kind = [0] * H + [1] * (R - H) + [1] * X                     # receivers R.. join (second kind)
    ar = torch.arange(N_DISTINCT * D, device="cuda", dtype=torch.int64)
    spans = []                                                   # every receiver's span s back to back (receiver 0 first)
    for s in range(N_DISTINCT):
        parts = []
        for r in range(R + X):
            c = cls[kind[r]]
            parts.append(c["dev"][(ar[s * D:(s + 1) * D] + 7919 * r) % c["L"]].reshape(-1))
        spans.append(torch.cat(parts).contiguous())
    del parts
    torch.cuda.synchronize()
    rx = []
    for r in range(R + X):
        centre = bench.CENTER + 1000 * (r - H)
        offs = cls[kind[r]]["offs"]
        rx.append((centre, [centre + int(offs[(r * C + i) % len(offs)]) for i in range(C)], KINDS[kind[r]][0], KINDS[kind[r]][1]))
    stream = torch.cuda.current_stream()
    g = vd.Vdl2MixedReceivers(rx[:R], max_chunk_bytes=D * 80, ragged=True)
    k_span = [0]

    def feed():
        n = np.full(g.n_receivers, D, np.uint32)                 # a prefix of the packed span: receivers 0 .. n - 1
        g.submit_ragged_device(spans[k_span[0] % N_DISTINCT].data_ptr(), n, stream.cuda_stream)
        k_span[0] += 1

    def pipelined():
        for _ in range(a.warmup):
            feed()
        g.flush_count()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(a.spans):
            feed()
            g.poll_count()
        g.flush_count()
        g.stream_wait(stream.cuda_stream)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.spans

    def one_span():
        t0 = time.perf_counter()
        feed()
        g.flush_count()
        return (time.perf_counter() - t0) * 1e3

    def update(to):
        """to: the receiver ids of the new list (a prefix of rx); returns ms of the call, of the first span after it, of a
        steady span"""
        old = {r: k for k, r in enumerate(range(g.n_receivers))}
        g.flush_count()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g.update_receivers([rx[r] for r in to], [old.get(r, -1) for r in to])
        t1 = time.perf_counter()
        first = one_span()
        return dict(update_ms=(t1 - t0) * 1e3, first_span_ms=first, steady_span_ms=one_span())

    sampler = bench.ClockSampler(torch.cuda.current_device())
    sampler.start()
    t0 = time.time()
    ms = dict(before=[], after_add_1=[])
    for _ in range(a.repeats):
        ms["before"].append(pipelined())
        update(list(range(R + 1)))
        ms["after_add_1"].append(pipelined())
        update(list(range(R)))
    walls = dict(add_1=update(list(range(R + 1))), remove_1=update(list(range(R))), add_64=update(list(range(R + X))))
    t1 = time.time()
    st = g.stats()
    g.close()
    res = dict(gpu=torch.cuda.get_device_name(), receivers=R, channels_per_receiver=C, full_span=D, timed_spans=a.spans,
               pipelined_ms_per_span=ms, update_wall=walls, overflows=st["pool_overflows"] + st["out_overflows"],
               clocks=sampler.stop(t0, t1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
