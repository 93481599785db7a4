#!/usr/bin/env python
"""tools/bench_push_receivers.py — pushed input (Vdl2MixedReceivers.push / submit_pushed) against ragged spans from host
buffers (submit_ragged) on the same data.  The fleet of tools/bench_ragged_receivers.py: R receivers x C channels (default
2048 x 8 = 16384 channels), the first half cu8 at oversample 10, the second half cs16 at oversample 20; receiver r of a
class is that class's synthetic traffic stream started 7919 r decimated samples later.  Every span brings D decimated
samples of every receiver (default 4000: 320000 bytes of a cs16 receiver, the reference's RTL_BUFSIZE); the push feed
pushes each receiver's D x oversample samples as one buffer and then calls submit_pushed, the ragged feed packs the same
bytes into one buffer per span and calls submit_ragged.  The two feeds alternate.  One process reports, with the GPU name
and power limit read in the same run:
  - the period per span (wall time from the first submit to the end of flush, over the timed spans);
  - the time inside push calls per pushed byte, twice: in the pipelined run, where it includes the waits of back-pressure
    (a push waits for the spans still converting its receiver's ring), and with the GPU idle (after a flush, so no push
    waits), where it is the host's copy into pinned memory and the copy calls alone;
  - whether both feeds end with the same per-channel counters.

    python tools/bench_push_receivers.py [--receivers 2048] [--channels 8] [--n-dec 4000] [--spans 16] > push.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import bench
import dumpvdl2_b200 as vd
from dumpvdl2_b200 import synth

N_DISTINCT = 2                      # distinct spans per receiver, submitted round robin
DEC_RATE = 105000
KINDS = [(10, vd.FMT_U8, 2), (20, vd.FMT_S16, 4)]      # (oversample, format, bytes per complex sample)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--receivers", type=int, default=2048, help="even: half of each rate")
    ap.add_argument("--channels", type=int, default=8, help="channels per receiver")
    ap.add_argument("--n-dec", type=int, default=4000, help="decimated samples of every receiver per span")
    ap.add_argument("--spans", type=int, default=16, help="timed spans per measurement")
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=2, help="alternating repetitions of the two feeds")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_push_receivers.py needs a CUDA device: the demodulator path has no CPU fallback")
    R, C, D = a.receivers, a.channels, a.n_dec
    H = R // 2
    seconds = N_DISTINCT * D / DEC_RATE + 0.05
    cls = []
    for k, (os_, fmt, bpp) in enumerate(KINDS):
        iq, offs, _ = synth.traffic_stream(DEC_RATE * os_, seconds, 32 if os_ == 10 else 64, 4.0, 22.0, -20.0, 0x52414700 + k,
                                           "s16" if fmt else "u8")
        w = os_ * bpp
        host = np.ascontiguousarray(iq).view(np.uint8).reshape(-1)
        L = host.size // w
        groups = host[:L * w].reshape(L, w)
        ar = np.arange(N_DISTINCT * D)
        blk = np.empty((N_DISTINCT, H, D * w), np.uint8)            # [span, receiver of the class, bytes]
        for j in range(H):
            g = groups[(ar + 7919 * j) % L].reshape(N_DISTINCT, D * w)
            blk[:, j] = g
        cls.append(dict(os=os_, fmt=fmt, w=w, offs=offs, blk=blk))
    rx = [(bench.CENTER + 1000 * (r - H), [bench.CENTER + 1000 * (r - H) + int(cls[r // H]["offs"][(r * C + i) % len(cls[r // H]["offs"])])
                                           for i in range(C)], KINDS[r // H][0], KINDS[r // H][1]) for r in range(R)]
    bufs = [[cls[r // H]["blk"][s, r % H] for r in range(R)] for s in range(N_DISTINCT)]
    packed = [np.concatenate(b) for b in bufs]
    counts = np.full(R, D, np.uint32)
    max_bytes = D * max(c["w"] for c in cls)
    span_bytes = int(packed[0].size)

    def run(push):
        g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=max_bytes, ragged=True)
        in_push = [0.0]

        def feed(k):
            if push:
                t0 = time.perf_counter()
                for r, b in enumerate(bufs[k % N_DISTINCT]):
                    g.push(r, b)
                in_push[0] += time.perf_counter() - t0
                g.submit_pushed()
            else:
                g.L.vdl2gpu_submit_ragged(g.h, packed[k % N_DISTINCT].ctypes.data, counts.ctypes.data)
        for k in range(a.warmup):
            feed(k)
        g.flush_count()
        in_push[0] = 0.0
        frames = 0
        t0 = time.perf_counter()
        for k in range(a.spans):
            feed(k)
            frames += g.poll_count()
        frames += g.flush_count()
        t1 = time.perf_counter()
        st = g.stats()
        out = dict(period_ms_per_span=(t1 - t0) * 1e3 / a.spans, frames_per_span=frames / a.spans,
                   overflows=st["pool_overflows"] + st["out_overflows"])
        cnt = g.channel_counters()               # (before the idle-GPU spans below, which the ragged feed does not run)
        if push:
            out["push_call_ns_per_byte_pipelined"] = in_push[0] * 1e9 / (a.spans * span_bytes)
            in_push[0] = 0.0
            for k in range(4):
                g.flush_count()                  # nothing in flight: the next span's pushes find their rings free
                feed(k)
            g.flush_count()
            out["push_call_ns_per_byte_idle_gpu"] = in_push[0] * 1e9 / (4 * span_bytes)
        g.close()
        return out, cnt

    res = dict(gpu=torch.cuda.get_device_name(), card=card(), receivers=R, channels_per_receiver=C, channels=R * C,
               n_dec_per_span=D, span_bytes=span_bytes, timed_spans=a.spans, repeats=[])
    for _ in range(a.repeats):
        rag, cr = run(False)
        pus, cp = run(True)
        res["repeats"].append(dict(submit_ragged=rag, push=pus, counters_equal=bool(np.array_equal(cr, cp)),
                                   push_over_ragged=pus["period_ms_per_span"] / rag["period_ms_per_span"]))
    res["card_after"] = card()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
