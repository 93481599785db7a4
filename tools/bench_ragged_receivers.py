#!/usr/bin/env python
"""tools/bench_ragged_receivers.py — ragged spans (Vdl2MixedReceivers(..., ragged=True), vdl2gpu_submit_ragged_device)
against the lock-step mixed context on the same fleet.  R receivers x C channels (default 2048 x 8 = 16384 channels),
grouped by rate: the first half RTL-SDR-like (cu8, oversample 10), the second half SDRplay-like (cs16, oversample 20);
spans of up to 13107 decimated samples.  Receiver r of a class is that class's synthetic traffic stream started 7919 r
decimated samples later, built on the device.  Feeds:
  (a) full spans, on a ragged context and, in the same run and alternating with it, on a plain mixed context;
  (b) 10 % of the receivers (seeded) at half width, the others full;
  (c) 10 % of the receivers absent, the others full.
One process reports, with the GPU name, SM clock and power limit read in the same run:
  - per-kernel ms per launch, serialised (FLAG_NO_OVERLAP + enable_timing);
  - pipelined ms per span;
  - whether the ragged context fed (a) ends with the same per-channel counters as the plain context.

    python tools/bench_ragged_receivers.py [--receivers 2048] [--channels 8] [--spans 16] > ragged.json
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

N_DISTINCT = 3                      # distinct spans resident per receiver, submitted round robin
DEC_RATE = 105000
KINDS = [(10, vd.FMT_U8, 2), (20, vd.FMT_S16, 4)]      # (oversample, format, bytes per complex sample)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--receivers", type=int, default=2048, help="even: half of each rate")
    ap.add_argument("--channels", type=int, default=8, help="channels per receiver")
    ap.add_argument("--n-dec", type=int, default=13107, help="decimated samples of a full span")
    ap.add_argument("--spans", type=int, default=16, help="timed spans per measurement")
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=2, help="alternating repetitions of feed (a) on both contexts")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged_receivers.py needs a CUDA device: the demodulator path has no CPU fallback")
    R, C, D = a.receivers, a.channels, a.n_dec
    H = R // 2
    seconds = N_DISTINCT * D / DEC_RATE + 0.05
    cls = []
    for k, (os_, fmt, bpp) in enumerate(KINDS):
        n_slots = 32 if os_ == 10 else 64
        iq, offs, _ = synth.traffic_stream(DEC_RATE * os_, seconds, n_slots, 4.0, 22.0, -20.0, 0x52414700 + k, "s16" if fmt else "u8")
        w = os_ * bpp
        host = np.ascontiguousarray(iq).view(np.uint8).reshape(-1)
        L = host.size // w
        cls.append(dict(os=os_, fmt=fmt, w=w, offs=offs, L=L, dev=torch.from_numpy(host[:L * w].reshape(L, w)).cuda()))
    ar = torch.arange(N_DISTINCT * D, device="cuda", dtype=torch.int64)
    blocks = []                                    # per class: [N_DISTINCT, H, D, w] bytes, receiver j of the class
    for c in cls:
        blk = torch.empty(N_DISTINCT, H, D, c["w"], dtype=torch.uint8, device="cuda")
        for j0 in range(0, H, 64):
            sh = (torch.arange(j0, min(j0 + 64, H), device="cuda", dtype=torch.int64) * 7919) % c["L"]
            g = c["dev"][(ar[None, :] + sh[:, None]) % c["L"]]
            for s in range(N_DISTINCT):
                blk[s, j0:j0 + g.shape[0]] = g[:, s * D:(s + 1) * D]
        del g
        blocks.append(blk)
    widths = [cls[0]["w"]] * H + [cls[1]["w"]] * H

    def pack(counts):
        """[N_DISTINCT] device spans with receiver r's first counts[r] decimated samples, back to back"""
        out = []
        for s in range(N_DISTINCT):
            parts = [blocks[r // H][s, r % H, :int(counts[r])].reshape(-1) for r in range(R) if counts[r]]
            out.append(torch.cat(parts).contiguous())
        return out

    rng = np.random.default_rng(0x52414700)
    some = rng.choice(R, R // 10, replace=False)
    full = np.full(R, D, np.uint32)
    half = full.copy()
    half[some] = D // 2
    absent = full.copy()
    absent[some] = 0
    feeds = dict(full=(full, pack(full)), half_width_10pct=(half, pack(half)), absent_10pct=(absent, pack(absent)))
    torch.cuda.synchronize()

    rx = [(bench.CENTER + 1000 * (r - H), [bench.CENTER + 1000 * (r - H) + int(cls[r // H]["offs"][(r * C + i) % len(cls[r // H]["offs"])])
                                           for i in range(C)], KINDS[r // H][0], KINDS[r // H][1]) for r in range(R)]
    n_ch = R * C
    max_bytes = D * max(c["w"] for c in cls)
    stream = torch.cuda.current_stream()

    def run(ragged, counts, src, spans, timing):
        g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=max_bytes, flags=vd.FLAG_NO_OVERLAP if timing else 0, ragged=ragged)
        if ragged:
            def feed(k):
                g.submit_ragged_device(src[k % N_DISTINCT].data_ptr(), counts, stream.cuda_stream)
        else:
            def feed(k):
                g.submit_span_device(src[k % N_DISTINCT].data_ptr(), D, stream.cuda_stream)
        out = dict(kernel_ms={}, frames=0)
        for k in range(a.warmup):
            feed(k)
        g.flush_count()
        if timing:
            g.enable_timing(True)
            k0 = g.kernel_ms()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for k in range(spans):
            feed(k)
            out["frames"] += g.poll_count()
        out["frames"] += g.flush_count()
        g.stream_wait(stream.cuda_stream)
        e1.record(stream)
        torch.cuda.synchronize()
        out["ms"] = e0.elapsed_time(e1) / spans
        if timing:
            k1 = g.kernel_ms()
            out["kernel_ms"] = {n: (k1[n][0] - k0[n][0]) / max(k1[n][1] - k0[n][1], 1) for n in k1}
        st = g.stats()
        out["overflows"] = st["pool_overflows"] + st["out_overflows"]
        out["graph_launches"] = st["graph_launches"]
        out["counters"] = g.channel_counters()
        g.close()
        return out

    def measure(ragged, name, sample_clocks=False):
        counts, src = feeds[name]
        ser = run(ragged, counts, src, a.spans, True)
        sampler = bench.ClockSampler(torch.cuda.current_device()) if sample_clocks else None
        if sampler:
            sampler.start()
        t0 = time.time()
        pip = run(ragged, counts, src, a.spans, False)
        t1 = time.time()
        res = dict(kernel_ms_per_launch_serialised=ser["kernel_ms"], pipelined_ms_per_span=pip["ms"],
                   frames_per_span=pip["frames"] / a.spans, overflows=pip["overflows"], graph_launches=pip["graph_launches"])
        if sampler:
            res["clocks"] = sampler.stop(t0, t1)
        return res, pip["counters"]

    res = dict(gpu=torch.cuda.get_device_name(), sms=torch.cuda.get_device_properties(0).multi_processor_count,
               receivers=R, channels_per_receiver=C, channels=n_ch, full_span=D, timed_spans=a.spans,
               classes=[dict(oversample=c["os"], fmt="cs16" if c["fmt"] else "cu8", receivers=H) for c in cls],
               lagging_receivers=len(some))
    reps = []
    for i in range(a.repeats):                     # (a): the two contexts alternate
        plain, cp = measure(False, "full", sample_clocks=(i == 0))
        rag, cr = measure(True, "full")
        reps.append(dict(plain_mixed=plain, ragged=rag, counters_equal=bool(np.array_equal(cp, cr)),
                         pipelined_ragged_over_plain=rag["pipelined_ms_per_span"] / plain["pipelined_ms_per_span"]))
    res["a_full_spans"] = reps
    res["b_half_width_10pct"] = measure(True, "half_width_10pct")[0]
    res["c_absent_10pct"] = measure(True, "absent_10pct")[0]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
