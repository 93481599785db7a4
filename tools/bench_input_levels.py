#!/usr/bin/env python
"""tools/bench_input_levels.py — the cost of input levels (VDL2GPU_FLAG_INPUT_LEVELS) on the 2048 receivers x 8 channels
ragged fleet (16384 channels): the first half RTL-SDR-like (cu8, oversample 10), the second half SDRplay-like (cs16,
oversample 20), fed full device spans of 13107 decimated samples through vdl2gpu_submit_ragged_device.  Receiver r of a
class is that class's synthetic traffic stream started 7919 r decimated samples later, built on the device.  The flag is
off and on in alternation (A-B-A-B) in one process; each run reports
  - the pipelined period (ms per span, device events around the spans);
  - ms per launch of every kernel, serialised (FLAG_NO_OVERLAP + enable_timing): K0 is the kernel that changes;
  - whether the per-channel counters of the two contexts are identical;
with the GPU name, SM clock and power limit read in the same run.

    python tools/bench_input_levels.py [--receivers 2048] [--channels 8] [--spans 16] [--repeats 2] > levels.json
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
    ap.add_argument("--n-dec", type=int, default=13107, help="decimated samples of a span")
    ap.add_argument("--spans", type=int, default=16, help="timed spans per measurement")
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=2, help="alternating repetitions of off and on")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_input_levels.py needs a CUDA device: the demodulator path has no CPU fallback")
    R, C, D = a.receivers, a.channels, a.n_dec
    H = R // 2
    seconds = N_DISTINCT * D / DEC_RATE + 0.05
    cls = []
    for k, (os_, fmt, bpp) in enumerate(KINDS):
        iq, offs, _ = synth.traffic_stream(DEC_RATE * os_, seconds, 32 if os_ == 10 else 64, 4.0, 22.0, -20.0, 0x4C564C00 + k,
                                           "s16" if fmt else "u8")
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
    counts = np.full(R, D, np.uint32)
    src = [torch.cat([blocks[r // H][s, r % H].reshape(-1) for r in range(R)]).contiguous() for s in range(N_DISTINCT)]
    torch.cuda.synchronize()
    rx = [(bench.CENTER + 1000 * (r - H), [bench.CENTER + 1000 * (r - H) + int(cls[r // H]["offs"][(r * C + i) % len(cls[r // H]["offs"])])
                                           for i in range(C)], KINDS[r // H][0], KINDS[r // H][1]) for r in range(R)]
    max_bytes = D * max(c["w"] for c in cls)
    stream = torch.cuda.current_stream()

    def run(levels, timing):
        g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=max_bytes, flags=vd.FLAG_NO_OVERLAP if timing else 0, ragged=True, levels=levels)

        def feed(k):
            g.submit_ragged_device(src[k % N_DISTINCT].data_ptr(), counts, stream.cuda_stream)
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
        for k in range(a.spans):
            feed(k)
            out["frames"] += g.poll_count()
        out["frames"] += g.flush_count()
        g.stream_wait(stream.cuda_stream)
        e1.record(stream)
        torch.cuda.synchronize()
        out["ms"] = e0.elapsed_time(e1) / a.spans
        if timing:
            k1 = g.kernel_ms()
            out["kernel_ms"] = {n: (k1[n][0] - k0[n][0]) / max(k1[n][1] - k0[n][1], 1) for n in k1}
        st = g.stats()
        out["overflows"] = st["pool_overflows"] + st["out_overflows"]
        out["counters"] = g.channel_counters()
        if levels:
            out["dbfs"] = [vd.level_metrics(x)["power_dbfs"] for x in g.input_levels()]
        g.close()
        return out

    def measure(levels, sample_clocks=False):
        ser = run(levels, True)
        sampler = bench.ClockSampler(torch.cuda.current_device()) if sample_clocks else None
        if sampler:
            sampler.start()
        t0 = time.time()
        pip = run(levels, False)
        t1 = time.time()
        res = dict(kernel_ms_per_launch_serialised=ser["kernel_ms"], pipelined_ms_per_span=pip["ms"],
                   frames_per_span=pip["frames"] / a.spans, overflows=pip["overflows"])
        if sampler:
            res["clocks"] = sampler.stop(t0, t1)
        if levels:
            d = np.array(pip["dbfs"][:H]), np.array(pip["dbfs"][H:])
            res["input_dbfs_median"] = dict(cu8=float(np.median(d[0])), cs16=float(np.median(d[1])))
        return res, pip["counters"]

    res = dict(gpu=torch.cuda.get_device_name(), sms=torch.cuda.get_device_properties(0).multi_processor_count,
               receivers=R, channels_per_receiver=C, channels=R * C, span=D, timed_spans=a.spans)
    reps = []
    for i in range(a.repeats):
        off, c_off = measure(False, sample_clocks=(i == 0))
        on, c_on = measure(True)
        reps.append(dict(off=off, on=on, counters_equal=bool(np.array_equal(c_off, c_on)),
                         pipelined_on_over_off=on["pipelined_ms_per_span"] / off["pipelined_ms_per_span"],
                         k0_ms_off=off["kernel_ms_per_launch_serialised"]["K0"], k0_ms_on=on["kernel_ms_per_launch_serialised"]["K0"]))
    res["runs"] = reps
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
