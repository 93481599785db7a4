#!/usr/bin/env python
"""tools/bench_spectrum.py — the cost of the spectrum (VDL2GPU_FLAG_SPECTRUM), which k_spectrum measures from the sample
plane, on two workloads:
  - fanout: bench.py's 16384 channels (2.1 Msps cu8, oversample 20, interleaved over its 64 frequency slots) fed chunks of
    262144 complex samples from device memory;
  - ragged: 2048 receivers x 8 channels (1024 cu8 at oversample 10, then 1024 cs16 at oversample 20) fed full ragged
    device spans of 13107 decimated samples.
The flag is off and on in alternation (A-B-A-B) in one process; each run reports
  - the pipelined period (ms per chunk or span, device events around them);
  - ms per launch of every kernel, serialised (FLAG_NO_OVERLAP + enable_timing), and, with the flag on, of k_spectrum in a
    separate serialised run under torch.profiler;
  - whether the per-channel counters of the two contexts are identical;
with the GPU name, SM clock and power limit read in the same run.

    python tools/bench_spectrum.py [--workload fanout ragged] [--steps 16] [--repeats 2] > spectrum.json
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

DEC_RATE = 105000
N_DISTINCT = 3                      # ragged: distinct spans resident per receiver, submitted round robin
KINDS = [(10, vd.FMT_U8, 2), (20, vd.FMT_S16, 4)]      # (oversample, format, bytes per complex sample)


def power_limit_w():
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
    except Exception:
        return None


def fanout_workload(a):
    """(make(spec, timing) -> context, feed(g, k)) of bench.py's workload"""
    chunks, offs, _ = bench.make_stream(a.seconds)
    freqs = bench.channel_freqs(offs, 16384, "interleaved")
    dev = torch.from_numpy(np.ascontiguousarray(chunks)).cuda()
    stream = torch.cuda.current_stream()

    def make(spec, timing):
        return vd.Vdl2Channels(bench.FS, bench.OVERSAMPLE, vd.FMT_U8, bench.CENTER, freqs, max_chunk_bytes=bench.CHUNK_BYTES,
                               flags=vd.FLAG_NO_OVERLAP if timing else 0, spectrum=spec)

    def feed(g, k):
        g.submit_device(dev[k % dev.shape[0]].data_ptr(), bench.CHUNK_BYTES, stream.cuda_stream)
    return make, feed, dict(channels=16384, chunk_pairs=bench.CHUNK_PAIRS)


def ragged_workload(a):
    R, C, D = 2048, 8, 13107
    H = R // 2
    seconds = N_DISTINCT * D / DEC_RATE + 0.05
    cls = []
    for k, (os_, fmt, bpp) in enumerate(KINDS):
        iq, offs, _ = synth.traffic_stream(DEC_RATE * os_, seconds, 32 if os_ == 10 else 64, 4.0, 22.0, -20.0, 0x4C564C00 + k,
                                           "s16" if fmt else "u8")
        w = os_ * bpp
        host = np.ascontiguousarray(iq).view(np.uint8).reshape(-1)
        L = host.size // w
        cls.append(dict(w=w, offs=offs, L=L, dev=torch.from_numpy(host[:L * w].reshape(L, w)).cuda()))
    ar = torch.arange(N_DISTINCT * D, device="cuda", dtype=torch.int64)
    blocks = []                                    # per class: [N_DISTINCT, H, D, w] bytes; receiver j starts 7919 j later
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
    rx = [(bench.CENTER + 1000 * (r - H), [bench.CENTER + 1000 * (r - H) + int(cls[r // H]["offs"][(r * C + i) % len(cls[r // H]["offs"])])
                                           for i in range(C)], KINDS[r // H][0], KINDS[r // H][1]) for r in range(R)]
    max_bytes = D * max(c["w"] for c in cls)
    stream = torch.cuda.current_stream()

    def make(spec, timing):
        return vd.Vdl2MixedReceivers(rx, max_chunk_bytes=max_bytes, flags=vd.FLAG_NO_OVERLAP if timing else 0, ragged=True,
                                     spectrum=spec)

    def feed(g, k):
        g.submit_ragged_device(src[k % N_DISTINCT].data_ptr(), counts, stream.cuda_stream)
    return make, feed, dict(receivers=R, channels_per_receiver=C, channels=R * C, span=D)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=["fanout", "ragged"], choices=["fanout", "ragged"])
    ap.add_argument("--steps", type=int, default=16, help="timed chunks or spans per measurement")
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=2, help="alternating repetitions of off and on")
    ap.add_argument("--seconds", type=float, default=1.5, help="fanout: seconds of synthetic stream resident on the device")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_spectrum.py needs a CUDA device: the demodulator path has no CPU fallback")
    stream = torch.cuda.current_stream()
    res = dict(gpu=torch.cuda.get_device_name(), sms=torch.cuda.get_device_properties(0).multi_processor_count,
               power_limit_w=power_limit_w(), timed_steps=a.steps, workloads={})
    for wl in a.workload:
        make, feed, desc = (fanout_workload if wl == "fanout" else ragged_workload)(a)
        torch.cuda.synchronize()

        def run(spec, timing, profile=False):
            g = make(spec, timing)
            out = dict(frames=0)
            for k in range(a.warmup):
                feed(g, k)
            g.flush_count()
            if timing:
                g.enable_timing(True)
                k0 = g.kernel_ms()
            torch.cuda.synchronize()
            if profile:
                # the spectrum kernel's own device time, from the CUDA activity records of a serialised run
                from torch.profiler import profile as prof, ProfilerActivity
                with prof(activities=[ProfilerActivity.CUDA]) as p:
                    for k in range(a.steps):
                        feed(g, k)
                        g.poll_count()
                    g.flush_count()
                    torch.cuda.synchronize()
                ks = [e for e in p.events() if e.name.startswith("k_spectrum")]
                g.close()
                return dict(k_spectrum_ms=sum(e.device_time_total for e in ks) / 1000.0 / max(len(ks), 1), launches=len(ks))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for k in range(a.steps):
                feed(g, k)
                out["frames"] += g.poll_count()
            out["frames"] += g.flush_count()
            g.stream_wait(stream.cuda_stream)
            e1.record(stream)
            torch.cuda.synchronize()
            out["ms"] = e0.elapsed_time(e1) / a.steps
            if timing:
                k1 = g.kernel_ms()
                out["kernel_ms"] = {n: (k1[n][0] - k0[n][0]) / max(k1[n][1] - k0[n][1], 1) for n in k1}
            st = g.stats()
            out["overflows"] = st["pool_overflows"] + st["out_overflows"]
            out["counters"] = g.channel_counters()
            if spec:
                rec = g.spectrum(0, 1)[0]
                out["segments_input0"] = int(rec["segments"])
            g.close()
            return out

        def measure(spec, sample_clocks=False):
            ser = run(spec, True)
            sampler = bench.ClockSampler(torch.cuda.current_device()) if sample_clocks else None
            if sampler:
                sampler.start()
            t0 = time.time()
            pip = run(spec, False)
            t1 = time.time()
            r = dict(kernel_ms_per_launch_serialised=ser["kernel_ms"], pipelined_ms_per_step=pip["ms"],
                     frames_per_step=pip["frames"] / a.steps, overflows=pip["overflows"])
            if sampler:
                r["clocks"] = sampler.stop(t0, t1)
            if spec:
                r["segments_input0"] = pip["segments_input0"]
                r["k_spectrum_serialised"] = run(spec, True, profile=True)
            return r, pip["counters"]

        reps = []
        for i in range(a.repeats):
            off, c_off = measure(False, sample_clocks=(i == 0))
            on, c_on = measure(True)
            reps.append(dict(off=off, on=on, counters_equal=bool(np.array_equal(c_off, c_on)),
                             pipelined_on_over_off=on["pipelined_ms_per_step"] / off["pipelined_ms_per_step"],
                             k_spectrum_ms=on["k_spectrum_serialised"]["k_spectrum_ms"]))
        res["workloads"][wl] = dict(desc, runs=reps)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
