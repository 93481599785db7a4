#!/usr/bin/env python
"""tools/bench_k2_stage.py — where the pipeline period of bench.py's workload goes: each kernel alone, and the pipelined
period, in one process.  bench.py's fan-out context (16384 interleaved channels, cu8, 262144-pair chunks, chunks resident
in HBM) is run twice:
  - serialised (FLAG_NO_OVERLAP + enable_timing): K0, K1, K2a, K2 and K3 ms per launch, CUDA events over --chunks launches;
  - the default pipeline (K2a of chunk c alone, then K0/K1 of chunk c+1 beside K2/K3 of chunk c, graph replay): ms per
    chunk between two events over --chunks chunks.
The pipelined period is K2a plus the longer of K1 and K2 (+K3) when the overlap is perfect; `model_period_ms` prints that
sum from the serialised times beside the measured period.  The GPU name, SM clock and power limit are read by NVML in
the same run.

--order replica lays the 256 replicas of a slot side by side, so the 32 lanes of a warp carry one signal and never
diverge; set against the default interleaved order it shows what divergence between lanes costs each kernel.

    python tools/bench_k2_stage.py [--channels 16384] [--order interleaved|replica] [--chunks 48] [--warmup 8] > k2_stage.json
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench
import dumpvdl2_b200 as vd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=16384)
    ap.add_argument("--chunks", type=int, default=48, help="timed launches per measurement")
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--order", default="interleaved", choices=["interleaved", "replica"], help="channel order, as bench.py --channel-order")
    ap.add_argument("--label", default="", help="free text copied into the result (e.g. which build)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_k2_stage.py needs a CUDA device: the demodulator path has no CPU fallback")
    chunks, offs, _ = bench.make_stream(2.0)
    d_chunks = torch.from_numpy(chunks).cuda()
    n_chunks = d_chunks.shape[0]
    freqs = bench.channel_freqs(offs, a.channels, a.order)
    stream = torch.cuda.current_stream()

    def make(flags):
        return vd.Vdl2Channels(bench.FS, bench.OVERSAMPLE, vd.FMT_U8, bench.CENTER, freqs, max_chunk_bytes=bench.CHUNK_BYTES,
                               flags=flags)

    def feed(g, k):
        g.submit_device(d_chunks[k % n_chunks].data_ptr(), bench.CHUNK_BYTES, stream.cuda_stream)

    res = dict(gpu=torch.cuda.get_device_name(), label=a.label, order=a.order, channels=a.channels, chunk_pairs=bench.CHUNK_PAIRS,
               timed_chunks=a.chunks)

    g = make(vd.FLAG_NO_OVERLAP)
    for k in range(a.warmup):
        feed(g, k)
    g.flush_count()
    g.enable_timing(True)
    k0 = g.kernel_ms()
    for k in range(a.chunks):
        feed(g, a.warmup + k)
        g.poll_count()
    g.flush_count()
    k1 = g.kernel_ms()
    g.close()
    kms = {k: (k1[k][0] - k0[k][0]) / max(k1[k][1] - k0[k][1], 1) for k in k1}
    res["kernel_ms_serialised"] = kms

    g = make(0)
    for k in range(a.warmup):
        feed(g, k)
    g.flush_count()
    sampler = bench.ClockSampler(torch.cuda.current_device())
    sampler.start()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.time()
    e0.record(stream)
    for k in range(a.chunks):
        feed(g, a.warmup + k)
        g.poll_count()
    g.flush_count()
    g.stream_wait(stream.cuda_stream)
    e1.record(stream)
    torch.cuda.synchronize()
    t1 = time.time()
    g.close()
    period = e0.elapsed_time(e1) / a.chunks
    res["pipelined_ms_per_chunk"] = period
    res["pipelined_g_chsamples_per_s"] = a.channels * bench.CHUNK_PAIRS / (period * 1e-3) / 1e9
    res["model_period_ms"] = kms.get("K2a", 0.0) + max(kms.get("K0", 0.0) + kms.get("K1", 0.0), kms.get("K2", 0.0) + kms.get("K3", 0.0))
    res["paced_by"] = "K2+K3" if kms.get("K2", 0.0) + kms.get("K3", 0.0) > kms.get("K0", 0.0) + kms.get("K1", 0.0) else "K0+K1"
    res["clocks"] = sampler.stop(t0, t1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
