#!/usr/bin/env python
"""tools/bench_receivers.py — many receivers in one context (vdl2gpu_create_receivers) against the fan-out context at the
same channel count.  R receivers x C channels (default 2048 x 8 = 16384 channels), cu8, 262144-pair chunks.  Receiver r is
bench.py's stream started 7919 r samples later, built on the device; it has its own centre frequency, and its channels sit
at that centre plus the stream's slot offsets (channel j of receiver r on slot (r C + j) mod 64), so every channel sees
traffic.  One process reports, with the GPU name, SM clock and power limit read in the same run:
  - per-kernel ms, serialised (FLAG_NO_OVERLAP + enable_timing), receivers and fan-out;
  - pipelined ms per chunk and channel-samples/s, receivers and fan-out (bench.py's workload at the same channel count);
  - frame and counter parity of a sample of receivers against the oracle run per receiver.

    python tools/bench_receivers.py [--receivers 2048] [--channels 8] [--chunks 24] > receivers.json
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

N_DISTINCT = 3                      # distinct chunks resident per receiver (R x 512 KB each), submitted round robin


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--receivers", type=int, default=2048)
    ap.add_argument("--channels", type=int, default=8, help="channels per receiver")
    ap.add_argument("--chunks", type=int, default=24, help="timed chunks per measurement")
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--parity", default="0,1,63,64,79,1023,last", help="receivers checked against the oracle")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_receivers.py needs a CUDA device: the demodulator path has no CPU fallback")
    R, C, P = a.receivers, a.channels, bench.CHUNK_PAIRS
    nbytes = 2 * P
    chunks, offs, _ = bench.make_stream(2.0)
    base = torch.from_numpy(chunks.reshape(-1)).cuda()
    L = base.numel() // 2
    base2 = base.view(L, 2)
    raw = torch.empty(N_DISTINCT, R, P, 2, dtype=torch.uint8, device="cuda")
    ar = torch.arange(N_DISTINCT * P, device="cuda", dtype=torch.int64)
    for r0 in range(0, R, 32):                      # receiver r = the stream started 7919 r samples later (wrapping)
        sh = (torch.arange(r0, min(r0 + 32, R), device="cuda", dtype=torch.int64) * 7919) % L
        blk = base2[(ar[None, :] + sh[:, None]) % L]
        for k in range(N_DISTINCT):
            raw[k, r0:r0 + blk.shape[0]] = blk[:, k * P:(k + 1) * P]
    del blk
    fan = torch.from_numpy(chunks[:N_DISTINCT]).cuda()
    torch.cuda.synchronize()
    centres = [bench.CENTER + 1000 * (r - R // 2) for r in range(R)]
    rx = [(centres[r], [centres[r] + int(offs[(r * C + j) % bench.N_SLOTS]) for j in range(C)]) for r in range(R)]
    n_ch = R * C
    stream = torch.cuda.current_stream()

    def receivers(flags=0):
        return vd.Vdl2Receivers(bench.FS, bench.OVERSAMPLE, vd.FMT_U8, rx, max_chunk_bytes=nbytes, flags=flags)

    def fanout(flags=0):
        return vd.Vdl2Channels(bench.FS, bench.OVERSAMPLE, vd.FMT_U8, bench.CENTER, bench.channel_freqs(offs, n_ch, "interleaved"),
                               max_chunk_bytes=nbytes, flags=flags)

    def feed(g, src, k):
        g.submit_device(src[k % N_DISTINCT].data_ptr(), nbytes, stream.cuda_stream)

    def measure(make, src, sample_clocks=False):
        out = {}
        g = make(vd.FLAG_NO_OVERLAP)                # serialised: one stream, per-kernel events
        for k in range(a.warmup):
            feed(g, src, k)
        g.flush_count()
        g.enable_timing(True)
        k0 = g.kernel_ms()
        for k in range(a.chunks):
            feed(g, src, k)
            g.poll_count()
        g.flush_count()
        k1 = g.kernel_ms()
        out["kernel_ms_serialised"] = {k: (k1[k][0] - k0[k][0]) / max(k1[k][1] - k0[k][1], 1) for k in k1}
        g.close()
        g = make(0)                                 # the default pipeline (graphs, K2(c) beside K1(c+1))
        for k in range(a.warmup):
            feed(g, src, k)
        g.flush_count()
        sampler = bench.ClockSampler(torch.cuda.current_device()) if sample_clocks else None
        if sampler:
            sampler.start()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.time()
        e0.record(stream)
        frames = 0
        for k in range(a.chunks):
            feed(g, src, k)
            frames += g.poll_count()
        frames += g.flush_count()
        g.stream_wait(stream.cuda_stream)
        e1.record(stream)
        torch.cuda.synchronize()
        t1 = time.time()
        ms = e0.elapsed_time(e1) / a.chunks
        st = g.stats()
        out.update(pipelined_ms_per_chunk=ms, pipelined_g_chsamples_per_s=n_ch * P / (ms * 1e-3) / 1e9,
                   frames_per_chunk=frames / a.chunks, pool_overflows=st["pool_overflows"], out_overflows=st["out_overflows"])
        if sampler:
            out["clocks"] = sampler.stop(t0, t1)
        g.close()
        return out

    res = dict(gpu=torch.cuda.get_device_name(), sms=torch.cuda.get_device_properties(0).multi_processor_count,
               receivers=R, channels_per_receiver=C, channels=n_ch, chunk_pairs=P, timed_chunks=a.chunks)
    res["receivers_ctx"] = measure(receivers, raw, sample_clocks=True)
    res["fanout_ctx"] = measure(fanout, fan)
    rk, fk = res["receivers_ctx"], res["fanout_ctx"]
    res["ratio_receivers_over_fanout"] = dict(
        k1_ms=rk["kernel_ms_serialised"]["K1"] / fk["kernel_ms_serialised"]["K1"],
        k0_ms=rk["kernel_ms_serialised"]["K0"] / fk["kernel_ms_serialised"]["K0"],
        pipelined_ms=rk["pipelined_ms_per_chunk"] / fk["pipelined_ms_per_chunk"])

    # parity: a fresh context on the first N_DISTINCT chunks, sampled receivers against the oracle run per receiver
    from oracle import pyoracle as po
    g = receivers()
    for k in range(N_DISTINCT):
        feed(g, raw, k)
    got = {}
    for f in g.flush():
        got.setdefault(g.receiver_of(f.channel), []).append(f)
    cnt = g.channel_counters()
    g.close()
    host = chunks.reshape(-1)[:2 * L]
    par = []
    for s in a.parity.split(","):
        r = R - 1 if s == "last" else int(s)
        iq = np.roll(host, -2 * ((7919 * r) % L))[:N_DISTINCT * nbytes]
        o = po.Oracle(bench.FS, bench.OVERSAMPLE, po.FMT_U8, centres[r], rx[r][1])
        o.process_chunked(iq, nbytes)
        want = sorted((f.channel, f.burst_seq, f.idx, f.data, f.num_fec_corrections, f.sync_dec_index,
                       np.float32(f.frame_pwr).tobytes(), np.float32(f.ppm_error).tobytes()) for f in o.frames())
        mine = sorted((f.channel - r * C, f.burst_seq, f.idx, f.data, f.num_fec_corrections, f.sync_dec_index,
                       np.float32(f.frame_pwr).tobytes(), np.float32(f.ppm_error).tobytes()) for f in got.get(r, []))
        par.append(dict(receiver=r, frames=len(want), frames_equal=mine == want,
                        counters_equal=bool(np.array_equal(cnt[r * C:(r + 1) * C], o.counters()))))
    res["parity"] = dict(chunks=N_DISTINCT, receivers=par, all_equal=all(p["frames_equal"] and p["counters_equal"] for p in par))
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
