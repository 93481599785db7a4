#!/usr/bin/env python
"""tools/bench_mixed_receivers.py — receivers of different sample rates and formats in one context
(vdl2gpu_create_mixed_receivers) against two uniform receiver contexts run one after the other on the same signal.
R receivers x C channels (default 2048 x 8 = 16384 channels), half RTL-SDR-like (cu8, oversample 10, 1.05 Msps), half
SDRplay-like (cs16, oversample 20, 2.1 Msps), spans of 13107 decimated samples (the largest 1 MiB of cs16 allows).
Receiver r of a class is that class's synthetic traffic stream started 7919 r decimated samples later, built on the
device, tuned to its own centre.  The mixed context runs with the receivers in two orders: grouped by rate (all cu8
receivers first) and interleaved (rates alternate receiver by receiver, so nearly every K1 warp runs two arms).  One
process reports, with the GPU name, SM clock and power limit read in the same run:
  - per-kernel ms per launch, serialised (FLAG_NO_OVERLAP + enable_timing);
  - pipelined ms per span and real-time channels = channels x (n_dec / 105000 s) / period;
  - frame and counter parity of a sample of receivers against the oracle run per receiver.

    python tools/bench_mixed_receivers.py [--receivers 2048] [--channels 8] [--spans 16] > mixed.json
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
    ap.add_argument("--n-dec", type=int, default=13107, help="decimated samples per span")
    ap.add_argument("--spans", type=int, default=16, help="timed spans per measurement")
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--parity", default="0,1,63,64,79,1023,1024,last", help="receivers (grouped order) checked against the oracle")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mixed_receivers.py needs a CUDA device: the demodulator path has no CPU fallback")
    R, C, D = a.receivers, a.channels, a.n_dec
    H = R // 2
    seconds = N_DISTINCT * D / DEC_RATE + 0.05
    # per class: host stream (bytes, whole decimated samples), its slot offsets, device copy [L, width]
    cls = []
    for k, (os_, fmt, bpp) in enumerate(KINDS):
        n_slots = 32 if os_ == 10 else 64          # the 25 kHz slots that fit the class's bandwidth
        iq, offs, _ = synth.traffic_stream(DEC_RATE * os_, seconds, n_slots, 4.0, 22.0, -20.0, 0x4D495800 + k, "s16" if fmt else "u8")
        w = os_ * bpp
        host = np.ascontiguousarray(iq).view(np.uint8).reshape(-1)
        L = host.size // w
        host = host[:L * w]
        cls.append(dict(os=os_, fmt=fmt, w=w, host=host, offs=offs, L=L, dev=torch.from_numpy(host.reshape(L, w)).cuda()))
    ar = torch.arange(N_DISTINCT * D, device="cuda", dtype=torch.int64)
    blocks = []                                    # per class: [N_DISTINCT, H, D x w] bytes, receiver j of the class
    for c in cls:
        blk = torch.empty(N_DISTINCT, H, D * c["w"], dtype=torch.uint8, device="cuda")
        for j0 in range(0, H, 64):
            sh = (torch.arange(j0, min(j0 + 64, H), device="cuda", dtype=torch.int64) * 7919) % c["L"]
            g = c["dev"][(ar[None, :] + sh[:, None]) % c["L"]]
            for s in range(N_DISTINCT):
                blk[s, j0:j0 + g.shape[0]] = g[:, s * D:(s + 1) * D].reshape(g.shape[0], -1)
        del g
        blocks.append(blk)
    grouped = torch.cat([blocks[0].reshape(N_DISTINCT, -1), blocks[1].reshape(N_DISTINCT, -1)], dim=1).contiguous()
    interleaved = torch.cat([blocks[0], blocks[1]], dim=2).reshape(N_DISTINCT, -1).contiguous()
    torch.cuda.synchronize()

    def rx_of(k, j):                               # receiver j of class k: (centre, freqs)
        c = cls[k]
        centre = bench.CENTER + 1000 * (k * H + j - H)
        return centre, [centre + int(c["offs"][(j * C + i) % len(c["offs"])]) for i in range(C)]
    rx = [[rx_of(k, j) for j in range(H)] for k in range(2)]
    mixed_grouped = [(*rx[k][j], KINDS[k][0], KINDS[k][1]) for k in range(2) for j in range(H)]
    mixed_inter = [(*rx[k][j], KINDS[k][0], KINDS[k][1]) for j in range(H) for k in range(2)]
    n_ch = R * C
    max_bytes = D * max(c["w"] for c in cls)
    stream = torch.cuda.current_stream()

    def run(contexts, spans, timing):
        """contexts: [(make(flags), feed(g, k))]: each context fed `spans` spans, one context after the other"""
        out = dict(kernel_ms={}, ms=0.0, frames=0, pool_overflows=0, out_overflows=0)
        for make, feed in contexts:
            g = make(vd.FLAG_NO_OVERLAP if timing else 0)
            for k in range(a.warmup):
                feed(g, k)
            g.flush_count()
            if timing:
                g.enable_timing(True)
                k0 = g.kernel_ms()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for k in range(spans):
                feed(g, k)
                out["frames"] += g.poll_count()
            out["frames"] += g.flush_count()
            g.stream_wait(stream.cuda_stream)
            e1.record(stream)
            torch.cuda.synchronize()
            out["ms"] += e0.elapsed_time(e1) / spans
            if timing:
                k1 = g.kernel_ms()
                for n in k1:
                    out["kernel_ms"][n] = out["kernel_ms"].get(n, 0.0) + (k1[n][0] - k0[n][0]) / max(k1[n][1] - k0[n][1], 1)
            st = g.stats()
            out["pool_overflows"] += st["pool_overflows"]
            out["out_overflows"] += st["out_overflows"]
            g.close()
        return out

    def measure(contexts, sample_clocks=False):
        ser = run(contexts, a.spans, True)
        sampler = bench.ClockSampler(torch.cuda.current_device()) if sample_clocks else None
        if sampler:
            sampler.start()
        t0 = time.time()
        pip = run(contexts, a.spans, False)
        t1 = time.time()
        res = dict(k0_ms=ser["kernel_ms"]["K0"], k1_ms=ser["kernel_ms"]["K1"], kernel_ms_serialised=ser["kernel_ms"],
                   pipelined_ms_per_span=pip["ms"], realtime_channels=n_ch * (D / DEC_RATE) / (pip["ms"] * 1e-3),
                   frames_per_span=pip["frames"] / a.spans, pool_overflows=pip["pool_overflows"], out_overflows=pip["out_overflows"])
        if sampler:
            res["clocks"] = sampler.stop(t0, t1)
        return res

    def mixed(order, src):
        def make(flags):
            return vd.Vdl2MixedReceivers(order, max_chunk_bytes=max_bytes, flags=flags)

        def feed(g, k):
            g.submit_span_device(src[k % N_DISTINCT].data_ptr(), D, stream.cuda_stream)
        return [(make, feed)]

    def uniform():
        ctxs = []
        for k, (os_, fmt, bpp) in enumerate(KINDS):
            def make(flags, k=k, os_=os_, fmt=fmt):
                return vd.Vdl2Receivers(DEC_RATE * os_, os_, fmt, rx[k], max_chunk_bytes=max_bytes, flags=flags)

            def feed(g, j, k=k):
                g.submit_device(blocks[k][j % N_DISTINCT].data_ptr(), D * cls[k]["w"], stream.cuda_stream)
            ctxs.append((make, feed))
        return ctxs

    res = dict(gpu=torch.cuda.get_device_name(), sms=torch.cuda.get_device_properties(0).multi_processor_count,
               receivers=R, channels_per_receiver=C, channels=n_ch, n_dec_per_span=D, timed_spans=a.spans,
               classes=[dict(oversample=c["os"], fmt="cs16" if c["fmt"] else "cu8", receivers=H) for c in cls])
    res["mixed_grouped"] = measure(mixed(mixed_grouped, grouped), sample_clocks=True)
    res["mixed_interleaved"] = measure(mixed(mixed_inter, interleaved))
    res["two_uniform_contexts"] = measure(uniform())
    gk, ik, uk = res["mixed_grouped"], res["mixed_interleaved"], res["two_uniform_contexts"]
    res["ratios"] = dict(k1_grouped_over_uniform=gk["k1_ms"] / uk["k1_ms"], k1_interleaved_over_grouped=ik["k1_ms"] / gk["k1_ms"],
                         pipelined_grouped_over_uniform=gk["pipelined_ms_per_span"] / uk["pipelined_ms_per_span"],
                         pipelined_interleaved_over_grouped=ik["pipelined_ms_per_span"] / gk["pipelined_ms_per_span"])

    # parity: a fresh grouped context on the N_DISTINCT spans, sampled receivers against the oracle run per receiver
    from oracle import pyoracle as po
    g = vd.Vdl2MixedReceivers(mixed_grouped, max_chunk_bytes=max_bytes)
    for k in range(N_DISTINCT):
        g.submit_span_device(grouped[k].data_ptr(), D, stream.cuda_stream)
    got = {}
    for f in g.flush():
        got.setdefault(g.receiver_of(f.channel), []).append(f)
    cnt = g.channel_counters()
    g.close()
    par = []
    for s in a.parity.split(","):
        r = R - 1 if s == "last" else int(s)
        k, j = divmod(r, H)
        c = cls[k]
        iq = np.roll(c["host"], -((7919 * j) % c["L"]) * c["w"])[:N_DISTINCT * D * c["w"]]
        o = po.Oracle(DEC_RATE * c["os"], c["os"], po.FMT_S16 if c["fmt"] else po.FMT_U8, rx[k][j][0], rx[k][j][1])
        o.process_chunked(iq, D * c["w"])
        want = sorted((f.channel, f.burst_seq, f.idx, f.data, f.num_fec_corrections, f.sync_dec_index,
                       np.float32(f.frame_pwr).tobytes(), np.float32(f.ppm_error).tobytes()) for f in o.frames())
        mine = sorted((f.channel - r * C, f.burst_seq, f.idx, f.data, f.num_fec_corrections, f.sync_dec_index,
                       np.float32(f.frame_pwr).tobytes(), np.float32(f.ppm_error).tobytes()) for f in got.get(r, []))
        par.append(dict(receiver=r, oversample=c["os"], frames=len(want), frames_equal=mine == want,
                        counters_equal=bool(np.array_equal(cnt[r * C:(r + 1) * C], o.counters()))))
    res["parity"] = dict(spans=N_DISTINCT, receivers=par, all_equal=all(p["frames_equal"] and p["counters_equal"] for p in par))
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
