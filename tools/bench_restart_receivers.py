#!/usr/bin/env python
"""tools/bench_restart_receivers.py — the cost of receiver restarts (vdl2gpu_restart_receiver) on the 2048 x 8 fleet of
bench_ragged_receivers.py: grouped by rate, the first half cu8 at oversample 10, the second half cs16 at oversample 20,
full ragged spans of 13107 decimated samples fed through submit_ragged_device.  Reports, with the GPU name, SM clock and
power limit read in the same run:
  (a) the pipelined period of ordinary ragged spans (CUDA graphs) of this build against another build of the library
      (--parent: the root of a checkout whose dumpvdl2_b200/libvdl2gpu.so has been built), alternated, each in its own
      process, --repeats times;
  (b) on a context without graphs (every span takes the direct path, as a restart span does): the pipelined period of
      spans in each of which 10 % of the receivers (seeded, a third of them retuned) restart, against ordinary spans,
      alternated; and the serialised per-kernel times of both.

    python tools/bench_restart_receivers.py [--parent DIR] [--spans 16] > restart.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_DISTINCT = 3                      # distinct spans resident per receiver, submitted round robin
DEC_RATE = 105000


def _fleet(a, vd, synth, torch, bench):
    R, C, D = a.receivers, a.channels, a.n_dec
    H = R // 2
    kinds = [(10, vd.FMT_U8, 2), (20, vd.FMT_S16, 4)]
    seconds = N_DISTINCT * D / DEC_RATE + 0.05
    cls = []
    for k, (os_, fmt, bpp) in enumerate(kinds):
        iq, offs, _ = synth.traffic_stream(DEC_RATE * os_, seconds, 32 if os_ == 10 else 64, 4.0, 22.0, -20.0, 0x52414700 + k,
                                           "s16" if fmt else "u8")
        w = os_ * bpp
        host = np.ascontiguousarray(iq).view(np.uint8).reshape(-1)
        L = host.size // w
        cls.append(dict(w=w, offs=offs, L=L, dev=torch.from_numpy(host[:L * w].reshape(L, w)).cuda()))
    ar = torch.arange(N_DISTINCT * D, device="cuda", dtype=torch.int64)
    spans = [[] for _ in range(N_DISTINCT)]
    for c in cls:
        for j0 in range(0, H, 64):
            sh = (torch.arange(j0, min(j0 + 64, H), device="cuda", dtype=torch.int64) * 7919) % c["L"]
            g = c["dev"][(ar[None, :] + sh[:, None]) % c["L"]]
            for s in range(N_DISTINCT):
                spans[s].append(g[:, s * D:(s + 1) * D].reshape(-1))
    src = [torch.cat(p).contiguous() for p in spans]
    rx = [(bench.CENTER + 1000 * (r - H), [bench.CENTER + 1000 * (r - H) + int(cls[r // H]["offs"][(r * C + i) % len(cls[r // H]["offs"])])
                                           for i in range(C)], kinds[r // H][0], kinds[r // H][1]) for r in range(R)]
    return rx, src, D * max(c["w"] for c in cls)


def child(a):
    """one build, in this process: (a) only, or (b) with --restarts"""
    import torch
    import bench
    import dumpvdl2_b200 as vd
    from dumpvdl2_b200 import synth
    rx, src, max_bytes = _fleet(a, vd, synth, torch, bench)
    R, D = a.receivers, a.n_dec
    counts = np.full(R, D, np.uint32)
    stream = torch.cuda.current_stream()
    rng = np.random.default_rng(0x52535400)
    some = sorted(int(r) for r in rng.choice(R, R // 10, replace=False))

    def run(flags, restart, spans, timing):
        g = vd.Vdl2MixedReceivers(rx, max_chunk_bytes=max_bytes, flags=flags | (vd.FLAG_NO_OVERLAP if timing else 0), ragged=True)

        def feed(k):
            if restart:
                for r in some:
                    g.restart_receiver(r, None, rx[r][1][::-1] if r % 3 == 0 and k % 2 == 0 else rx[r][1] if r % 3 == 0 else None)
            g.submit_ragged_device(src[k % N_DISTINCT].data_ptr(), counts, stream.cuda_stream)
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
            g.poll_count()
        g.flush_count()
        g.stream_wait(stream.cuda_stream)
        e1.record(stream)
        torch.cuda.synchronize()
        out = dict(ms=e0.elapsed_time(e1) / spans)
        if timing:
            k1 = g.kernel_ms()
            out["kernel_ms"] = {n: (k1[n][0] - k0[n][0]) / max(k1[n][1] - k0[n][1], 1) for n in k1}
        st = g.stats()
        out.update(overflows=st["pool_overflows"] + st["out_overflows"], graph_launches=st["graph_launches"],
                   counters_sum=int(g.channel_counters().astype(np.int64).sum()))
        g.close()
        return out

    if not a.restarts:
        sampler = bench.ClockSampler(torch.cuda.current_device())
        sampler.start()
        t0 = time.time()
        r = run(0, False, a.spans, False)
        r["clocks"] = sampler.stop(t0, time.time())
        print(json.dumps(r))
        return
    res = dict(restarting_receivers=len(some), retuned=sum(1 for r in some if r % 3 == 0), reps=[])
    for i in range(a.repeats):
        plain = run(vd.FLAG_NO_GRAPH, False, a.spans, False)
        rs = run(vd.FLAG_NO_GRAPH, True, a.spans, False)
        res["reps"].append(dict(ordinary_direct_ms_per_span=plain["ms"], restart_10pct_ms_per_span=rs["ms"],
                                overflows=plain["overflows"] + rs["overflows"]))
    res["serialised_kernel_ms_ordinary"] = run(vd.FLAG_NO_GRAPH, False, a.spans, True)["kernel_ms"]
    res["serialised_kernel_ms_restart_10pct"] = run(vd.FLAG_NO_GRAPH, True, a.spans, True)["kernel_ms"]
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--receivers", type=int, default=2048, help="even: half of each rate")
    ap.add_argument("--channels", type=int, default=8, help="channels per receiver")
    ap.add_argument("--n-dec", type=int, default=13107, help="decimated samples of a full span")
    ap.add_argument("--spans", type=int, default=16, help="timed spans per measurement")
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=3, help="alternating repetitions")
    ap.add_argument("--parent", default=None, help="root of another build to compare ordinary spans against")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--restarts", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        return child(a)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_restart_receivers.py needs a CUDA device: the demodulator path has no CPU fallback")
    common = ["--receivers", str(a.receivers), "--channels", str(a.channels), "--n-dec", str(a.n_dec), "--spans", str(a.spans),
              "--warmup", str(a.warmup), "--repeats", str(a.repeats)]

    def sub(root, extra=()):
        env = dict(os.environ, PYTHONPATH=os.path.abspath(root) + os.pathsep + ROOT)
        out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", *common, *extra], env=env, check=True,
                             capture_output=True, text=True).stdout
        return json.loads(out.strip().splitlines()[-1])

    res = dict(gpu=torch.cuda.get_device_name(), receivers=a.receivers, channels_per_receiver=a.channels,
               channels=a.receivers * a.channels, full_span=a.n_dec, timed_spans=a.spans)
    reps = []
    for i in range(a.repeats):                     # (a): the two builds alternate
        mine = sub(ROOT)
        rep = dict(this_build=mine)
        if a.parent:
            other = sub(a.parent)
            rep.update(other_build=other, this_over_other=mine["ms"] / other["ms"], counters_equal=mine["counters_sum"] == other["counters_sum"])
        reps.append(rep)
    res["a_ordinary_ragged_spans"] = reps
    res["b_restart_spans"] = sub(ROOT, ["--restarts"])
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
