#!/usr/bin/env python
"""A/B timing of the kernel variants on the bench workload (one GPU): per-kernel launch durations with the stream
overlap off, and the pipelined period per chunk with it on, for both channel orders.

    python tools/variant_sweep.py [--channels 16384] [--chunks 48] > variant_sweep.json
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


def run(env, order, channels, n_run, d_chunks, offs, flags=0):
    old = {k: os.environ.get(k) for k in env}
    for k, v in env.items():
        os.environ[k] = str(v)
    try:
        freqs = bench.channel_freqs(offs, channels, order)
        stream = torch.cuda.current_stream()
        out = {}
        # serial: per-kernel durations
        g = vd.Vdl2Channels(bench.FS, 20, vd.FMT_U8, bench.CENTER, freqs, max_chunk_bytes=bench.CHUNK_BYTES, flags=flags | vd.FLAG_NO_OVERLAP)
        n = d_chunks.shape[0]
        for i in range(8):
            g.submit_device(d_chunks[i % n].data_ptr(), bench.CHUNK_BYTES, stream.cuda_stream)
        g.flush_count()
        g.enable_timing(True)
        k0 = g.kernel_ms()
        for i in range(n_run):
            g.submit_device(d_chunks[i % n].data_ptr(), bench.CHUNK_BYTES, stream.cuda_stream)
            g.poll_count()
        g.flush_count()
        k1 = g.kernel_ms()
        out["kernel_ms"] = {k: round((k1[k][0] - k0[k][0]) / max(k1[k][1] - k0[k][1], 1), 4) for k in k1}
        g.close()
        # pipelined
        g = vd.Vdl2Channels(bench.FS, 20, vd.FMT_U8, bench.CENTER, freqs, max_chunk_bytes=bench.CHUNK_BYTES, flags=flags)
        for i in range(16):
            g.submit_device(d_chunks[i % n].data_ptr(), bench.CHUNK_BYTES, stream.cuda_stream)
        g.flush_count()
        if os.environ.get("VDL2GPU_SWEEP_TIMELINE"):
            g.enable_timing(True)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        t0 = time.perf_counter()
        frames = 0
        for i in range(2 * n_run):
            g.submit_device(d_chunks[i % n].data_ptr(), bench.CHUNK_BYTES, stream.cuda_stream)
            frames += g.poll_count()
        t_host = time.perf_counter() - t0
        frames += g.flush_count()
        g.stream_wait(stream.cuda_stream)
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / (2 * n_run)
        st = g.stats()
        if os.environ.get("VDL2GPU_SWEEP_TIMELINE"):
            tl = g.timeline()
            if len(tl) > 24:
                rows = tl[16:24]
                out["timeline_ms"] = [[round(float(x - rows[0][1]), 3) for x in r[1:]] for r in rows]
        out.update(pipelined_ms_per_chunk=round(ms, 4), g_chsamples_per_s=round(channels * bench.CHUNK_PAIRS / ms / 1e6, 1),
                   frames=frames, host_us_per_chunk=round(t_host / (2 * n_run) * 1e6, 1), graph_launches=st["graph_launches"],
                   overflows=st["pool_overflows"] + st["out_overflows"])
        g.close()
        return out
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=16384)
    ap.add_argument("--chunks", type=int, default=48)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    chunks, offs, _ = bench.make_stream(4.0)
    d_chunks = torch.from_numpy(chunks).cuda()
    variants = [("default", {}, 0), ("no_graph", {}, vd.FLAG_NO_GRAPH), ("k2a_libm", dict(VDL2GPU_K2A=0), 0),
                ("k2_plane", dict(VDL2GPU_K2_VARIANT=2), 0), ("k2_ring_cpasync", dict(VDL2GPU_K2_VARIANT=4), 0),
                ("k2_ring_staged", dict(VDL2GPU_K2_VARIANT=5), 0), ("k1_one_warp", dict(VDL2GPU_K1_VARIANT=8), 0),
                ("k2_staged_1warp", dict(VDL2GPU_K2_VARIANT=261), 0), ("k2_plane_1warp", dict(VDL2GPU_K2_VARIANT=258), 0),
                ("all_1warp", dict(VDL2GPU_K2_VARIANT=261, VDL2GPU_K1_VARIANT=8), 0),
                ("split8", dict(VDL2GPU_K2A_SPLIT=8), 0), ("split16", dict(VDL2GPU_K2A_SPLIT=16), 0), ("split32", dict(VDL2GPU_K2A_SPLIT=32), 0),
                ("split64", dict(VDL2GPU_K2A_SPLIT=64), 0), ("stages3", dict(VDL2GPU_STAGES=3), 0),
                ("default_again", {}, 0), ("no_graph_again", {}, vd.FLAG_NO_GRAPH)]
    extra = os.environ.get("VDL2GPU_SWEEP_EXTRA")          # "name:KEY=V,KEY=V;name2:..."
    if extra:
        for item in extra.split(";"):
            name, kv = item.split(":")
            variants.append((name, dict(x.split("=") for x in kv.split(",") if x), 0))
    res = {}
    for name, env, flags in variants:
        if args.only and name not in args.only.split(","):
            continue
        for order in ("interleaved", "replica"):
            try:
                res[f"{name}/{order}"] = run(env, order, args.channels, args.chunks, d_chunks, offs, flags)
            except Exception as e:      # noqa: BLE001
                res[f"{name}/{order}"] = dict(error=str(e))
            print(f"{name}/{order}: {res[f'{name}/{order}']}", file=sys.stderr, flush=True)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
