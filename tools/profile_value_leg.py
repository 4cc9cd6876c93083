#!/usr/bin/env python3
"""Kernel / stage / host-gap breakdown of one step of bench.py's `value` leg (ASCII genomes resident in HBM:
sk_sketch_batch_dev -> sk_screen_triangle -> sk_chain_pairs on one stream), recorded with torch.profiler (CUDA activities:
CUB and every other library kernel are listed too, not only the SK_LAUNCH ones that sk_ctx_set_timing brackets).

  python tools/profile_value_leg.py [--config north|c2|dense|c5] [--genomes N] [--warmup W] [--steps K] [--out DIR]

Prints, for the profiled step: device time per kernel (grouped by name), per stage the wall time, the device-busy time and
the host gap (wall time the stream had nothing running), host synchronisations (cudaStreamSynchronize calls) per stage,
and the card's name and power limit read in the same run.  `--steps K` also times K unprofiled steps (wall clock, ms).
The chrome trace lands in DIR (default: a temporary directory)."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

CONFIGS = {   # the same workloads as bench.py's configurations of the same names
    "north": dict(genomes=5000, genome_len=5_000_000, cluster=20, c=125, marker_c=1000, rescue_small=True),
    "c2": dict(genomes=1000, genome_len=5_000_000, cluster=20, c=125, marker_c=1000, rescue_small=True),
    "dense": dict(genomes=2000, genome_len=5_000_000, cluster=2000, c=125, marker_c=1000, rescue_small=True),
    "c5": dict(genomes=200000, genome_len=30_000, cluster=10, c=30, marker_c=200, rescue_small=False),
}
STAGES = ("sketch", "screen", "chain")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(int(os.environ.get("LOCAL_RANK", "0"))),
                              "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


def short_name(n):
    """'void cub::...::DeviceRadixSortOnesweepKernel<...>(...)' -> 'cub::DeviceRadixSortOnesweepKernel'"""
    n = re.sub(r"^void ", "", n)
    depth, cut = 0, len(n)
    for i, ch in enumerate(n):
        if ch in "<(" and depth == 0:
            cut = i
            break
    base = n[:cut]
    parts = base.split("::")
    return ("cub::" if base.startswith("cub::") or "cub::" in base else "") + parts[-1] if len(parts) > 1 else base


def union_us(iv):
    """total length of the union of [start, end) intervals"""
    tot, cur_s, cur_e = 0.0, None, None
    for s, e in sorted(iv):
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                tot += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    if cur_e is not None:
        tot += cur_e - cur_s
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="north", choices=sorted(CONFIGS))
    ap.add_argument("--genomes", type=int, default=None)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    cfg = dict(CONFIGS[a.config])
    if a.genomes:
        cfg["genomes"] = a.genomes
    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    import skani_b200 as sk
    from bench_support import synth

    N, L, G = cfg["genomes"], cfg["genome_len"], cfg["cluster"]
    ids = np.arange(N, dtype=np.uint64)
    pinned = torch.empty(N * L, dtype=torch.uint8, pin_memory=True)
    host = pinned.numpy()
    synth.generate_ids(ids, L, G=G, out=host)
    off, goc = synth.layout_ids(ids, L, G)
    dev = pinned.to("cuda")
    ctx = sk.Context(0)
    sp = sk.sketch_params(cfg["c"], 15, cfg["marker_c"])
    mp = sk.map_params(rescue_small=cfg["rescue_small"])

    def step(annotate):
        kept = 0
        t = {}
        for stage in STAGES:
            with record_function("stage:" + stage) if annotate else _null():
                t0 = time.perf_counter()
                if stage == "sketch":
                    gs = sk.sketch_contigs(ctx, None, off, goc, N, sp, device_ptr=dev.data_ptr())
                elif stage == "screen":
                    pairs = sk.screen_triangle(ctx, gs, mp)
                else:
                    res = sk.chain_pairs(ctx, gs, gs, pairs, mp, as_array=True)
                    kept = int((res["ani"] > 0.1).sum())
                    gs.free()
                torch.cuda.synchronize()
                t[stage] = (time.perf_counter() - t0) * 1e3
        return kept, t

    for _ in range(a.warmup):
        step(False)
    walls = []
    for _ in range(a.steps):
        t0 = time.perf_counter()
        kept, _t = step(False)
        walls.append((time.perf_counter() - t0) * 1e3)
    l0 = ctx.launches
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        kept, st_wall = step(True)
    launches = ctx.launches - l0
    out_dir = a.out or tempfile.mkdtemp(prefix="profile_value_leg_")
    os.makedirs(out_dir, exist_ok=True)
    trace = os.path.join(out_dir, "value_leg_%s.json" % a.config)
    prof.export_chrome_trace(trace)
    ev = json.load(open(trace))["traceEvents"]

    ranges = {}
    for e in ev:
        if e.get("ph") == "X" and e.get("cat") == "user_annotation" and e.get("name", "").startswith("stage:"):
            ranges[e["name"][6:]] = (e["ts"], e["ts"] + e["dur"])

    def stage_of(ts):
        for s, (b, en) in ranges.items():
            if b <= ts < en:
                return s
        return "other"

    per_kernel = defaultdict(lambda: [0.0, 0, set()])
    busy = defaultdict(list)
    dev_sum = defaultdict(float)
    syncs = defaultdict(int)
    for e in ev:
        if e.get("ph") != "X":
            continue
        cat = e.get("cat", "")
        if cat in ("kernel", "gpu_memcpy", "gpu_memset"):
            s = stage_of(e["ts"])
            nm = short_name(e["name"]) if cat == "kernel" else cat + ":" + e["name"].split(" ")[0]
            k = per_kernel[nm]
            k[0] += e["dur"]; k[1] += 1; k[2].add(s)
            busy[s].append((e["ts"], e["ts"] + e["dur"]))
            dev_sum[s] += e["dur"]
        elif cat == "cuda_runtime" and e.get("name") in ("cudaStreamSynchronize", "cudaDeviceSynchronize"):
            syncs[stage_of(e["ts"])] += 1

    cardinfo = card()
    step_ms = sum(st_wall.values())
    print("card: %s" % cardinfo)
    print("config %s: %d genomes x %d bp, cluster %d, c=%d, marker_c=%d; kept %d pairs; %d launches (SK_LAUNCH + counted)"
          % (a.config, N, L, G, cfg["c"], cfg["marker_c"], kept, launches))
    print("unprofiled steps (wall ms): %s" % ", ".join("%.1f" % w for w in walls))
    print("profiled step: %.1f ms wall" % step_ms)
    print()
    print("| stage | wall ms | device busy ms | host gap ms | kernel+copy sum ms | host syncs |")
    print("|---|---:|---:|---:|---:|---:|")
    rows = {}
    for s in STAGES:
        b = union_us(busy[s]) / 1e3
        rows[s] = dict(wall_ms=st_wall[s], busy_ms=b, gap_ms=st_wall[s] - b, sum_ms=dev_sum[s] / 1e3, syncs=syncs[s])
        print("| %s | %.1f | %.1f | %.1f | %.1f | %d |" % (s, st_wall[s], b, st_wall[s] - b, dev_sum[s] / 1e3, syncs[s]))
    print()
    print("| kernel / copy | stage | ms | calls | share of step |")
    print("|---|---|---:|---:|---:|")
    items = sorted(per_kernel.items(), key=lambda kv: -kv[1][0])
    for nm, (us, cnt, stg) in items:
        if us / 1e3 < 0.05:
            continue
        print("| `%s` | %s | %.2f | %d | %.1f %% |" % (nm, "+".join(sorted(stg)), us / 1e3, cnt, 100.0 * us / 1e3 / step_ms))
    summary = {"card": cardinfo, "config": a.config, "kept": kept, "launches": launches, "unprofiled_wall_ms": walls,
               "stages": rows, "kernels": {nm: {"ms": us / 1e3, "calls": cnt, "stages": sorted(stg)} for nm, (us, cnt, stg) in items}}
    with open(os.path.join(out_dir, "value_leg_%s.summary.json" % a.config), "w") as f:
        json.dump(summary, f, indent=1)
    ctx.close()
    return 0


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


if __name__ == "__main__":
    sys.exit(main())
