#!/usr/bin/env python3
"""Neighbour-joining measurements, printed as JSON lines with the card's name and power limit read in the same call.

1. Library: sk_neighbor_joining (skani_b200.neighbor_joining) on synthetic sparse graphs from tests/cluster_ref.py (families
   of 20 plus random cross edges, 10 edges per genome) at --sizes genomes (default 5 000, 10 000 and 20 000).  One warm-up
   call per graph, then --reps timed calls (host clock around the call, which ends in a device synchronise; t_device from
   the stats).  Next to each time: the bytes the scan has to read, the sum over the steps of the pairs of the square it scans
   (the live nodes' square, compacted to at most 4/3 of them) times 8 B, and that over the call's time.  At n <= 1 500 the
   CPU reference of the tests (tests/nj_ref.py) runs once and its join table must be equal bit for bit.  With --gpus N > 1
   each rep also times sk_neighbor_joining_multi (skani_b200.neighbor_joining_multi) on N contexts, context d on device
   d % the visible devices (so contexts share a device when fewer are visible), alternating with the one-context call; its
   join table must equal the one-context table byte for byte.
2. End to end: `tree` against `triangle --full-matrix --distance` on a seeded synthetic set (bench_support/synth, the set
   tools/bench_cluster.py uses; default 1 000 x 5 Mbp) written as one FASTA file per genome, the two commands alternated
   --reps times (wall time of the process).

  python tools/bench_tree.py [--sizes 1500,5000,10000,20000] [--reps 2] [--gpus 1] [--genomes 1000] [--length 5000000]
                             [--skip-e2e] [--skip-lib] [--json OUT]
The FASTA files go to a temporary directory that is removed at the end."""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")

from bench_sketch import card, write_fasta   # noqa: E402

TILE = 64


def scan_bytes(n):
    """sum over the steps of the scanned square's pairs x 8 B, with nj.cu's compaction schedule (m <= 3/4 of the square's
    dimension, while the square is more than one tile)"""
    total, S = 0, n
    for t in range(max(n - 2, 0)):
        m = n - t
        if S > TILE and 4 * m <= 3 * S:
            S = m
        total += S * (S - 1) // 2 * 8
    return total


def emit(rec, sink):
    print(json.dumps(rec), flush=True)
    sink.append(rec)


def bench_lib(sizes, reps, gpus, sink):
    import skani_b200 as sk
    import cluster_ref as R
    import nj_ref as N
    ctx = sk.Context(0)
    ndev = max(ctx.L.sk_device_count(), 1)
    devs = [d % ndev for d in range(gpus)]
    ctxs = [ctx] + [sk.Context(dev) for dev in devs[1:]]
    rng = np.random.default_rng(20261017)
    for n in sizes:
        g_n, a, b, ani = R.families(rng, n, 20, 10 * n - (n // 20) * 190, inside=(0.95, 1.0))
        res = R.as_results(a, b, ani)
        calls = {1: lambda: sk.neighbor_joining(ctx, g_n, res)}
        if gpus > 1:
            calls[gpus] = lambda: sk.neighbor_joining_multi(ctxs, g_n, res)
        base, _ = calls[1]()     # warm-up
        for call in list(calls.values())[1:]:
            call()
        nbytes = scan_bytes(g_n)
        for rep in range(reps):
            for k, call in calls.items():
                t = time.perf_counter()
                joins, st = call()
                wall = time.perf_counter() - t
                assert joins.tobytes() == base.tobytes()
                emit({"bench": "nj", "genomes": g_n, "rows": len(res), "contexts": k, "devices": len(set(devs[:k])),
                      "rep": rep, "wall_s": round(wall, 4), "t_device_s": round(st.t_device, 4), "compactions": st.compactions,
                      "scan_bytes": nbytes, "scan_GB_per_s": round(nbytes / wall / 1e9, 1)}, sink)
        if g_n <= 1500:
            t = time.perf_counter()
            want = N.nj_results(g_n, a, b, ani)
            emit({"bench": "nj_cpu_reference", "genomes": g_n, "wall_s": round(time.perf_counter() - t, 3),
                  "equal": want.tobytes() == base.tobytes()}, sink)
            if want.tobytes() != base.tobytes():
                raise SystemExit("the GPU join table differs from the CPU reference at n = %d" % g_n)
    for c in ctxs:
        c.close()


def bench_e2e(n, L, reps, sink):
    d = tempfile.mkdtemp(prefix="bench_tree_")
    try:
        files = write_fasta(d, n, L)
        lst = os.path.join(d, "list.txt")
        with open(lst, "w") as f:
            f.write("\n".join(files) + "\n")
        cmds = {"triangle --full-matrix --distance": ["triangle", "--full-matrix", "--distance", "-l", lst, "-o", os.path.join(d, "tri.txt")],
                "tree": ["tree", "-l", lst, "-o", os.path.join(d, "tree.nwk")]}
        for rep in range(reps):
            for name, args in cmds.items():
                t = time.perf_counter()
                p = subprocess.run([BIN] + args + ["-t", str(min(os.cpu_count() or 1, 32))], capture_output=True, text=True)
                wall = time.perf_counter() - t
                if p.returncode != 0:
                    raise SystemExit("%s failed:\n%s" % (name, p.stderr[-2000:]))
                rec = {"bench": "end_to_end", "command": name, "rep": rep, "genomes": n, "length": L, "wall_s": round(wall, 3)}
                m = re.search(r"INFO (\d+) genomes, tree by nj \((\d+) compactions\), ([\d.]+) ms", p.stderr)
                if m:
                    rec.update(compactions=int(m.group(2)), tree_ms=float(m.group(3)))
                emit(rec, sink)
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1500,5000,10000,20000")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--genomes", type=int, default=1000)
    ap.add_argument("--length", type=int, default=5_000_000)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--skip-lib", action="store_true")
    ap.add_argument("--json")
    a = ap.parse_args()
    sink = []
    emit({"card": card()}, sink)
    if not a.skip_lib:
        bench_lib([int(x) for x in a.sizes.split(",")], a.reps, a.gpus, sink)
    if not a.skip_e2e:
        bench_e2e(a.genomes, a.length, a.reps, sink)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(sink, f, indent=1)


if __name__ == "__main__":
    main()
