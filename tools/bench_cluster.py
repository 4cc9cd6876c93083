#!/usr/bin/env python3
"""Clustering measurements, printed as JSON lines with the card's name and power limit read in the same call.

1. Library: sk_cluster (skani_b200.cluster, greedy and single linkage) on synthetic graphs of 50,000 genomes in families of
   20 plus random cross edges, at 10^6 and 5 x 10^7 edges (tests/cluster_ref.py), and on a 50,000-genome path ranked along
   the path (the greedy worst case: about one genome decided per round).  One warm-up call per graph and method, then --reps
   timed calls (host clock around the call, which ends in a device synchronise; t_device from the stats).  Next to it, the
   Python/scipy reference of the tests on the CPU, once per graph and method, and the results must agree.
2. Library: sk_cluster_linkage (skani_b200.cluster_linkage, average and complete, cut and dendrogram mode) on the same two
   50,000-genome graphs, where min_ani does not filter the edges (every row is one); then the adversarial cases: a 50,000-
   genome path with ANI decreasing along it, and a 20,000-leaf star in dendrogram mode (one leaf merges per round).  One
   warm-up call, then --reps timed calls.  scipy's linkage of the dense 1 - similarity matrix is the CPU reference where
   n <= 20,000 (the star); its cophenetic distances must agree to 1e-12.
3. End to end: `cluster` against `triangle -E` on a seeded synthetic set (bench_support/synth, clusters of 20; default 1,000
   x 5 Mbp) written as one FASTA file per genome, the two commands alternated --reps times (wall time of the process).

  python tools/bench_cluster.py [--genomes 1000] [--length 5000000] [--reps 3] [--skip-e2e] [--skip-lib] [--skip-linkage]
                                [--only-linkage] [--json OUT]
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


def emit(rec, sink):
    print(json.dumps(rec), flush=True)
    sink.append(rec)


def bench_lib(reps, sink):
    import skani_b200 as sk
    import cluster_ref as R
    ctx = sk.Context(0)
    rng = np.random.default_rng(20261017)
    n = 50_000
    graphs = []
    for target in (1_000_000, 50_000_000):
        inside = (n // 20) * 190
        graphs.append(("families+cross %.0e edges" % target, lambda t=target: R.families(rng, n, 20, t - inside, inside=(0.95, 1.0)), 0.97))
    graphs.append(("path in rank order", lambda: R.path(rng, n), 0.95))
    for name, make, min_ani in graphs:
        t = time.perf_counter()
        g_n, a, b, ani = make()
        res = R.as_results(a, b, ani)
        rank = np.arange(g_n, dtype=np.uint32) if name.startswith("path") else rng.permutation(g_n).astype(np.uint32)
        gen_s = time.perf_counter() - t
        for single in (False, True):
            got = sk.cluster(ctx, g_n, res, rank, min_ani=min_ani, single_linkage=single)      # warm-up (kernels, pinned staging)
            walls, devs = [], []
            for _ in range(reps):
                t = time.perf_counter()
                _, _, _, st = sk.cluster(ctx, g_n, res, rank, min_ani=min_ani, single_linkage=single)
                walls.append(time.perf_counter() - t)
                devs.append(st.t_device)
            t = time.perf_counter()
            exp = R.reference(g_n, res["ref_id"], res["query_id"], res["ani"], min_ani, rank, single)
            cpu = time.perf_counter() - t
            same = all(np.array_equal(x, y) for x, y in zip(got[:3], exp))
            emit({"bench": "sk_cluster", "graph": name, "method": "single linkage" if single else "greedy", "genomes": g_n,
                  "rows": len(res), "edges": int(st.n_edges), "clusters": int(st.n_clusters), "rounds": int(st.rounds),
                  "gpu_call_s": [round(x, 4) for x in walls], "gpu_t_device_s": [round(x, 4) for x in devs],
                  "cpu_reference_s": round(cpu, 3), "equal_to_reference": same, "graph_build_s": round(gen_s, 2)}, sink)
            if not same:
                raise SystemExit("sk_cluster differs from the reference on %s" % name)
        del res, a, b, ani
    ctx.close()


def bench_linkage(reps, sink):
    import skani_b200 as sk
    import cluster_ref as R
    import linkage_ref as LR
    ctx = sk.Context(0)
    rng = np.random.default_rng(20261017)
    n = 50_000
    graphs = []
    for target in (1_000_000, 50_000_000):
        inside = (n // 20) * 190
        graphs.append(("families+cross %.0e edges" % target, lambda t=target: R.families(rng, n, 20, t - inside, inside=(0.95, 1.0)),
                       (False, True)))

    def decreasing_path():
        p = np.stack([np.arange(n - 1), np.arange(1, n)], 1)
        return R._finish(rng, n, p, np.linspace(0.999, 0.9, n - 1).astype(np.float32))

    def star():
        g_n, a, b, ani = R.stars(rng, 20_001, 1)
        return g_n, a, b, LR.tie_free(rng, ani, 0.96, 1.0)
    graphs.append(("path, ANI decreasing along it", decreasing_path, (False, True)))
    graphs.append(("star of 20,000 leaves", star, (True,)))
    for name, make, modes in graphs:
        t = time.perf_counter()
        g_n, a, b, ani = make()
        res = R.as_results(a, b, ani)
        rank = rng.permutation(g_n).astype(np.uint32)
        gen_s = time.perf_counter() - t
        for method in LR.METHODS:
            for dendrogram in modes:
                sk.cluster_linkage(ctx, g_n, res, rank, method=method, min_ani=0.97, dendrogram=dendrogram)      # warm-up
                walls, devs = [], []
                for _ in range(reps):
                    t = time.perf_counter()
                    _, cl, _, Z, st = sk.cluster_linkage(ctx, g_n, res, rank, method=method, min_ani=0.97, dendrogram=dendrogram)
                    walls.append(time.perf_counter() - t)
                    devs.append(st.t_device)
                rec = {"bench": "sk_cluster_linkage", "graph": name, "method": method, "dendrogram": dendrogram, "genomes": g_n,
                       "rows": len(res), "edges": int(st.n_edges), "clusters": int(st.n_clusters), "rounds": int(st.rounds),
                       "gpu_call_s": [round(x, 4) for x in walls], "gpu_t_device_s": [round(x, 4) for x in devs],
                       "graph_build_s": round(gen_s, 2), "cpu_reference_s": "not measured"}
                if dendrogram and g_n <= 20_000:
                    from scipy.cluster.hierarchy import cophenet, linkage
                    from scipy.spatial.distance import squareform
                    D = 1.0 - LR.dense_similarity(g_n, a, b, ani)
                    np.fill_diagonal(D, 0.0)
                    t = time.perf_counter()
                    Zs = linkage(squareform(D, checks=False), method)
                    rec["cpu_reference_s"] = round(time.perf_counter() - t, 3)
                    del D
                    rec["cophenet_max_diff"] = float(np.max(np.abs(cophenet(Z) - cophenet(Zs))))
                    if rec["cophenet_max_diff"] > 1e-12:
                        raise SystemExit("sk_cluster_linkage differs from scipy on %s" % name)
                emit(rec, sink)
        del res, a, b, ani
    ctx.close()


def bench_e2e(n, L, reps, sink):
    d = tempfile.mkdtemp(prefix="bench_cluster_")
    try:
        files = write_fasta(d, n, L)
        lst = os.path.join(d, "list.txt")
        with open(lst, "w") as f:
            f.write("\n".join(files) + "\n")
        cmds = {"triangle -E": ["triangle", "-E", "-l", lst, "-o", os.path.join(d, "tri.tsv")],
                "cluster": ["cluster", "-l", lst, "-o", os.path.join(d, "cl.tsv")]}
        for rep in range(reps):
            for name, args in cmds.items():
                t = time.perf_counter()
                p = subprocess.run([BIN] + args + ["-t", str(min(os.cpu_count() or 1, 32))], capture_output=True, text=True)
                wall = time.perf_counter() - t
                if p.returncode != 0:
                    raise SystemExit("%s failed:\n%s" % (name, p.stderr[-2000:]))
                m = re.search(r"INFO (\d+) genomes in (\d+) clusters .*clustering ([\d.]+) ms", p.stderr)
                rec = {"bench": "end_to_end", "command": name, "rep": rep, "genomes": n, "length": L, "wall_s": round(wall, 3)}
                if m:
                    rec.update(clusters=int(m.group(2)), clustering_ms=float(m.group(3)))
                emit(rec, sink)
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", type=int, default=1000)
    ap.add_argument("--length", type=int, default=5_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--skip-lib", action="store_true")
    ap.add_argument("--skip-linkage", action="store_true")
    ap.add_argument("--only-linkage", action="store_true")
    ap.add_argument("--json")
    a = ap.parse_args()
    sink = []
    emit({"card": card()}, sink)
    if not a.skip_lib and not a.only_linkage:
        bench_lib(a.reps, sink)
    if not a.skip_linkage:
        bench_linkage(a.reps, sink)
    if not a.skip_e2e and not a.only_linkage:
        bench_e2e(a.genomes, a.length, a.reps, sink)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(sink, f, indent=1)


if __name__ == "__main__":
    main()
