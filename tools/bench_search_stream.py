#!/usr/bin/env python3
"""`search` over query groups: a synthetic database and a few hundred synthetic query files, searched by the CLI with the
default groups and with small groups (SK_SKETCH_GROUP_FILES), whose outputs must be equal; and, through the C ABI, the marker
screen of the same queries as one sk_screen_query_ref call against sk_ref_index_screen over k groups.  Prints one JSON line
with wall times, the peak resident set of each CLI child, the screen times, and the card name and power limit read in the
same run.

  python tools/bench_search_stream.py [--refs 400] [--queries 300] [--genome-len 1000000] [--groups 8]

Synthetic data: clusters of 24 genomes (bench_support/synth); the database holds members 0..19 of every cluster, each query
file is one of members 20..23 of a random cluster, written as FASTA into a temporary directory that is removed afterwards."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")


def write_fasta(path, name, seq):
    with open(path, "wb") as f:
        f.write(b">" + name.encode() + b"\n")
        for i in range(0, len(seq), 80):
            f.write(seq[i:i + 80].tobytes() + b"\n")


def card():
    """(name, power limit) of GPU 0"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as e:   # noqa: BLE001 - reported, not hidden
        return "unknown (%s)" % e, "unknown"


def run_cli(args, env, tmp):
    """(stdout, stderr, wall seconds, peak resident set in MB) of one CLI run; the child is reaped with wait4 for its own rusage"""
    o, e = os.path.join(tmp, "stdout"), os.path.join(tmp, "stderr")
    with open(o, "wb") as fo, open(e, "wb") as fe:
        t0 = time.perf_counter()
        p = subprocess.Popen([BIN] + args, stdout=fo, stderr=fe, env=dict(os.environ, **env))
        _, status, ru = os.wait4(p.pid, 0)
        wall = time.perf_counter() - t0
    out, err = open(o, "rb").read(), open(e).read()
    if os.waitstatus_to_exitcode(status) != 0:
        raise RuntimeError("skani-b200 %s failed:\n%s" % (" ".join(args[:4]), err[-2000:]))
    return out, err, wall, ru.ru_maxrss / 1024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--refs", type=int, default=400)
    ap.add_argument("--queries", type=int, default=300)
    ap.add_argument("--genome-len", type=int, default=1_000_000)
    ap.add_argument("--groups", type=int, default=8, help="query groups of the small-group runs and of the C ABI comparison")
    ap.add_argument("--out", default=None, help="write the JSON line here too")
    a = ap.parse_args()
    import skani_b200 as sk
    from bench_support import synth
    G, GD, L = 24, 20, a.genome_len
    n_clusters = max(a.refs // GD, 1)
    n_ref = n_clusters * GD
    ref_ids = (np.arange(n_ref) // GD * G + np.arange(n_ref) % GD).astype(np.uint64)
    rng = np.random.default_rng(2026)
    q_ids = (rng.integers(0, n_clusters, a.queries) * G + GD + rng.integers(0, G - GD, a.queries)).astype(np.uint64)
    name, power = card()
    tmp = tempfile.mkdtemp(prefix="bench_search_stream_")
    try:
        # ---- inputs: one FASTA file per genome
        rb, roff, _ = synth.generate_ids(ref_ids, L, G=G)
        qb, qoff, _ = synth.generate_ids(q_ids, L, G=G)
        rfiles, qfiles = [], []
        for i in range(n_ref):
            rfiles.append(os.path.join(tmp, "r%06d.fa" % i))
            write_fasta(rfiles[-1], "ref%d" % i, rb[i * L:(i + 1) * L])
        for i in range(a.queries):
            qfiles.append(os.path.join(tmp, "q%06d.fa" % i))
            write_fasta(qfiles[-1], "query%d" % i, qb[i * L:(i + 1) * L])
        db = os.path.join(tmp, "db")
        t0 = time.perf_counter()
        run_cli(["sketch"] + rfiles + ["-o", db, "-t", "8"], {}, tmp)
        t_db = time.perf_counter() - t0
        # ---- CLI: default groups (one here) against small groups; the RSS is each child's own peak (wait4)
        per_group = -(-a.queries // max(a.groups, 1))
        runs = {}
        for label, env in (("default", {}), ("small_groups", {"SK_SKETCH_GROUP_FILES": str(per_group)})):
            out, err, wall, rss = run_cli(["search", "-d", db, "-t", "8"] + qfiles, env, tmp)
            runs[label] = dict(out=out, wall_s=round(wall, 3), peak_rss_mb=round(rss, 1),
                               groups=sum(ln.startswith("INFO Query group ") for ln in err.splitlines()),
                               rows=out.count(b"\n") - 1)
        equal = runs["default"]["out"] == runs["small_groups"]["out"]
        for r in runs.values():
            del r["out"]
        # ---- C ABI: one sk_screen_query_ref call against the index screened over k groups, same queries
        ctx = sk.Context(0)
        sp = sk.sketch_params()
        mp = sk.map_params(rescue_small=False)
        _, rgoc = synth.layout_ids(ref_ids, L, G)
        _, qgoc = synth.layout_ids(q_ids, L, G)
        rset = sk.sketch_contigs(ctx, rb, roff, rgoc, n_ref, sp)
        qset = sk.sketch_contigs(ctx, qb, qoff, qgoc, a.queries, sp)
        bounds = [a.queries * k // a.groups for k in range(a.groups + 1)]
        qgroups = []
        for k in range(a.groups):
            g0, g1 = bounds[k], bounds[k + 1]
            c0, c1 = np.searchsorted(qgoc, g0), np.searchsorted(qgoc, g1)
            o = qoff[c0:c1 + 1]
            qgroups.append((g0, sk.sketch_contigs(ctx, qb[int(o[0]):int(o[-1])], o - o[0], qgoc[c0:c1] - g0, g1 - g0, sp)))
        sk.screen_query_ref(ctx, rset, qset, mp, 1)            # warm-up of every kernel and of the arena
        t0 = time.perf_counter()
        one = sk.screen_query_ref(ctx, rset, qset, mp, 1)
        t_one = time.perf_counter() - t0
        t0 = time.perf_counter()
        idx = sk.RefIndex(ctx, rset)
        t_create = time.perf_counter() - t0
        idx.screen(qgroups[0][1], mp, 1)                      # warm-up
        t0 = time.perf_counter()
        parts = []
        for g0, s in qgroups:
            p = idx.screen(s, mp, 1)
            parts.append((p & ~np.uint64(0xFFFFFFFF)) | ((p & np.uint64(0xFFFFFFFF)) + np.uint64(g0)))
        t_groups = time.perf_counter() - t0
        grouped = np.sort(np.concatenate(parts))
        _, n_parts, idx_bytes = idx.info()
        abi_equal = bool(np.array_equal(grouped, one))
        idx.free()
        ctx.close()
        line = {"card": name, "power_limit": power, "refs": n_ref, "queries": a.queries, "genome_len": L, "db_sketch_s": round(t_db, 2),
                "cli": runs, "cli_outputs_equal": bool(equal),
                "abi": {"groups": a.groups, "pairs": int(len(one)), "screen_query_ref_s": round(t_one, 4), "ref_index_create_s": round(t_create, 4),
                        "ref_index_screen_groups_s": round(t_groups, 4), "index_parts": n_parts, "index_mb": round(idx_bytes / 1e6, 1),
                        "pairs_equal": abi_equal}}
        print(json.dumps(line))
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                f.write(json.dumps(line) + "\n")
        if not (equal and abi_equal):
            sys.exit(1)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
