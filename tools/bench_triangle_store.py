#!/usr/bin/env python3
"""The triangle over a host sketch store (sk_triangle_store) against the in-memory triangle (sk_triangle) on bench.py's
synthetic clustered set (default 5,000 x 5 Mbp, clusters of 20, seed 20260924), on ONE GPU.

In-memory leg: sk_triangle from host ASCII (sketch + screen + chain).  Store legs: the genomes are sketched in groups of 500
into a SketchStore (each group's set freed after sk_sketch_store_add), then sk_triangle_store runs with budgets that force
about 4 and about 16 working sets, with one context and with two contexts on the device.  Reported per leg: wall time, the
t_screen / t_gather / t_chain split (gather and chain summed over contexts), gathered GB and GB/s, mean gathers per genome
(gathered bytes / store bytes), kept pairs and bench.py's order-independent checksum, which must equal the in-memory leg's.
A 200-pair oracle spot check runs on the kept pairs, and the card name and power limit are read in the same run.

  python tools/bench_triangle_store.py [--genomes 5000] [--beyond-memory] [--database]
--beyond-memory adds 10,000 x 5 Mbp at c = 30 (about 93 GB of sketches, more than one 80 GB device holds): no in-memory leg,
the kept-pair count must be n / 20 * 190 and the oracle spot check must pass.  It needs about 150 GB of host memory and is
skipped with a message when less is available.
--database runs the database leg INSTEAD of the legs above: the set is sketched from host ASCII in groups of 500 (timed:
the comparison point of loading a database) and written once as a consolidated skani v0.3.0 database (sketches.db,
index.db, markers.bin) in a temporary directory; then `skani-b200 triangle DB -E` runs on the in-memory path and on the
store path (SK_DEVICE_BUDGET_MB = a quarter of the sketches), and each run's stderr gives the split read + decode /
import / screen + chain, next to the wall time of the process.  The kept-pair count must be n / 20 * 190."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")[:2]]
        return {"name": name, "power_limit": limit}
    except Exception as e:       # noqa: BLE001
        return {"name": None, "power_limit": None, "error": str(e)}


def host_available_gb():
    for ln in open("/proc/meminfo"):
        if ln.startswith("MemAvailable:"):
            return int(ln.split()[1]) / 1e6
    return 0.0


def fill_store(sk, ctx, N, L, G, sp, group=500):
    from bench_support import synth
    t0 = time.perf_counter()
    st = sk.SketchStore(sp)
    for g0 in range(0, N, group):
        g1 = min(N, g0 + group)
        bases, off, goc = synth.generate(g0, g1, L, G=G)
        s = sk.sketch_contigs(ctx, bases, off, goc, g1 - g0, sp)
        st.add(s)
        s.free()
    return st, time.perf_counter() - t0


def db_sketch_bytes(name, e, total_len, c, k, seeds=True):
    """one Sketch (src/types.rs:253-277) in bincode, from SketchSet.export (records sorted by k-mer); seeds=False gives the
    markers-only form of markers.bin.  Contigs are named ctg<i>."""
    u64 = lambda v: np.uint64(v).tobytes()                       # noqa: E731
    nm = name.encode()
    out = [u64(len(nm)), nm]
    kmer, pos, cc = e["kmer"], e["pos"].astype(np.uint64), e["cc"].astype(np.uint64)
    if not seeds:
        out += [b"\x00", u64(0)]
    else:
        n = len(kmer)
        starts = np.flatnonzero(np.r_[True, kmer[1:] != kmer[:-1]]) if n else np.zeros(0, np.int64)
        cnt = np.diff(np.r_[starts, n])
        single = cnt == 1
        vals = np.empty(len(starts), np.uint64)
        vals[single] = (((pos[starts[single]] << np.uint64(31)) | cc[starts[single]]) << np.uint64(1)) | np.uint64(1)
        vals[~single] = np.arange(int((~single).sum()), dtype=np.uint64) << np.uint64(1)
        kv = np.empty(len(starts), [("k", "<u4"), ("v", "<u8")])
        kv["k"], kv["v"] = kmer[starts], vals
        # multi_position_storage: per multi-position k-mer a u64 length, then (pos, contig_index_canonical) u32 pairs
        mc = cnt[~single]
        words = np.zeros(int((2 + 2 * mc).sum()), np.uint32)
        gstart = np.r_[0, np.cumsum(2 + 2 * mc)[:-1]].astype(np.int64)
        words[gstart] = mc
        rec = np.flatnonzero(np.repeat(~single, cnt))        # the records of multi-position k-mers, in group order
        within = rec - np.repeat(starts[~single], mc)
        at = np.repeat(gstart, mc) + 2 + 2 * within
        words[at], words[at + 1] = e["pos"][rec], e["cc"][rec]
        out += [b"\x01", u64(len(starts)), kv.tobytes(), u64(len(mc)), words.tobytes()]
    names = [b"ctg%d" % i for i in range(len(e["contig_lengths"]))]
    out += [u64(len(names))] + [u64(len(cn)) + cn for cn in names]
    cl = e["contig_lengths"] if seeds else np.zeros(0, np.uint32)
    out += [u64(total_len), u64(len(cl)), cl.astype("<u4").tobytes(), u64(0), u64(len(e["markers"])), e["markers"].astype("<u8").tobytes(),
            u64(c), u64(c), u64(k), u64(0), b"\x00\x00"]
    return b"".join(out)


def write_database(sk, ctx, d, N, L, G, sp, group=500):
    """the synthetic set sketched from host ASCII in groups (timed) and written as sketches.db / index.db / markers.bin"""
    import skani_db_py as D
    from bench_support import synth
    par = D.expected_params_bytes(sp.c, sp.k, sp.marker_c)
    index, markers, off, t_sketch = [], [], 0, 0.0
    with open(os.path.join(d, "sketches.db"), "wb") as db:
        for g0 in range(0, N, group):
            g1 = min(N, g0 + group)
            bases, coff, goc = synth.generate(g0, g1, L, G=G)
            t0 = time.perf_counter()
            s = sk.sketch_contigs(ctx, bases, coff, goc, g1 - g0, sp)
            t_sketch += time.perf_counter() - t0
            del bases
            for g in range(g1 - g0):
                e, name = s.export(g), "g%06d" % (g0 + g)
                tl = s.info(g)["total_len"]
                b = par + db_sketch_bytes(name, e, tl, sp.c, sp.k)
                db.write(b)
                index.append((name, off, len(b)))
                off += len(b)
                markers.append(db_sketch_bytes(name, e, tl, sp.c, sp.k, seeds=False))
            s.free()
    u64 = lambda v: np.uint64(v).tobytes()                       # noqa: E731
    with open(os.path.join(d, "index.db"), "wb") as f:
        f.write(u64(len(index)) + b"".join(u64(len(n)) + n.encode() + u64(o) + u64(ln) for n, o, ln in index))
    with open(os.path.join(d, "markers.bin"), "wb") as f:
        f.write(par + u64(len(markers)) + b"".join(markers))
    return t_sketch, off


def cli_triangle_leg(db, out_dir, threads, budget_mb=None):
    """`skani-b200 triangle DB -E` as a process; the split from its INFO lines"""
    import re
    env = {k: v for k, v in os.environ.items() if k not in ("SK_DEVICE_BUDGET_MB", "SK_SKETCH_GROUP_RECORDS")}
    if budget_mb:
        env["SK_DEVICE_BUDGET_MB"] = str(budget_mb)
    out = os.path.join(out_dir, "triangle.tsv")
    t0 = time.perf_counter()
    p = subprocess.run([os.path.join(ROOT, "skani_b200", "skani-b200"), "triangle", db, "-E", "-t", str(threads), "-o", out],
                       capture_output=True, text=True, env=env)
    wall = time.perf_counter() - t0
    if p.returncode != 0:
        return {"error": p.stderr[-2000:]}
    m = re.search(r"INFO (\d+) sketches loaded in (\d+) group\(s\): read \+ decode ([\d.]+) s, import ([\d.]+) s", p.stderr)
    w = re.search(r"INFO Screen \+ chain ([\d.]+) s", p.stderr)
    kept = sum(1 for _ in open(out)) - 1
    os.remove(out)
    return {"store_path": "INFO Store path" in p.stderr, "budget_mb": budget_mb, "wall_s": round(wall, 3), "sketches": int(m.group(1)),
            "groups": int(m.group(2)), "read_decode_s": float(m.group(3)), "import_s": float(m.group(4)),
            "screen_chain_s": float(w.group(1)), "kept_pairs": kept}


def database_leg(sk, ctx, N, L, G, threads):
    import tempfile
    sp = sk.sketch_params()
    with tempfile.TemporaryDirectory() as d:
        db = os.path.join(d, "db")
        os.makedirs(db)
        t0 = time.perf_counter()
        t_sketch, db_bytes = write_database(sk, ctx, db, N, L, G, sp)
        res = {"sketch_from_host_ascii_s": round(t_sketch, 3), "write_s": round(time.perf_counter() - t0, 3),
               "sketches_db_gb": round(db_bytes / 1e9, 3), "threads": threads, "expected_kept": N // G * G * (G - 1) // 2, "legs": []}
        for budget_mb in (None, max(1, int(3 * db_bytes / 4 / 2 ** 20))):
            leg = cli_triangle_leg(db, d, threads, budget_mb)
            leg["kept_ok"] = leg.get("kept_pairs") == res["expected_kept"]
            res["legs"].append(leg)
            print(json.dumps({"database_leg": leg}), file=sys.stderr, flush=True)
    return res


def store_leg(sk, ctxs, st, mp, budget, store_bytes):
    t0 = time.perf_counter()
    res, s = sk.triangle_store(ctxs, st, mp, device_budget=budget)
    wall = time.perf_counter() - t0
    return res, {"contexts": len(ctxs), "budget_gb": round(budget / 1e9, 3), "wall_s": round(wall, 3), "working_sets": s.n_working_sets,
                 "split_components": s.n_split_components, "max_working_set_gb": round(s.max_working_set_bytes / 1e9, 3),
                 "t_screen_s": round(s.t_screen, 3), "t_gather_s": round(s.t_gather, 3), "t_chain_s": round(s.t_chain, 3),
                 "gathered_gb": round(s.gathered_bytes / 1e9, 3), "gather_gb_per_s": round(s.gathered_bytes / 1e9 / max(s.t_gather, 1e-9), 2),
                 "gathers_per_genome": round(s.gathered_bytes / store_bytes, 3), "kept_pairs": int(len(res))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", type=int, default=5000)
    ap.add_argument("--genome-len", type=int, default=5_000_000)
    ap.add_argument("--cluster", type=int, default=20)
    ap.add_argument("--spot-check", type=int, default=200)
    ap.add_argument("--beyond-memory", action="store_true")
    ap.add_argument("--database", action="store_true")
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 8)
    a = ap.parse_args()
    import skani_b200 as sk
    from bench import oracle_spot_check, result_checksum
    from bench_support import synth
    N, L, G = a.genomes, a.genome_len, a.cluster
    out = {"card": card(), "genomes": N, "genome_len": L, "cluster": G, "seed": synth.PRIMARY_SEED}
    cfg = dict(genome_len=L, cluster=G, c=125, marker_c=1000, rescue_small=True)
    if a.database:
        ctx = sk.Context(0)
        out["database"] = database_leg(sk, ctx, N, L, G, a.threads)
        ctx.close()
        print(json.dumps(out))
        return
    ctxs = [sk.Context(0), sk.Context(0)]
    sp, mp = sk.sketch_params(), sk.map_params()
    # ---- in-memory leg
    bases, off, goc = synth.generate(0, N, L, G=G)
    t0 = time.perf_counter()
    want, _ = sk.triangle(ctxs[0], bases, off, goc, N, sp, mp, as_array=True)
    t_mem = time.perf_counter() - t0
    del bases
    want_ck = result_checksum(want)
    out["in_memory"] = {"wall_s": round(t_mem, 3), "kept_pairs": int(len(want)), "checksum": want_ck}
    # ---- store legs
    st, t_fill = fill_store(sk, ctxs[0], N, L, G, sp)
    gb = np.array([st.genome_bytes(g) for g in range(N)], np.uint64)
    total = int(gb.sum())
    out["store"] = {"fill_s": round(t_fill, 3), "store_gb": round(total / 1e9, 3), "legs": []}
    res = None
    for k in (4, 16):
        budget = max(int(total / k * 1.02), int(2 * gb.max()) + 1)
        for n_ctx in (1, 2):
            res, leg = store_leg(sk, ctxs[:n_ctx], st, mp, budget, total)
            leg["target_working_sets"] = k
            leg["checksum"] = result_checksum(res)
            leg["checksum_equals_in_memory"] = bool(leg["checksum"] == want_ck and len(res) == len(want))
            out["store"]["legs"].append(leg)
            print(json.dumps({"leg": leg}), file=sys.stderr, flush=True)
    st.free()
    out["oracle_spot_check"] = oracle_spot_check(res, np.arange(N, dtype=np.uint64), cfg, a.spot_check, 7)
    # ---- beyond one device's memory
    if a.beyond_memory:
        NB, cB = 10_000, 30
        avail = host_available_gb()
        if avail < 150:
            out["beyond_memory"] = {"skipped": "not measured: %.0f GB of host memory available, about 150 GB needed" % avail}
        else:
            spB = sk.sketch_params(c=cB)
            stB, t_fillB = fill_store(sk, ctxs[0], NB, L, G, spB)
            totalB = sum(stB.genome_bytes(g) for g in range(NB))
            resB, legB = store_leg(sk, ctxs, stB, mp, 0, totalB)
            stB.free()
            cfgB = dict(cfg, c=cB)
            legB.update({"genomes": NB, "c": cB, "fill_s": round(t_fillB, 3), "store_gb": round(totalB / 1e9, 3),
                         "expected_kept": NB // G * G * (G - 1) // 2, "checksum": result_checksum(resB),
                         "oracle_spot_check": oracle_spot_check(resB, np.arange(NB, dtype=np.uint64), cfgB, a.spot_check, 7)})
            legB["kept_ok"] = legB["kept_pairs"] == legB["expected_kept"]
            out["beyond_memory"] = legB
    for c in ctxs:
        c.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
