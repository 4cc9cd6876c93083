#!/usr/bin/env python3
"""BASELINE.json configs[2] shape (`skani search`: many query genomes against a large pre-sketched database) on ONE H100,
through the C ABI.  The database is sketched once (outside the timed region, as a pre-sketched `sketches.db` would be) and
kept resident in HBM; a timed step = sketch the query genomes from host memory -> marker screen of every (query, ref) pair
(check_markers_quickly without rescue, the `search` default, src/search.rs:127) -> chain the passing pairs -> keep ani > 0.5
(src/search.rs:174).  Prints one JSON line in bench.py's shape; a sample of kept pairs is re-chained by the CPU oracle.

  python tools/bench_search.py [--refs 6500] [--queries 1000] [--steps 3] [--warmup 1]
Default = 1/10 of configs[2] on both axes (65 000 x 10 000 needs ~150 GB of resident sketches + tables; --refs scales it).
Synthetic data: clusters of 24 genomes (bench_support/synth); the database holds members 0..19 of every cluster, the queries
are members 20..23 of random clusters (fresh genomes related to 20 database entries each)."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--refs", type=int, default=6500)
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--genome-len", type=int, default=5_000_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--spot-check", type=int, default=100)
    a = ap.parse_args()
    import torch
    import skani_b200 as sk
    import oracle_py as O
    from bench_support import synth
    G, GD, L = 24, 20, a.genome_len
    n_clusters = a.refs // GD
    n_ref = n_clusters * GD
    ref_ids = (np.arange(n_ref) // GD * G + np.arange(n_ref) % GD).astype(np.uint64)
    rng = np.random.default_rng(2026)
    q_ids = (rng.integers(0, n_clusters, a.queries) * G + GD + rng.integers(0, G - GD, a.queries)).astype(np.uint64)
    ctx = sk.Context(0)
    sp = sk.sketch_params()
    mp = sk.map_params(rescue_small=False, min_af=-1.0)     # search: --min-af unset -> 15 % (src/chain.rs:101-107)
    # ---- database: sketched in chunks, appended into one resident set (not timed: it stands for a pre-sketched sketches.db)
    t0 = time.perf_counter()
    db = None
    chunk = 400
    for b in range(0, n_ref, chunk):
        ids = ref_ids[b:b + chunk]
        bases, off, goc = synth.generate_ids(ids, L, G=G)
        part = sk.sketch_contigs(ctx, bases, off, goc, len(ids), sp)
        if db is None:
            db = part
        else:
            db.append(part)
            part.free()
    t_db = time.perf_counter() - t0
    # ---- queries in pinned host memory
    pinned = torch.empty(a.queries * L, dtype=torch.uint8, pin_memory=True)
    qh = pinned.numpy()
    synth.generate_ids(q_ids, L, G=G, out=qh)
    qoff, qgoc = synth.layout_ids(q_ids, L, G)
    stream = torch.cuda.ExternalStream(ctx.stream)
    out = {}

    def step():
        qs = sk.sketch_contigs(ctx, qh, qoff, qgoc, a.queries, sp)
        pairs = sk.screen_query_ref(ctx, db, qs, mp, mode=1)
        res = sk.chain_pairs(ctx, db, qs, pairs, mp, as_array=True)
        res = res[res["ani"] > 0.5]
        qs.free()
        out["pairs"], out["res"] = len(pairs), res

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    l0 = ctx.launches
    t0 = time.perf_counter()
    ev0.record(stream)
    for _ in range(a.steps):
        step()
    ev1.record(stream)
    torch.cuda.synchronize()
    ms = max(ev0.elapsed_time(ev1), (time.perf_counter() - t0) * 1e3) / a.steps
    launches = ctx.launches - l0
    res = out["res"]
    # ---- oracle spot check
    worst, n_chk = 0.0, 0
    if a.spot_check and len(res):
        pick = res[np.sort(np.random.default_rng(5).choice(len(res), min(a.spot_check, len(res)), replace=False))]
        rs, qsl = np.unique(pick["ref_id"]), np.unique(pick["query_id"])
        rb, roff, rgoc = synth.generate_ids(ref_ids[rs], L, G=G)
        qb, qo, qg = synth.generate_ids(q_ids[qsl], L, G=G)
        thr = len(os.sched_getaffinity(0))
        # file-name order for switch_qr ties: refs rank before queries (two different sets, include/skani_b200.h)
        ro = O.sketch_many(rb, roff, rgoc, len(rs), threads=thr)
        qo_ = O.sketch_many(qb, qo, qg, len(qsl), threads=thr)
        for r in pick:
            o = O.chain(ro[int(np.searchsorted(rs, r["ref_id"]))], qo_[int(np.searchsorted(qsl, r["query_id"]))], O.cmd(rescue_small=False, min_af=-1.0))
            for f in ("ani", "af_ref", "af_query"):
                worst = max(worst, abs(float(r[f]) - float(getattr(o, f))))
            n_chk += 1
    tot = a.queries * n_ref
    line = {"metric": "query-ref genome pairs/sec, skani search %d queries x %d-genome resident DB (BASELINE.json configs[2] shape)" % (a.queries, n_ref),
            "value": tot / (ms * 1e-3), "unit": "genome-pairs/s", "n_gpus": 1, "steps": a.steps, "warmup": a.warmup, "ms_per_step": ms,
            "higher_is_better": True, "dtype": "u64", "data": "synthetic",
            "config": {"workload": "search: %d x %d bp queries (host, pinned) vs %d resident reference sketches; clusters of 24, DB = members 0-19" % (a.queries, L, n_ref),
                       "screened_pairs_passing": out["pairs"], "kept_pairs": int(len(res)), "expected_kept": int(a.queries * GD),
                       "db_sketch_s": round(t_db, 1),
                       "oracle_spot_check": {"pairs": n_chk, "max_abs_diff": worst, "ok": bool(worst <= 1e-4)}},
            "e2e": {"value": tot / (ms * 1e-3), "unit": "genome-pairs/s", "h2d_bytes_per_step": int(a.queries * L * (1 - 0.75 * ctx.last_pack_share)),
                    "d2h_bytes_per_step": int(len(res) * 72), "host_pack_share": round(ctx.last_pack_share, 3)},
            "chained_pairs_per_s": out["pairs"] / (ms * 1e-3), "gpu_launches": int(launches)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
