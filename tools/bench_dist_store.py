#!/usr/bin/env python3
"""dist over host sketch stores (sk_query_ref_store) against the in-memory dist (sk_screen_query_ref + sk_chain_pairs) on
bench.py's synthetic clustered genomes (seed 20260924), on ONE GPU.  Default: 5,000 x 5 Mbp in clusters of 25; genomes
g % 25 in {0, 5, 10, 15, 20} are the 1,000 queries, the other 4,000 the references, so every query passes the screen for
about 20 references of its cluster.

In-memory leg: both sides sketched, sk_screen_query_ref in mode 2 (dist with the marker index), sk_chain_pairs, keep
ani > 0.1.  Store legs: both sides sketched in groups of 500 into one SketchStore each (each group's set freed after
sk_sketch_store_add), then sk_query_ref_store in mode 2 with budgets that force about 4 and about 16 working sets, with one
context and with two contexts on the device.  Reported per leg: wall time, the t_screen / t_gather / t_chain split (gather
and chain summed over contexts), gathered GB and GB/s, mean gathers per reference and per query genome (from the SK_TRACE
working-set lines), kept pairs and bench.py's order-independent checksum, which must equal the in-memory leg's.  A 200-pair
oracle spot check runs on the kept pairs, and the card name and power limit are read in the same run.

  python tools/bench_dist_store.py [--refs 4000] [--queries 1000]"""
import argparse
import json
import os
import re
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_triangle_store import card  # noqa: E402


def sketch_ids(sk, ctx, ids, L, G, sp, ranks):
    from bench_support import synth
    bases, off, goc = synth.generate_ids(ids, L, G=G)
    s = sk.sketch_contigs(ctx, bases, off, goc, len(ids), sp)
    s.set_name_ranks(ranks)
    return s


def fill_store(sk, ctx, ids, L, G, sp, group=500):
    st = sk.SketchStore(sp)
    for g0 in range(0, len(ids), group):
        s = sketch_ids(sk, ctx, ids[g0:g0 + group], L, G, sp, ids[g0:g0 + group])
        st.add(s)
        s.free()
    st.set_name_ranks(ids)           # both sides ranked by global genome id: one file-name order
    return st


def traced(fn):
    """fn() with SK_TRACE=1 and the process's stderr captured; returns (fn's value, the captured text)."""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+b") as f:
        os.dup2(f.fileno(), 2)
        os.environ["SK_TRACE"] = "1"
        try:
            v = fn()
        finally:
            del os.environ["SK_TRACE"]
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        return v, f.read().decode(errors="replace")


def store_leg(sk, ctxs, rs, qs, mp, budget, NR, NQ):
    t0 = time.perf_counter()
    (res, s), trace = traced(lambda: sk.query_ref_store(ctxs, rs, qs, mp, mode=2, device_budget=budget))
    wall = time.perf_counter() - t0
    sets = re.findall(r"\[sk_query_ref_store\].*: (\d+) references, (\d+) queries, (\d+) pairs", trace)
    assert len(sets) == s.n_working_sets, trace[-2000:]
    return res, {"contexts": len(ctxs), "budget_gb": round(budget / 1e9, 3), "wall_s": round(wall, 3), "working_sets": s.n_working_sets,
                 "split_components": s.n_split_components, "max_working_set_gb": round(s.max_working_set_bytes / 1e9, 3),
                 "t_screen_s": round(s.t_screen, 3), "t_gather_s": round(s.t_gather, 3), "t_chain_s": round(s.t_chain, 3),
                 "gathered_gb": round(s.gathered_bytes / 1e9, 3), "gather_gb_per_s": round(s.gathered_bytes / 1e9 / max(s.t_gather, 1e-9), 2),
                 "gathers_per_ref": round(sum(int(x[0]) for x in sets) / NR, 3), "gathers_per_query": round(sum(int(x[1]) for x in sets) / NQ, 3),
                 "kept_pairs": int(len(res))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--refs", type=int, default=4000)
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--genome-len", type=int, default=5_000_000)
    ap.add_argument("--spot-check", type=int, default=200)
    a = ap.parse_args()
    import skani_b200 as sk
    from bench import oracle_spot_check, result_checksum
    from bench_support import synth
    N, L = a.refs + a.queries, a.genome_len
    G = 25
    per = G * a.queries // N                       # queries per cluster
    is_q = np.array([(g % G) % (G // per) == 0 and (g % G) // (G // per) < per for g in range(N)])
    qid, rid = np.nonzero(is_q)[0].astype(np.uint64), np.nonzero(~is_q)[0].astype(np.uint64)
    NR, NQ = len(rid), len(qid)
    out = {"card": card(), "refs": NR, "queries": NQ, "genome_len": L, "cluster": G, "seed": synth.PRIMARY_SEED,
           "not_measured": ["several GPUs (--gpus N): one GPU here", "a reference set beyond one device's memory (needs a matching amount of pinned host memory)"]}
    cfg = dict(genome_len=L, cluster=G, c=125, marker_c=1000, rescue_small=True)
    ctxs = [sk.Context(0), sk.Context(0)]
    sp, mp = sk.sketch_params(), sk.map_params()
    # ---- in-memory leg
    t0 = time.perf_counter()
    R = sketch_ids(sk, ctxs[0], rid, L, G, sp, rid)
    Q = sketch_ids(sk, ctxs[0], qid, L, G, sp, qid)
    t_sketch = time.perf_counter() - t0
    t0 = time.perf_counter()
    pairs = sk.screen_query_ref(ctxs[0], R, Q, mp, mode=2)
    want = sk.chain_pairs(ctxs[0], R, Q, pairs, mp, as_array=True)
    want = want[want["ani"] > np.float32(0.1)]
    t_mem = time.perf_counter() - t0
    R.free(); Q.free()
    want_ck = result_checksum(want)
    out["in_memory"] = {"sketch_s": round(t_sketch, 3), "screen_chain_s": round(t_mem, 3), "screened_pairs": int(len(pairs)),
                        "kept_pairs": int(len(want)), "checksum": want_ck}
    # ---- store legs
    t0 = time.perf_counter()
    rs = fill_store(sk, ctxs[0], rid, L, G, sp)
    qs = fill_store(sk, ctxs[0], qid, L, G, sp)
    t_fill = time.perf_counter() - t0
    rb = np.array([rs.genome_bytes(g) for g in range(NR)], np.uint64)
    qb = np.array([qs.genome_bytes(g) for g in range(NQ)], np.uint64)
    total = int(rb.sum() + qb.sum())
    out["store"] = {"fill_s": round(t_fill, 3), "store_gb": round(total / 1e9, 3), "legs": []}
    res = None
    for k in (4, 16):
        budget = max(int(total / k * 1.02), int(2 * max(rb.max(), qb.max())) + 1)
        for n_ctx in (1, 2):
            res, leg = store_leg(sk, ctxs[:n_ctx], rs, qs, mp, budget, NR, NQ)
            leg["target_working_sets"] = k
            leg["checksum"] = result_checksum(res)
            leg["checksum_equals_in_memory"] = bool(leg["checksum"] == want_ck and len(res) == len(want))
            out["store"]["legs"].append(leg)
            print(json.dumps({"leg": leg}), file=sys.stderr, flush=True)
    rs.free(); qs.free()
    glob = res.copy()                              # store ids -> global genome ids for the oracle
    glob["ref_id"] = rid[res["ref_id"]].astype(np.uint32)
    glob["query_id"] = qid[res["query_id"]].astype(np.uint32)
    out["oracle_spot_check"] = oracle_spot_check(glob, np.arange(N, dtype=np.uint64), cfg, a.spot_check, 7)
    for c in ctxs:
        c.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
