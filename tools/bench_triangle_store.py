#!/usr/bin/env python3
"""The triangle over a host sketch store (sk_triangle_store) against the in-memory triangle (sk_triangle) on bench.py's
synthetic clustered set (default 5,000 x 5 Mbp, clusters of 20, seed 20260924), on ONE GPU.

In-memory leg: sk_triangle from host ASCII (sketch + screen + chain).  Store legs: the genomes are sketched in groups of 500
into a SketchStore (each group's set freed after sk_sketch_store_add), then sk_triangle_store runs with budgets that force
about 4 and about 16 working sets, with one context and with two contexts on the device.  Reported per leg: wall time, the
t_screen / t_gather / t_chain split (gather and chain summed over contexts), gathered GB and GB/s, mean gathers per genome
(gathered bytes / store bytes), kept pairs and bench.py's order-independent checksum, which must equal the in-memory leg's.
A 200-pair oracle spot check runs on the kept pairs, and the card name and power limit are read in the same run.

  python tools/bench_triangle_store.py [--genomes 5000] [--beyond-memory]
--beyond-memory adds 10,000 x 5 Mbp at c = 30 (about 93 GB of sketches, more than one 80 GB device holds): no in-memory leg,
the kept-pair count must be n / 20 * 190 and the oracle spot check must pass.  It needs about 150 GB of host memory and is
skipped with a message when less is available."""
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
    a = ap.parse_args()
    import skani_b200 as sk
    from bench import oracle_spot_check, result_checksum
    from bench_support import synth
    N, L, G = a.genomes, a.genome_len, a.cluster
    out = {"card": card(), "genomes": N, "genome_len": L, "cluster": G, "seed": synth.PRIMARY_SEED}
    cfg = dict(genome_len=L, cluster=G, c=125, marker_c=1000, rescue_small=True)
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
