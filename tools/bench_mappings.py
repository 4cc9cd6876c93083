#!/usr/bin/env python3
"""Cost of mappings: sk_chain_pairs against sk_chain_pairs_mappings on the same screened pairs of a bench-like synthetic set
(bench_support/synth families of --family genomes of --length bases), printed as one JSON line with the card's name and
power limit read in the same call.  One warm-up call of each, then --reps calls of each alternated (host clock around calls
that end in a device synchronise).  out must be byte-identical between the two.  Reports the median time of each, the
records per pair and the bytes of records copied to the host.

  python tools/bench_mappings.py [--genomes 400] [--length 1000000] [--family 20] [--reps 5] [--json OUT]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_sketch import card   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", type=int, default=400)
    ap.add_argument("--length", type=int, default=1_000_000)
    ap.add_argument("--family", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json")
    a = ap.parse_args()
    import skani_b200 as sk
    from bench_support import synth
    ctx = sk.Context(0)
    bases, off, goc = synth.generate(0, a.genomes, a.length, G=a.family)
    s = sk.sketch_contigs(ctx, bases, off, goc, a.genomes)
    mp = sk.map_params()
    pairs = sk.screen_triangle(ctx, s, mp)
    plain = sk.chain_pairs(ctx, s, s, pairs, mp, as_array=True)
    res, moff, maps = sk.chain_pairs_mappings(ctx, s, s, pairs, mp)
    assert res.tobytes() == plain.tobytes(), "out differs between sk_chain_pairs and sk_chain_pairs_mappings"
    t_plain, t_maps = [], []
    for _ in range(a.reps):
        t0 = time.perf_counter(); r1 = sk.chain_pairs(ctx, s, s, pairs, mp, as_array=True); t_plain.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); r2 = sk.chain_pairs_mappings(ctx, s, s, pairs, mp); t_maps.append(time.perf_counter() - t0)
        assert r1.tobytes() == plain.tobytes() and r2[0].tobytes() == plain.tobytes() and r2[2].tobytes() == maps.tobytes()
    np_ = len(pairs)
    rec = dict(card=card(), genomes=a.genomes, length=a.length, family=a.family, pairs=np_, reps=a.reps,
               t_chain_s=float(np.median(t_plain)), t_chain_mappings_s=float(np.median(t_maps)),
               t_chain_all=[round(t, 4) for t in t_plain], t_mappings_all=[round(t, 4) for t in t_maps],
               us_per_pair_chain=float(np.median(t_plain)) / max(np_, 1) * 1e6,
               us_per_pair_mappings=float(np.median(t_maps)) / max(np_, 1) * 1e6,
               mappings=int(len(maps)), mappings_per_pair=len(maps) / max(np_, 1), bytes_copied=int(maps.nbytes),
               out_identical=True)
    rec["overhead_pct"] = (rec["t_chain_mappings_s"] / rec["t_chain_s"] - 1) * 100
    print(json.dumps(rec), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(rec, f)
    ctx.close()


if __name__ == "__main__":
    main()
