#!/usr/bin/env python3
"""Record, hit-record, anchor and chunk counts of one step of bench.py's `value` leg, and the distribution of anchors per
chunk that the chain back end's DP sees (the sizes that decide dp_group_kernel's on-chip bound).  Records are the
query-role genomes' records the probe reads; hit records are those with anchors (the records chunk_anchor_kernel scans).

  python tools/count_chain_shapes.py [--config north|c2|dense|c5] [--genomes N] [--batch P]

Sketches and screens the same synthetic genomes as tools/profile_value_leg.py, then re-chains the screened pairs with
sk_chain_pairs_debug, P pairs per call (the same batching and kernels as chain_pairs), keeping only each pair's chunk
boundaries and its distinct anchor query positions.  Prints the totals and a histogram of anchors per chunk."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.dont_write_bytecode = True

from profile_value_leg import CONFIGS, card  # noqa: E402

EDGES = (1, 2, 3, 8, 16, 32, 64, 96, 128, 160, 192, 256, 320, 384, 512, 1024, 4096, 1 << 32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="north", choices=sorted(CONFIGS))
    ap.add_argument("--genomes", type=int, default=None)
    ap.add_argument("--batch", type=int, default=2000)
    a = ap.parse_args()
    cfg = dict(CONFIGS[a.config])
    if a.genomes:
        cfg["genomes"] = a.genomes
    import torch
    import skani_b200 as sk
    from bench_support import synth

    N, L, G = cfg["genomes"], cfg["genome_len"], cfg["cluster"]
    ids = np.arange(N, dtype=np.uint64)
    pinned = torch.empty(N * L, dtype=torch.uint8, pin_memory=True)
    synth.generate_ids(ids, L, G=G, out=pinned.numpy())
    off, goc = synth.layout_ids(ids, L, G)
    dev = pinned.to("cuda")
    ctx = sk.Context(0)
    sp = sk.sketch_params(cfg["c"], 15, cfg["marker_c"])
    mp = sk.map_params(rescue_small=cfg["rescue_small"])
    gs = sk.sketch_contigs(ctx, None, off, goc, N, sp, device_ptr=dev.data_ptr())
    del dev
    pairs = sk.screen_triangle(ctx, gs, mp)
    n_pairs = len(pairs)
    sizes = []
    n_anchors = 0
    n_iv = 0
    n_rec = 0
    n_hit = 0
    n_rec_of = {}
    for b in range(0, n_pairs, a.batch):
        for pid, d in zip(pairs[b:b + a.batch], sk.chain_pairs_debug(ctx, gs, gs, pairs[b:b + a.batch], mp)):
            g = int(pid) >> 32 if d["switched"] else int(pid) & 0xFFFFFFFF      # the query-role (iterated) genome
            if g not in n_rec_of:
                n_rec_of[g] = gs.info(g)["n_records"]
            n_rec += n_rec_of[g]
            an = d["anchors"]
            if len(an):                                       # one hit record = one (query contig, query position)
                n_hit += len(np.unique(an[:, 0].astype(np.uint64) << np.uint64(32) | an[:, 1].astype(np.uint64)))
            cf = d["chunk_first"].astype(np.int64)
            sizes.append(np.diff(cf))
            n_anchors += int(d["anchors"].shape[0])
            n_iv += int(d["intervals"].shape[0])
    sizes = np.concatenate(sizes) if sizes else np.zeros(0, np.int64)
    print("card: %s" % card())
    print("config %s: %d genomes x %d bp, cluster %d, c=%d: %d pairs chained" % (a.config, N, L, G, cfg["c"], n_pairs))
    print("query-role records %d, hit records %d (%.1f %% of records), anchors %d (%.3f per hit record)"
          % (n_rec, n_hit, 100.0 * n_hit / max(n_rec, 1), n_anchors, n_anchors / max(n_hit, 1)))
    print("anchors %d, chunks %d (%d with anchors), DP intervals %d" % (n_anchors, len(sizes), int((sizes > 0).sum()), n_iv))
    nz = sizes[sizes > 0]
    if len(nz):
        print("anchors per non-empty chunk: mean %.1f, median %d, p90 %d, p99 %d, p99.9 %d, max %d"
              % (nz.mean(), np.median(nz), np.percentile(nz, 90), np.percentile(nz, 99), np.percentile(nz, 99.9), nz.max()))
    print("| anchors per chunk | chunks | share of chunks | share of anchors |")
    print("|---|---:|---:|---:|")
    for lo, hi in zip((0,) + EDGES[:-1], EDGES):
        m = (sizes >= lo) & (sizes < hi)
        print("| [%d, %s) | %d | %.3f %% | %.3f %% |" % (lo, hi if hi < (1 << 32) else "inf", int(m.sum()),
                                                       100.0 * m.sum() / max(len(sizes), 1),
                                                       100.0 * sizes[m].sum() / max(n_anchors, 1)))
    gs.free()
    ctx.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
