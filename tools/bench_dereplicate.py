#!/usr/bin/env python3
"""Dereplication measurements: `cluster` (triangle + greedy clustering) against `dereplicate`, printed as JSON lines with the
card's name and power limit read in the same call.

1. Library: sk_screen_triangle + sk_chain_pairs + sk_cluster (greedy) against sk_dereplicate on the same in-memory set of
   synthetic families (bench_support/synth, genome ids shuffled over the indices as bench.py lays them out, so that length
   ties rank families in scattered order).  Families of 20 and of 200.  One warm-up call of each, then --reps timed calls
   alternated (host clock around calls that end in a device synchronise).  rep and cluster must be equal and every member's
   joining row byte-identical.  Pairs chained by each side are printed.
2. End to end: `cluster` against `dereplicate` on the same sets written as one FASTA file per genome, alternated --reps
   times (wall time of the process); stdout must be identical.
3. --host-store (instead of 1 and 2): sk_dereplicate on the in-memory set against sk_dereplicate_store on a host sketch
   store of the same genomes (sketched in four groups, each added and freed), with one context, two contexts on one device
   (derived budgets) and two contexts with a budget of about one family's bytes (many working sets).  Families of 20 and of
   200.  rep, cluster and join must be byte-identical.  Each row prints the pairs chained, the working sets, the bytes
   gathered, and how the time splits: the marker gather, the screens on ctxs[0] (t_screen), the chain steps (t_chain, wall
   time of gathers plus chaining) and the gather / chain seconds summed over the contexts.
4. --update F (instead of 1 and 2): a catalogue update.  The first 1 - F of the genome indices (families scattered over
   them) are dereplicated as the catalogue; then its representatives are fixed (in their catalogue rank order) and the other
   F of the genomes added (sk_dereplicate_fixed, and sk_dereplicate_store_fixed on two contexts of one device), against
   dereplicating all genomes again (sk_dereplicate, sk_dereplicate_store).  Families of 20 and of 200.  Each store call must
   equal its in-memory call byte for byte, and every catalogue representative must stay one.  Each row prints the pairs
   screened and chained and the times.

  python tools/bench_dereplicate.py [--genomes 2000] [--length 1000000] [--reps 3] [--skip-e2e] [--host-store] [--update F]
                                    [--json OUT]
The FASTA files go to a temporary directory that is removed at the end."""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")

from bench_sketch import card   # noqa: E402


def emit(rec, sink):
    print(json.dumps(rec), flush=True)
    sink.append(rec)


def family_set(n, L, G, seed):
    from bench_support import synth
    return synth.generate_ids(synth.shuffled_ids(n, seed), L, G=G)


def bench_lib(n, L, G, reps, sink):
    import skani_b200 as sk
    ctx = sk.Context(0)
    bases, off, goc = family_set(n, L, G, 20261018)
    s = sk.sketch_contigs(ctx, bases, off, goc, n)
    total = np.bincount(goc, weights=np.diff(off).astype(np.float64), minlength=n)
    order = np.lexsort((np.arange(n), -total))          # longest first, ties by genome index (cluster's ranking)
    rank = np.empty(n, np.uint32); rank[order] = np.arange(n)
    mp = sk.map_params()

    def via_triangle():
        pairs = sk.screen_triangle(ctx, s, mp)
        rows = sk.chain_pairs(ctx, s, s, pairs, mp, as_array=True)
        rep, cl, edge, _ = sk.cluster(ctx, n, rows, rank, min_ani=0.95)
        return rep, cl, edge, rows

    def via_derep():
        return sk.dereplicate(ctx, s, rank, min_ani=0.95, mp=mp)

    tri, der = via_triangle(), via_derep()                 # warm-up, and the equality check
    rep, cl, edge, rows = tri
    mem = rep != np.arange(n)
    equal = bool(np.array_equal(rep, der[0]) and np.array_equal(cl, der[1]) and
                 der[2][mem].tobytes() == rows[edge[mem].astype(np.int64)].tobytes())
    t_tri, t_der = [], []
    for _ in range(reps):
        t = time.perf_counter(); via_triangle(); t_tri.append(time.perf_counter() - t)
        t = time.perf_counter(); via_derep(); t_der.append(time.perf_counter() - t)
    st = der[3]
    emit({"bench": "library", "genomes": n, "length": L, "family": G, "card": card(), "equal": equal, "clusters": int(st.n_clusters),
          "triangle_pairs_chained": int(len(rows)), "derep_pairs_chained": int(st.pairs_chained), "derep_pairs_screened": int(st.pairs_screened),
          "waves": int(st.waves), "t_triangle_cluster_s": sorted(t_tri), "t_dereplicate_s": sorted(t_der),
          "derep_split_s": {"screen": st.t_screen, "chain": st.t_chain, "decide": st.t_decide, "total": st.t_total}}, sink)
    s.free()
    ctx.close()
    return equal


def bench_store(n, L, G, reps, sink):
    import skani_b200 as sk
    ctxs = [sk.Context(0), sk.Context(0)]
    bases, off, goc = family_set(n, L, G, 20261018)
    s = sk.sketch_contigs(ctxs[0], bases, off, goc, n)
    s.set_name_ranks(np.arange(n))
    st = sk.SketchStore()
    bounds = np.linspace(0, n, 5).astype(int)
    for a, b in zip(bounds[:-1], bounds[1:]):
        idx = np.nonzero((goc >= a) & (goc < b))[0]
        lo, hi = int(off[idx[0]]), int(off[idx[-1] + 1])
        part = sk.sketch_contigs(ctxs[0], bases[lo:hi], off[idx[0]:idx[-1] + 2] - off[idx[0]], goc[idx] - a, b - a)
        st.add(part)
        part.free()
    st.set_name_ranks(np.arange(n))
    total = np.bincount(goc, weights=np.diff(off).astype(np.float64), minlength=n)
    order = np.lexsort((np.arange(n), -total))
    rank = np.empty(n, np.uint32); rank[order] = np.arange(n)
    mp = sk.map_params()
    gb = np.array([st.genome_bytes(g) for g in range(n)])
    small = int(max(1.05 * G * gb.max(), 2 * gb.max() + 1))
    runs = {"in_memory": lambda: sk.dereplicate(ctxs[0], s, rank, min_ani=0.95, mp=mp),
            "store_1ctx": lambda: sk.dereplicate_store(ctxs[:1], st, rank, min_ani=0.95, mp=mp),
            "store_2ctx": lambda: sk.dereplicate_store(ctxs, st, rank, min_ani=0.95, mp=mp),
            "store_2ctx_small_budget": lambda: sk.dereplicate_store(ctxs, st, rank, min_ani=0.95, mp=mp, device_budget=small)}
    last = {k: f() for k, f in runs.items()}              # warm-up, and the equality check
    ref = last["in_memory"]
    equal = all(np.array_equal(v[0], ref[0]) and np.array_equal(v[1], ref[1]) and v[2].tobytes() == ref[2].tobytes() for v in last.values())
    times = {k: [] for k in runs}
    for _ in range(reps):
        for k, f in runs.items():
            t = time.perf_counter(); last[k] = f(); times[k].append(time.perf_counter() - t)
    for k in runs:
        dst = last[k][3]
        rec = {"bench": "host_store", "run": k, "genomes": n, "length": L, "family": G, "card": card(), "equal": equal,
               "clusters": int(dst.n_clusters), "pairs_chained": int(dst.pairs_chained), "pairs_screened": int(dst.pairs_screened),
               "waves": int(dst.waves), "t_s": sorted(times[k]),
               "derep_split_s": {"screen": dst.t_screen, "chain": dst.t_chain, "decide": dst.t_decide, "total": dst.t_total}}
        if k != "in_memory":
            sst = last[k][4]
            rec.update({"device_budget": small if k.endswith("small_budget") else 0, "working_sets": int(sst.n_working_sets),
                        "split_components": int(sst.n_split_components), "gathered_bytes": int(sst.gathered_bytes),
                        "max_working_set_bytes": int(sst.max_working_set_bytes), "store_bytes": int(gb.sum()),
                        "store_split_s": {"marker_gather": sst.t_screen, "gather_summed": sst.t_gather, "chain_summed": sst.t_chain}})
        emit(rec, sink)
    st.free()
    s.free()
    for c in ctxs:
        c.close()
    return equal


def sketch_genomes(sk, ctx, bases, off, goc, genomes):
    """the genomes of the list (in list order) as one device set, name ranks = their order by genome id"""
    idx = [np.nonzero(goc == g)[0] for g in genomes]
    parts = [bases[int(off[i[0]]):int(off[i[-1] + 1])] for i in idx]
    lens = np.concatenate([np.diff(off[i[0]:i[-1] + 2]) for i in idx])
    s = sk.sketch_contigs(ctx, np.concatenate(parts), np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64),
                          np.concatenate([np.full(len(i), k, np.uint32) for k, i in enumerate(idx)]), len(genomes))
    names = np.empty(len(genomes), np.uint64); names[np.argsort(genomes, kind="stable")] = np.arange(len(genomes))
    s.set_name_ranks(names)
    return s, names


def bench_update(n, L, G, frac, reps, sink):
    import skani_b200 as sk
    ctxs = [sk.Context(0), sk.Context(0)]
    ctx = ctxs[0]
    bases, off, goc = family_set(n, L, G, 20261018)
    total = np.bincount(goc, weights=np.diff(off).astype(np.float64), minlength=n)

    def length_rank(genomes, n_first=0):
        t = total[np.asarray(genomes)]
        k = np.arange(len(genomes))
        order = np.concatenate([np.lexsort((k[:n_first], -t[:n_first])), n_first + np.lexsort((k[n_first:], -t[n_first:]))])
        rank = np.empty(len(genomes), np.uint32); rank[order] = np.arange(len(genomes))
        return rank

    def store_of(s, names):
        st = sk.SketchStore()
        st.add(s)
        st.set_name_ranks(names)
        return st

    m = int(round((1 - frac) * n))
    cat = list(range(m))
    cs, _ = sketch_genomes(sk, ctx, bases, off, goc, cat)
    crank = length_rank(cat)
    crep = sk.dereplicate(ctx, cs, crank, min_ani=0.95)[0]
    cs.free()
    fixed = [cat[g] for g in np.argsort(crank, kind="stable") if crep[g] == g]     # catalogue rank order
    upd = fixed + list(range(m, n))                                                 # fixed first, then the new genomes
    us, unames = sketch_genomes(sk, ctx, bases, off, goc, upd)
    ust = store_of(us, unames)
    urank = length_rank(upd, len(fixed))        # among the fixed genomes this is the catalogue's rank order again
    alls, anames = sketch_genomes(sk, ctx, bases, off, goc, list(range(n)))
    ast = store_of(alls, anames)
    arank = length_rank(list(range(n)))
    nf = len(fixed)
    runs = {"update_in_memory": lambda: sk.dereplicate_fixed(ctx, us, urank, nf, min_ani=0.95),
            "update_host_store": lambda: sk.dereplicate_store_fixed(ctxs, ust, urank, nf, min_ani=0.95),
            "full_in_memory": lambda: sk.dereplicate(ctx, alls, arank, min_ani=0.95),
            "full_host_store": lambda: sk.dereplicate_store(ctxs, ast, arank, min_ani=0.95)}
    last = {k: f() for k, f in runs.items()}              # warm-up, and the equality checks
    same = lambda a, b: all(x.tobytes() == y.tobytes() for x, y in zip(a[:3], b[:3]))
    equal = bool(same(last["update_in_memory"], last["update_host_store"]) and same(last["full_in_memory"], last["full_host_store"]) and
                 (last["update_in_memory"][0][:nf] == np.arange(nf)).all())
    times = {k: [] for k in runs}
    for _ in range(reps):
        for k, f in runs.items():
            t = time.perf_counter(); last[k] = f(); times[k].append(time.perf_counter() - t)
    for k in runs:
        dst = last[k][3]
        emit({"bench": "update", "run": k, "genomes": n, "length": L, "family": G, "update_fraction": frac, "catalogue_genomes": m,
              "fixed_representatives": nf, "set_genomes": len(upd) if k.startswith("update") else n, "card": card(), "equal": equal,
              "clusters": int(dst.n_clusters), "pairs_screened": int(dst.pairs_screened), "pairs_chained": int(dst.pairs_chained),
              "waves": int(dst.waves), "t_s": sorted(times[k]),
              "derep_split_s": {"screen": dst.t_screen, "chain": dst.t_chain, "decide": dst.t_decide, "total": dst.t_total}}, sink)
    for x in (ust, ast, us, alls):
        x.free()
    for c in ctxs:
        c.close()
    return equal


def write_fasta(d, n, L, G):
    bases, off, goc = family_set(n, L, G, 20261018)
    files = []
    for g in range(n):
        p = os.path.join(d, "g%06d.fa" % g)
        with open(p, "wb") as f:
            for i in np.nonzero(goc == g)[0]:
                f.write(b">g%06d_c%d\n" % (g, i) + bases[int(off[i]):int(off[i + 1])].tobytes() + b"\n")
        files.append(p)
    return files


def bench_e2e(n, L, G, reps, sink):
    d = tempfile.mkdtemp(prefix="bench_derep_")
    try:
        files = write_fasta(d, n, L, G)
        lst = os.path.join(d, "list.txt")
        with open(lst, "w") as f:
            f.write("\n".join(files) + "\n")
        out = {}
        times = {"cluster": [], "dereplicate": []}
        for r in range(reps + 1):
            for cmd in ("cluster", "dereplicate"):
                t = time.perf_counter()
                p = subprocess.run([BIN, cmd, "-l", lst], capture_output=True, text=True, check=True)
                if r:
                    times[cmd].append(time.perf_counter() - t)
                out[cmd] = p.stdout
                if cmd == "dereplicate":
                    info = [ln for ln in p.stderr.splitlines() if "pairs screened" in ln]
        emit({"bench": "end_to_end", "genomes": n, "length": L, "family": G, "card": card(), "equal": out["cluster"] == out["dereplicate"],
              "t_cluster_s": sorted(times["cluster"]), "t_dereplicate_s": sorted(times["dereplicate"]), "dereplicate_info": info[-1] if info else ""}, sink)
        return out["cluster"] == out["dereplicate"]
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", type=int, default=2000)
    ap.add_argument("--length", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--host-store", action="store_true", help="in-memory dereplicate against dereplicate_store only")
    ap.add_argument("--update", type=float, metavar="F", help="a catalogue update adding the last F of the genomes")
    ap.add_argument("--json")
    a = ap.parse_args()
    sink, ok = [], True
    if a.update is not None:
        for G in (20, 200):
            ok &= bench_update(a.genomes, a.length, G, a.update, a.reps, sink)
    elif a.host_store:
        for G in (20, 200):
            ok &= bench_store(a.genomes, a.length, G, a.reps, sink)
    else:
        for G in (20, 200):
            ok &= bench_lib(a.genomes, a.length, G, a.reps, sink)
    if not a.skip_e2e and not a.host_store and a.update is None:
        for G in (20, 200):
            ok &= bench_e2e(a.genomes, a.length, G, a.reps, sink)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(sink, f, indent=1)
    if not ok:
        sys.exit("outputs differ")


if __name__ == "__main__":
    main()
