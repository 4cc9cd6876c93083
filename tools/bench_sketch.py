#!/usr/bin/env python3
"""`skani-b200 sketch` end to end: a seeded synthetic set (bench_support/synth, clusters of 20, seed 20260924; default
1,000 x 5 Mbp) is written as one FASTA file per genome, then `sketch` writes a consolidated database from it with
--gpus 1 and, when more than one GPU is visible, with every visible GPU.  Reported per run: wall time of the process, the
INFO split (read, sketch, encode, write) and the bytes written.  With --parent-bin (a skani-b200 built from another
commit, its libskani_b200.so next to it) that build runs too, alternated with this one in the same call, and the
directories both builds wrote must be identical.  The card's name and power limit are read in the same call.

  python tools/bench_sketch.py [--genomes 1000] [--length 5000000] [--reps 2] [--parent-bin PATH] [--json OUT]
The FASTA files and databases go to a temporary directory that is removed at the end."""
import argparse
import filecmp
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30, check=True).stdout.strip().splitlines()
    name, limit = [x.strip() for x in out[0].split(",")[:2]]
    return {"name": name, "power_limit": limit, "gpus": len(out)}


def write_fasta(d, n, L):
    from bench_support import synth
    files, step = [], 100
    for g0 in range(0, n, step):
        g1 = min(n, g0 + step)
        bases, off, goc = synth.generate(g0, g1, L)
        for g in range(g0, g1):
            p = os.path.join(d, "g%06d.fa" % g)
            with open(p, "wb") as f:
                for i in [i for i in range(len(goc)) if goc[i] == g - g0]:
                    f.write(b">g%06d_c%d\n" % (g, i))
                    f.write(bases[int(off[i]):int(off[i + 1])].tobytes())
                    f.write(b"\n")
            files.append(p)
    return files


def run(binary, files, out, gpus, threads):
    t0 = time.perf_counter()
    p = subprocess.run([binary, "sketch", "-l", files, "-o", out, "--gpus", str(gpus), "-t", str(threads)], capture_output=True, text=True)
    wall = time.perf_counter() - t0
    if p.returncode != 0:
        raise SystemExit("sketch failed (%s):\n%s" % (binary, p.stderr[-2000:]))
    m = re.search(r"read ([\d.]+) s, sketch ([\d.]+) s, encode ([\d.]+) s, write ([\d.]+) s", p.stderr)
    split = dict(zip(("read", "sketch", "encode", "write"), map(float, m.groups()))) if m else None
    size = sum(os.path.getsize(os.path.join(out, f)) for f in os.listdir(out))
    return {"wall_s": round(wall, 3), "split_s": split, "bytes": size}


def same_dirs(a, b):
    fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
    return fa == fb and all(filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False) for f in fa)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", type=int, default=1000)
    ap.add_argument("--length", type=int, default=5_000_000)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 8)
    ap.add_argument("--parent-bin", default=None)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    info = card()
    builds = [("this", BIN)] + ([("parent", a.parent_bin)] if a.parent_bin else [])
    gpu_counts = [1] + ([info["gpus"]] if info["gpus"] > 1 else [])
    tmp = tempfile.mkdtemp(prefix="bench_sketch_")
    try:
        t0 = time.perf_counter()
        files = write_fasta(tmp, a.genomes, a.length)
        lst = os.path.join(tmp, "files.txt")
        with open(lst, "w") as f:
            f.write("\n".join(files) + "\n")
        res = {"card": info, "genomes": a.genomes, "length": a.length, "threads": a.threads, "fasta_write_s": round(time.perf_counter() - t0, 1),
               "runs": [], "identical": {}}
        if info["gpus"] == 1:
            res["multi_gpu"] = "not measured: one GPU visible"
        for rep in range(a.reps):
            for name, binary in (builds if rep % 2 == 0 else builds[::-1]):
                for g in gpu_counts:
                    out = os.path.join(tmp, "db_%s_%d_%d" % (name, g, rep))
                    r = run(binary, lst, out, g, a.threads)
                    r.update(build=name, gpus=g, rep=rep)
                    res["runs"].append(r)
                    print(json.dumps(r), flush=True)
        for g in gpu_counts:
            ref = os.path.join(tmp, "db_this_%d_0" % g)
            for name, _ in builds:
                for rep in range(a.reps):
                    res["identical"]["%s_%d_%d" % (name, g, rep)] = same_dirs(ref, os.path.join(tmp, "db_%s_%d_%d" % (name, g, rep)))
            if len(gpu_counts) > 1:
                res["identical"]["gpus_1_vs_%d" % g] = same_dirs(os.path.join(tmp, "db_this_1_0"), ref)
        print(json.dumps(res))
        if a.json:
            with open(a.json, "w") as f:
                json.dump(res, f, indent=1)
        if not all(res["identical"].values()):
            raise SystemExit("outputs differ")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
