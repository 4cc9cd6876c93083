"""sk_neighbor_joining's arithmetic (skani_b200/csrc/nj_core.cuh) on the CPU: tests/emu/emu_nj.cpp, built with
-ffp-contract=off, drives it through whole runs the way nj.cu does (padded square, dead slots, the minimum over the upper
triangle in a random visit order, compaction) and must give tests/nj_ref.py's join table bit for bit on 300 random graphs:
Erdos-Renyi and family graphs, equal ANIs, the all-missing graph, additive trees, and sizes 0 to 150 across the tile and
compaction edges."""
import os
import subprocess

import numpy as np

import cluster_ref as CR
import nj_ref as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cases():
    rng = np.random.default_rng(7)
    out = []
    for k in range(300):
        kind = k % 6
        n = int(rng.choice([0, 1, 2, 3, 4, 5, 31, 33, 63, 64, 65, 66, 90, 129, 150])) if k % 5 == 0 else int(rng.integers(2, 100))
        if kind == 0:
            n, a, b, ani = CR.erdos_renyi(rng, max(n, 2), 3 * n) if n >= 2 else (n, [], [], [])
        elif kind == 1 and n >= 2:
            n, a, b, ani = CR.families(rng, n, int(rng.integers(2, 8)), n)
        elif kind == 2 and n >= 2:         # ties everywhere: one ANI for every row
            n, a, b, ani = CR.families(rng, n, int(rng.integers(2, 8)), n)
            ani = np.full(len(a), np.float32(0.95))
        elif kind == 3:                    # all missing, plus rows that are never edges
            a = np.arange(max(n - 1, 0)); b = a + 1
            ani = np.array([np.nan, -1.0, 0.1][:len(a)] + [0.05] * max(len(a) - 3, 0), np.float32)
        elif kind == 4 and n >= 3:
            D, _, _ = N.random_additive(rng, n)
            a, b = np.triu_indices(n, 1)
            ani = (1.0 - D[a, b]).astype(np.float32)
        else:
            ani = np.float32(0.9) + np.float32(0.01) * rng.integers(0, 5, size=2 * n).astype(np.float32)   # few values: many ties
            n, a, b, ani = CR._finish(rng, max(n, 2), rng.integers(0, max(n, 2), size=(2 * n, 2)), ani) if n >= 2 else (n, [], [], [])
        out.append((n, np.asarray(a, np.uint32), np.asarray(b, np.uint32), np.asarray(ani, np.float32)))
    return out


def test_emu_matches_reference(tmp_path):
    exe = str(tmp_path / "emu_nj")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_nj.cpp")])
    cs = cases()
    text = []
    for n, a, b, ani in cs:
        text.append("%d %d\n" % (n, len(a)))
        text += ["%d %d %x\n" % (x, y, v) for x, y, v in zip(a, b, ani.view(np.uint32))]
    out = subprocess.run([exe], input="".join(text), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr
    blocks = out.stdout.split("case ")[1:]
    assert len(blocks) == len(cs)
    compacted = ties = 0
    for (n, a, b, ani), blk in zip(cs, blocks):
        lines = blk.strip().split("\n")
        assert int(lines[0]) == n
        got = [(int(x), int(y), float.fromhex(p), float.fromhex(q)) for x, y, p, q in (ln.split() for ln in lines[1:])]
        want = N.nj_results(n, a, b, ani)
        assert got == [(int(r["a"]), int(r["b"]), float(r["len_a"]), float(r["len_b"])) for r in want], (n, len(a))
        compacted += n > 85
        ties += len(np.unique(ani)) < len(ani) or len(a) == 0
    assert compacted >= 10 and ties >= 100
