"""dp_group_kernel's two homes for the chain bookkeeping: chunks of at most DP_SMEM_ANCHORS anchors keep it in their group's
slab of shared memory, longer ones in global memory.  The host emulation tests/emu/emu_dp_onchip.cpp mirrors that arrangement
(groups in lockstep over one slab per warp, the per-chunk size split, the packed-word emission) and is checked against the
oracle under every group-kernel instantiation: on the constructed chunks of tests/dp_select_cases.py (1 to 4,000 anchors,
both sides of the bound), and on chunks of DP_SMEM_ANCHORS - 1, DP_SMEM_ANCHORS and DP_SMEM_ANCHORS + 1 anchors side by side in
one warp, where a slab one word too small, or a bound that lets one anchor too many on chip, corrupts the neighbouring group's
chain and names the field."""
import os
import re
import subprocess

import numpy as np

import dp_select_cases as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (GL, NE, FULLBAND, band, c): the group-kernel instantiations sk_chain_pairs can choose
GROUP_CONFIGS = [(4, 5, 1, 20, 125), (4, 5, 0, 16, 150), (4, 6, 1, 24, 104), (4, 6, 0, 22, 110), (8, 3, 1, 24, 104), (8, 3, 0, 20, 125)]


def dp_smem_anchors():
    src = open(os.path.join(ROOT, "skani_b200", "csrc", "chain.cu")).read()
    return int(re.search(r"constexpr uint32_t DP_SMEM_ANCHORS = (\d+);", src).group(1))


def bound_chunks(bound, seed):
    """chunks around the bound, longest first as the size sort leaves them: each is one diagonal chain per strand with random
    steps and repeat anchors, so the chain ends are the chunk's last anchors; a few short chunks share the warp"""
    rng = np.random.default_rng(seed)
    out = []
    for t, n in enumerate((bound + 1, bound + 1, bound, bound - 1, 65, 33, 9, 4, bound + 1, bound)):
        rows, q, r = [], 1000, [50_000, 1_000_000]
        while len(rows) < n:
            q += int(rng.integers(1, 120))
            s = int(rng.integers(0, 2))
            r[s] += int(rng.integers(1, 140)) * (1 if s == 0 else -1)
            rows.append((q, s, r[s], s))
            if rng.random() < 0.1 and len(rows) < n:
                rows.append((q, int(rng.integers(0, 3)), int(rng.integers(1, 10**6)), int(rng.integers(0, 2))))
        out.append(D.chunk(rows[:n], qctg=t % 3))
    return out


def write_chunks(f, gl, ne, fb, band, c, chunks):
    f.write("D %d %d %d %d %d %d\n" % (gl, ne, fb, band, c, len(chunks)))
    for ch in chunks:
        f.write("%d\n" % len(ch))
        f.write("\n".join(" ".join(map(str, row)) for row in ch.tolist()) + "\n")


def test_onchip_bound_emulation_matches_oracle(tmp_path):
    exe = str(tmp_path / "emu_dp_onchip")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fopenmp", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_dp_onchip.cpp"),
                           os.path.join(ROOT, "oracle", "skani_oracle.cpp"), "-lz"])
    bound = dp_smem_anchors()
    got = subprocess.check_output([exe, "--constants"], text=True).split()
    assert got == ["DP_SMEM_ANCHORS=%d" % bound], ("emulation's on-chip bound differs from chain.cu", got, bound)
    inp = str(tmp_path / "cases.txt")
    with open(inp, "w") as f:
        for gl, ne, fb, band, c in GROUP_CONFIGS:
            write_chunks(f, gl, ne, fb, band, c, list(D.dp_cases(band, gl).values()) + list(D.length_cases(gl, seed=c).values()))
            write_chunks(f, gl, ne, fb, band, c, bound_chunks(bound, seed=c + gl))
    with open(inp) as f:
        out = subprocess.run([exe], stdin=f, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-2000:]
    m = re.search(r"dp configs (\d+), chunks on chip (\d+), chunks in global memory (\d+), anchors (\d+), intervals (\d+), 0 failures", out.stdout)
    assert m and int(m.group(1)) == 2 * len(GROUP_CONFIGS), out.stdout
    assert all(int(x) > 0 for x in m.groups()) and int(m.group(5)) > 100, out.stdout
