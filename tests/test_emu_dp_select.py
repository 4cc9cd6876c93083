"""Host emulation of the banded DP (dp_group_kernel for every (GL, NE, FULLBAND), dp_warp_kernel for every NB) and of
select_kernel's shared-memory and global-memory selection, in the kernels' own arrangement, against the oracle on the
constructed lists of tests/dp_select_cases.py.  See tests/emu/emu_dp_select.cpp."""
import os
import re
import subprocess

import dp_select_cases as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (GL, NE, FULLBAND, NB, band, c): every instantiation sk_chain_pairs can choose (GL = 0: dp_warp_kernel)
DP_CONFIGS = [(4, 5, 1, 0, 20, 125), (4, 5, 0, 0, 16, 150), (4, 6, 1, 0, 24, 104), (4, 6, 0, 0, 22, 110), (8, 3, 1, 0, 24, 104),
              (8, 3, 0, 0, 20, 125), (0, 0, 0, 2, 20, 125), (0, 0, 0, 2, 31, 80), (0, 0, 0, 4, 32, 78), (0, 0, 0, 4, 92, 27),
              (0, 0, 0, 8, 96, 26), (0, 0, 0, 8, 208, 12), (0, 0, 0, 16, 227, 11), (0, 0, 0, 16, 416, 6)]


def write_input(path):
    with open(path, "w") as f:
        for gl, ne, fb, nb, band, c in DP_CONFIGS:
            chunks = list(D.dp_cases(band, gl or 4).values()) + list(D.length_cases(gl or 32, seed=c).values())
            f.write("D %d %d %d %d %d %d %d\n" % (gl, ne, fb, nb, band, c, len(chunks)))
            for ch in chunks:
                f.write("%d\n" % len(ch))
                f.write("\n".join(" ".join(map(str, row)) for row in ch.tolist()) + "\n")
        lists = []
        for name, (lst, nc) in D.select_cases().items():
            lists.append((name, lst, nc))
            for n in (1025, 2100):
                lists.append(("%s_in_%d" % (name, n), D.padded(lst, n, seed=n), nc))
        for n in (1, 2, 31, 1024, 3000):
            lists.append(("random_%d" % n, D.random_intervals(n, seed=n), 50))
        for sw in (0, 1):
            for name, lst, nc in lists:
                f.write("S %s %d %d %d\n" % (name, nc, len(lst), sw))
                f.write("\n".join(" ".join(map(str, x)) for x in lst) + "\n")


def test_dp_and_selection_emulation_matches_oracle(tmp_path):
    exe = str(tmp_path / "emu_dp_select")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fopenmp", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_dp_select.cpp"),
                           os.path.join(ROOT, "oracle", "skani_oracle.cpp"), "-lz"])
    # the emulation's selection constants are the kernel's
    src = open(os.path.join(ROOT, "skani_b200", "csrc", "chain.cu")).read()
    want = {n: re.search(r"constexpr uint32_t %s = (\d+);" % n, src).group(1) for n in ("SEL_DEPS", "SEL_SMEM_MAX", "SEL_CELL_SHIFT", "SEL_MAP_BITS")}
    got = dict(kv.split("=") for kv in subprocess.check_output([exe, "--constants"], text=True).split())
    assert got == want, ("emulation constants differ from chain.cu", got, want)
    inp = str(tmp_path / "cases.txt")
    write_input(inp)
    with open(inp) as f:
        out = subprocess.run([exe], stdin=f, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-2000:]
    m = re.search(r"dp configs (\d+), chunks (\d+), anchors (\d+), intervals (\d+), lists (\d+), dependency-list candidates (\d+), "
                  r"full-scan candidates (\d+), bitmap skips (\d+), bitmap scans (\d+), wide spans scanned (\d+), edge-candidate wins "
                  r"(\d+), sentinel rejects (\d+), 0 failures", out.stdout)
    assert m, out.stdout
    assert int(m.group(1)) == len(DP_CONFIGS) and int(m.group(4)) > 100, out.stdout
    assert all(int(x) > 0 for x in m.groups()), out.stdout
