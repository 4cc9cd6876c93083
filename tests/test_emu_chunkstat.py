"""Host emulation of chunkstat_kernel's per-chunk logic (skani_b200/csrc/chain_core.cuh: padded_start, seed_in_padded,
chunk_estimate) against the oracle's chunk_stats on constructed chunks: every count, the filter decision, the weight and the
estimate bit for bit, at the span, tbcq, 1.05 x upper_lower and clamp edges, seeds on and next to the padded interval ends,
interval starts around c, 2^31, 2^31 + c and 2^32 - 65537, and chunks of more than 32 intervals.  It also proves that the
putative-ANI filter's pow() result is never within 2 ulps of 0.950 for k >= 4, so a device pow that differs from glibc's by
at most that cannot flip the decision there; for k <= 3 exact ties (a / num_in = 19^k / 20^k) exist and
tests/test_gpu_chunkstat.py checks the device's decision on them directly.  See tests/emu/emu_chunkstat.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_chunk_statistics_logic_matches_oracle(tmp_path):
    exe = str(tmp_path / "emu_chunkstat")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fopenmp", "-ffp-contract=off", "-o", exe,
                           os.path.join(ROOT, "tests", "emu", "emu_chunkstat.cpp"), os.path.join(ROOT, "oracle", "skani_oracle.cpp"), "-lz"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert re.search(r"^0 failures$", out.stdout, re.M), out.stdout
    edges = dict((m.group(1), int(m.group(2))) for m in re.finditer(r"^edge (.+) (\d+)$", out.stdout, re.M))
    assert len(edges) == 27, edges
    for e, n in edges.items():
        assert n > 0, (e, out.stdout)
    m = re.search(r"^filter margin k >= 4: ([0-9.]+) ulps", out.stdout, re.M)
    assert m and float(m.group(1)) > 2.0, out.stdout
    print(out.stdout)
