"""Host emulation of sk_chain_pairs_mappings' record logic (skani_b200/csrc/mapping_core.cuh: the un-switching, chunk join
and sort order, see tests/emu/emu_mappings.cpp) on the oracle's chain taps, against the restatement in mapping_ref.py.  The
E. coli goldens in both orientations, so that one of the two pairs is switched, at c = 125 and 200 and in the trim modes."""
import os
import subprocess

import numpy as np
import pytest

import oracle_py as O
import mapping_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
FILES = [os.path.join(GOLD, "e.coli-EC590.fasta.gz"), os.path.join(GOLD, "e.coli-K12.fasta.gz")]


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu") / "emu_mappings")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fopenmp", "-o", out, os.path.join(ROOT, "tests", "emu", "emu_mappings.cpp"),
                           os.path.join(ROOT, "oracle", "skani_oracle.cpp"), "-lz"])
    return out


def parse(text):
    pairs, cur = {}, None
    for line in text.splitlines():
        f = line.split()
        if f[0] == "PAIR":
            cur = pairs.setdefault((int(f[1]), int(f[2])), [])
            continue
        cur.append(tuple(int(x) for x in f[:8]) + (float.fromhex(f[8]),) + tuple(int(x) for x in f[9:]))
    return pairs


@pytest.mark.parametrize("c,robust,median,learned", [(125, 0, 0, 1), (200, 0, 0, 1), (125, 1, 0, 0), (125, 0, 1, 0)])
def test_records_match_restatement(exe, c, robust, median, learned):
    out = subprocess.run([exe, str(c), str(robust), str(median), str(learned)] + FILES, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr
    got = parse(out.stdout)
    sk, _ = O.sketch_files(FILES, c=c)
    cp = O.cmd(robust=bool(robust), median=bool(median), learned_ani=bool(learned))
    switched = set()
    for (a, b), recs in got.items():
        od = O.chain_debug(sk[a], sk[b], cp)
        exp = mapping_ref.expected(od, c, 15)
        assert len(recs) == len(exp) > 100, (a, b, len(recs), len(exp))
        for g, e in zip(recs, exp):
            assert g == tuple(e.tolist())[:13], (a, b, g, e)
        if od["switched"]:
            switched.add((a, b))
        assert np.all(np.diff([mapping_ref.sort_key(m) for m in exp], axis=0).any(axis=1))
    assert len(switched) == 1, switched        # one orientation chains the other genome in the query role
