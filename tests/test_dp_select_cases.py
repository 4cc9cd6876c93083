"""CPU checks of the DP / interval-selection harness (no GPU): the oracle's entries on given lists (orc_chain_chunks,
orc_select_intervals) reproduce chain_seeds' own taps on real pairs, and the constructed cases of tests/dp_select_cases.py
reach the edges they were built for at every band the DP instantiations cover."""
import os

import numpy as np
import pytest

import dp_select_cases as D
import oracle_py as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.mark.parametrize("c", [125, 30])
def test_oracle_entries_match_chain_seeds(c):
    sk, _ = O.sketch_files([os.path.join(GOLDEN, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz")], c=c)
    for r, q in ((0, 1), (1, 0)):
        d = O.chain_debug(sk[r], sk[q])
        first = d["chunk_first"]
        chunks = [d["anchors"][first[i]:first[i + 1]] for i in range(len(first) - 1)]
        o = O.chain_chunks(chunks, c, 15, d["switched"])
        assert np.array_equal(o["score"], d["score"]) and np.array_equal(o["pointer"], d["pointer"])
        assert np.array_equal(o["intervals"], d["intervals"])
        assert np.array_equal(o["chunk_acc"], d["chunk_stats"][:, :5])
        assert len(d["intervals"]) > 100
        s = O.select_intervals(d["intervals"][::-1, :10], len(chunks), c, 15, d["switched"])
        assert np.array_equal(s["intervals"], d["intervals"]) and np.array_equal(s["chunk_acc"], o["chunk_acc"])
        assert (s["pair_sumlen"], s["pair_nchains"]) == (o["pair_sumlen"], o["pair_nchains"])
        assert o["pair_sumlen"] // o["pair_nchains"] == d["result"].avg_chain_int_len


@pytest.mark.parametrize("band,gl", [(16, 4), (20, 4), (20, 8), (24, 8), (31, 32), (96, 32), (416, 32)])
def test_dp_cases_reach_their_edges(band, gl):
    cases = D.dp_cases(band, min(gl, 8))
    D.check_dp_edges(cases, {nm: O.chain_chunks([ch], 2500 // band, 15) for nm, ch in cases.items()}, band)
