"""Restatement of sk_chain_pairs_mappings' records from the CPU oracle's chain taps: the kept intervals of
get_nonoverlapping_chains in the caller's orientation, joined to chunk_estimate's est / weight / valid of their chunk and
sorted by (query_contig, q0, q1, ref_contig, r0, r1, reverse, chunk).  TEST INFRASTRUCTURE ONLY."""
import numpy as np

import oracle_py as O
from skani_b200.host import MAPPING_DTYPE

KEY = ("query_contig", "q0", "q1", "ref_contig", "r0", "r1", "reverse", "chunk")


def expected(od, c, k):
    """od: oracle_py.chain_debug(ref, query, cp) -> the pair's records (MAPPING_DTYPE)"""
    iv = od["intervals"]
    kept = iv[iv[:, 10] == 1] if len(iv) else iv
    cs = od["chunk_stats"]
    est, w, v = O.chunk_estimate(cs[:, :8], c, k) if len(cs) else (np.zeros(0), np.zeros(0), np.zeros(0))
    sw = bool(od["switched"])
    out = np.zeros(len(kept), MAPPING_DTYPE)
    for i, x in enumerate(kept):
        _, na, q0, q1, r0, r1, rctg, qctg, ch, rev = (int(t) for t in x[:10])
        if sw:
            q0, q1, r0, r1, qctg, rctg = r0, r1, q0, q1, rctg, qctg
        valid = int(v[ch])
        out[i] = (qctg, rctg, q0, q1, r0, r1, na, ch, float(est[ch]) if valid else 0.0, int(w[ch]) if valid else 0,
                  rev, int(sw), valid, 0)
    return np.sort(out, order=list(KEY), kind="stable")


def sort_key(m):
    return tuple(int(m[f]) for f in KEY)
