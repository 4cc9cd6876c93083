"""Constructed anchor and interval lists for the chain back end's banded DP and interval selection, built to sit on the edges
where those kernels can go wrong (see tests/test_gpu_dp_select.py, tests/test_emu_dp_select.py and
tests/test_dp_select_cases.py).

Anchors are (query_contig, query_pos, ref_contig, ref_pos, reverse) rows; a chunk is a list of them sorted by (query_pos,
ref_contig, ref_pos, reverse).  Intervals are (score, num_anchors, q0, q1, r0, r1, ref_contig, query_contig, chunk, reverse)
rows.  Every builder returns named cases so that a test can say which edge a mismatch sits on."""
import numpy as np

TOP = 2**32 - 65537          # largest position a sketch may hold
CTG_MAX = 2**30 - 1          # largest ref contig index (types.rs:135-138)
CELL = 1 << 14               # select_kernel's occupancy-bitmap cell


def chunk(rows, qctg=0):
    a = np.array([(qctg,) + tuple(r) for r in rows], np.int64).reshape(-1, 5)
    order = np.lexsort((a[:, 4], a[:, 3], a[:, 2], a[:, 1]))
    a = a[order]
    assert a.min() >= 0 and a[:, 1].max() <= TOP and a[:, 3].max() <= TOP and a[:, 2].max() <= CTG_MAX
    return a.astype(np.uint32)


def diag(q0, r0, steps, rctg=0, rev=0):
    """anchors along a diagonal (anti-diagonal when rev): steps = query / ref advances after the first anchor"""
    rows, q, r = [(q0, rctg, r0, rev)], q0, r0
    for dq, dr in steps:
        q += dq
        r = r - dr if rev else r + dr
        rows.append((q, rctg, r, rev))
    return rows


def fillers(qpos, n, first_ctg=1):
    """n anchors at one query position on distinct ref contigs: they take up DP index distance but never chain"""
    return [(qpos, first_ctg + t, 1000, 0) for t in range(n)]


def dp_cases(band, gl=4):
    """{name: chunk} for a DP band (anchors) and a group width gl (the lane offsets of the tie cases)"""
    cases = {}
    # a sole same-contig predecessor at distance band (chains) and band + 1 (does not); the others are other contigs
    for d in (band, band + 1):
        cases["band_%d" % (d - band)] = chunk([(1000, 0, 5000, 0)] + fillers(1001, d - 1) + [(1002, 0, 5002, 0)])
    # query gap 2,500 (chains) / 2,501 (does not), as 4-anchor chains with zero diagonal gap
    cases["qgap_2500"] = chunk(diag(100, 100, [(2500, 2500)] * 3))
    cases["qgap_2501"] = chunk(diag(100, 100, [(2501, 2501)] * 3))
    # repeats: two anchors on one query position, then a chain continuing from one of them
    cases["same_qpos"] = chunk([(500, 0, 1000, 0), (500, 0, 3000, 0), (600, 0, 1100, 0), (700, 0, 1200, 0), (700, 0, 3200, 0),
                                (800, 0, 3300, 0)])
    # ref gap 0 on either strand
    cases["rgap0_fwd"] = chunk([(100, 0, 500, 0), (150, 0, 500, 0), (200, 0, 550, 0)])
    cases["rgap0_rev"] = chunk([(100, 0, 500, 1), (150, 0, 500, 1), (200, 0, 450, 1)])
    # |dr - dq| of 300 / 301 after a 16-anchor chain (score 300): only then does a 300 gap still score > 0
    for g in (300, 301):
        rows = diag(10_000, 20_000, [(100, 100)] * 15)
        rows.append((rows[-1][0] + 400, 0, rows[-1][2] + 400 + g, 0))
        cases["diag_gap_%d" % g] = chunk(rows)
        rows = diag(10_000, 900_000, [(100, 100)] * 15, rev=1)
        rows.append((rows[-1][0] + 400, 0, rows[-1][2] - 400 + g, 1))
        cases["diag_gap_%d_rev" % g] = chunk(rows)
    # other ref contigs and the other strand between a chain's anchors
    rows = diag(1000, 1000, [(50, 50)] * 6)
    for t, (q, _, r, _) in enumerate(rows[:-1]):
        rows += [(q + 10, 7, r + 10, 0), (q + 20, 0, r + 20, 1), (q + 30, 0, r + 30 + 2 * t, 1)]
    cases["interleaved"] = chunk(rows)
    # equal new scores from two candidates at distances d1 > d2: j1 = (Q - 30, R - 20), j2 = (Q - 10, R - 20) score 10 each
    # for the anchor (Q, R) and cannot chain to each other (ref gap 0); the nearer one (largest j) must win.  The distances
    # range over lanes, register sets, the edge candidate and the block rotation (lead = anchors before j1).
    Q, R = 100_000, 200_000
    dmax = min(band, 40)
    ds = sorted(set(range(1, dmax + 1)) | {band - 1, band})
    for lead in range(gl):
        for d1 in ds:
            for d2 in ds:
                if d2 >= d1 or d2 < 1 or (band > 40 and d1 < band - 1 and d1 % 3):
                    continue
                rows = fillers(Q - 40, lead) + [(Q - 30, 0, R - 20, 0)] + fillers(Q - 30, d1 - d2 - 1)
                rows += [(Q - 10, 0, R - 20, 0)] + fillers(Q - 10, d2 - 1) + [(Q, 0, R, 0)]
                cases["tie_%d_%d_%d" % (lead, d1, d2)] = chunk(rows)
    # a component whose two chain ends share the maximal score (55, both from the same anchor): the larger index is the end
    c0 = diag(5000, 7000, [(10, 10)] * 2)
    qc, rc = c0[-1][0], c0[-1][2]
    cases["tied_ends"] = chunk(c0 + [(qc + 10, 0, rc + 5, 0), (qc + 10, 0, rc + 15, 0)])
    # score thresholds: a 3-anchor chain (40, dropped); 4-anchor chains with gap sums 15 (45, kept) and 16 (44, dropped)
    cases["three_anchors"] = chunk(diag(100, 100, [(100, 100)] * 2))
    cases["gapsum_15"] = chunk(diag(100, 100, [(100, 105), (100, 105), (100, 105)]))
    cases["gapsum_16"] = chunk(diag(100, 100, [(100, 105), (100, 105), (100, 106)]))
    # a 3-anchor component whose best path has 2 anchors (two anchors chain from one)
    cases["branch"] = chunk([(100, 0, 100, 0), (200, 0, 200, 0), (200, 0, 210, 0)])
    # positions past 2^31 and up to the sketch bound; ref position 0 on the reverse strand; the largest ref contig
    cases["high_pos"] = chunk(diag(2**31 + 5, 2**31 + 7, [(100, 100)] * 5) + diag(TOP - 500, TOP - 400, [(100, 100)] * 4, rctg=3))
    cases["rev_r0"] = chunk(diag(100, 400, [(100, 100)] * 4, rev=1))
    cases["ctg_max"] = chunk(diag(100, 100, [(100, 100)] * 4, rctg=CTG_MAX) + diag(150, 900, [(100, 100)] * 4, rctg=CTG_MAX, rev=1))
    return cases


def check_dp_edges(cases, o_by_case, band):
    """the constructed DP cases reach their edges (in the oracle, which the device then has to match)"""
    def last(name, key):
        return int(o_by_case[name][key][-1])
    n = len(cases["band_0"]) - 1
    assert last("band_0", "pointer") == 0 and last("band_0", "score") == 20, "predecessor at distance band chains"
    assert last("band_1", "pointer") == n + 1, "predecessor at band + 1 does not"
    assert len(o_by_case["qgap_2500"]["intervals"]) == 1 and len(o_by_case["qgap_2501"]["intervals"]) == 0
    assert last("diag_gap_300", "score") == 20 and last("diag_gap_301", "score") == 0
    assert last("diag_gap_300_rev", "score") == 20 and last("diag_gap_301_rev", "score") == 0
    assert o_by_case["gapsum_15"]["intervals"][:, 0].tolist() == [45] and len(o_by_case["gapsum_16"]["intervals"]) == 0
    assert len(o_by_case["three_anchors"]["intervals"]) == 0 and len(o_by_case["branch"]["intervals"]) == 0
    assert o_by_case["tied_ends"]["intervals"][0, 5] == cases["tied_ends"][-1, 3], "the larger index ends the chain"
    assert o_by_case["rev_r0"]["intervals"][0, 4] == 0
    n_tie = 0
    for name, ch in cases.items():
        if name.startswith("tie_"):
            j2 = len(ch) - 1 - int(name.split("_")[3])
            assert last(name, "pointer") == j2 and last(name, "score") == 10, name
            n_tie += 1
    assert n_tie >= band


def length_cases(gl, seed=1):
    """chunks of every length the group / warp arrangement treats differently, several thousand anchors included: diagonal
    chains of random small steps on two strands and contigs, with random repeat anchors"""
    rng = np.random.default_rng(seed + gl)
    cases = {}
    for n in sorted({1, 2, 3, gl - 1, gl, gl + 1, 31, 32, 33, 64, 65, 4000}):
        if n < 1:
            continue
        rows, q, r = [], 1000, [50_000, 1_000_000]
        while len(rows) < n:
            q += int(rng.integers(1, 120))
            s = int(rng.integers(0, 2))
            r[s] += int(rng.integers(1, 140)) * (1 if s == 0 else -1)
            rows.append((q, s, r[s], s))
            if rng.random() < 0.15 and len(rows) < n:
                rows.append((q, int(rng.integers(0, 3)), int(rng.integers(1, 10**6)), int(rng.integers(0, 2))))
        cases["len_%d" % n] = chunk(rows[:n], qctg=int(rng.integers(0, 5)))
    return cases


def iv(score, na, q0, q1, r0, r1, rctg=0, qctg=0, ch=0, rev=0):
    return (score, na, q0, q1, r0, r1, rctg, qctg, ch, rev)


def select_cases():
    """{name: (intervals, n_chunks)} for the selection; every list is also embedded in lists past 1,024 intervals"""
    cases = {}
    base = iv(100, 5, 1000, 2000, 5000, 6000, 1, 2, 0, 0)
    # a primary-key tie decided by each later field in turn; the two overlap, so the first in the order is the one kept
    for f, name in enumerate(("q0", "q1", "r0", "r1", "rctg", "qctg", "chunk", "rev")):
        other = list(base)
        other[2 + f] += 1
        cases["tie_" + name] = ([base, tuple(other)], 2)
    cases["identical"] = ([base, base, base], 1)
    # summed overlap of exactly floor(len / 2) and floor(len / 2) - 1, odd and even lengths, ref / query / both axes
    for L in (1000, 1001):
        for h in (L // 2, L // 2 - 1):
            c_r = iv(50, 4, 100_000, 101_000, 10_000, 10_000 + L)
            a_r = iv(90, 4, 500_000, 501_000, 10_000 + L - h, 20_000)
            c_q = iv(50, 4, 10_000, 10_000 + L, 700_000, 701_000)
            a_q = iv(90, 4, 10_000 + L - h, 20_000, 300_000, 301_000)
            a_b = iv(90, 4, 10_000 + L - h, 20_000, 10_000 + L - h, 20_000)
            cases["half_ref_%d_%d" % (L, h)] = ([c_r, a_r], 1)
            cases["half_query_%d_%d" % (L, h)] = ([c_q, a_q], 1)
            c_b = iv(50, 4, 10_000, 10_000 + L, 10_000, 10_000 + L)
            cases["half_both_%d_%d" % (L, h)] = ([c_b, a_b], 1)
            # the sum of two overlaps, one on each side
            a1 = iv(90, 4, 800_000, 801_000, 10_000 - 500, 10_000 + h // 2)
            a2 = iv(80, 4, 900_000, 901_000, 10_000 + L - (h - h // 2), 30_000)
            cases["half_sum_%d_%d" % (L, h)] = ([c_r, a1, a2], 1)
    cases["touching"] = ([iv(90, 4, 0, 1000, 0, 1000), iv(50, 4, 1000, 2000, 1000, 2000)], 1)
    cases["other_contig"] = ([iv(90, 4, 0, 1000, 0, 1000, 0, 0), iv(50, 4, 0, 1000, 0, 1000, 1, 1)], 1)
    cases["contains"] = ([iv(90, 4, 0, 10_000, 0, 10_000), iv(50, 4, 2000, 3000, 2000, 3000)], 1)
    cases["contained"] = ([iv(90, 4, 2000, 3000, 2000, 3000), iv(50, 4, 0, 10_000, 0, 10_000)], 1)
    # an overlap with a rejected earlier candidate does not count: A kept, B rejected by A, C overlaps only B
    cases["rejected_overlap"] = ([iv(90, 4, 0, 1000, 0, 1000), iv(80, 4, 100, 2000, 100, 2000), iv(70, 4, 1100, 1900, 1100, 1900)], 1)
    # exactly 4 / 5 earlier overlapping candidates of the last one (the dependency lists hold 4); in the 5-case all but one of
    # them are rejected, and the accepted one overlaps the last candidate by less than half
    for k in (4, 5):
        lst = [iv(200, 9, 50_000, 51_000, 0, 300)]                                 # kept, overlaps the last by 300 of 1000
        lst += [iv(190 - t, 9, 50_000 + t, 51_000, 10 + t, 900) for t in range(k - 1)]   # rejected by the first
        lst.append(iv(10, 3, 60_000, 61_000, 0, 1000))
        cases["deps_%d" % k] = (lst, 1)
        lst = [iv(200 - t, 9, 1000 * t, 1000 * t + 900, 200 * t, 200 * t + 110) for t in range(k)]   # all kept, disjoint
        # contributions min(c.r1 - a.r0, a.r1 - c.r0) = 110, 310, 510, 710, 910: 1,640 of 5,000 (kept) with 4, 2,550 with 5
        lst.append(iv(10, 3, 90_000, 91_000, 0, 5000))
        cases["deps_kept_%d" % k] = (lst, 1)
    # spans of 32 and 33 bitmap cells (ref spans past 512 kb): a higher-scoring accepted interval overlaps the candidate only in
    # its last ref cell and nowhere on the query axis, so only that cell tells the bitmap that the candidate must be scanned
    # (32 cells: the bitmap check covers it; 33: too wide for the check, always scanned).  The overlap is far below half the
    # candidate, which stays kept: the scan shows in the per-axis hit counts, not in the kept flag.
    for n_cells in (32, 33):
        s, e = 7 * CELL, 7 * CELL + n_cells * CELL
        cases["cells_%d" % n_cells] = ([iv(90, 4, 5_000_000, 5_001_000, e - 100, e + 5000),
                                         iv(50, 4, 9_000_000, 9_001_000, s, e)], 1)
    x = 3639 + 10                           # sel_cell_hash(0, x) == sel_cell_hash(1, 10)
    cases["cell_collision"] = ([iv(90, 4, x * CELL + 5, x * CELL + 900, x * CELL + 5, x * CELL + 900, 0, 0),
                                iv(50, 4, 10 * CELL + 5, 10 * CELL + 900, 10 * CELL + 5, 10 * CELL + 900, 1, 1)], 1)
    hi = 2**32 - 1
    cases["near_2_32"] = ([iv(90, 4, hi - 3000, hi, hi - 5000, hi - 1), iv(50, 4, hi - 1700, hi - 1, hi - 2000, hi), iv(40, 4, 0, hi, 0, hi, 2, 2)], 1)
    return cases


def random_intervals(n, seed, n_chunks=50):
    """n intervals crowded onto few contigs and positions: many overlaps, ties and dependency lists of every length"""
    rng = np.random.default_rng(seed)
    q0 = rng.integers(0, 200_000, n); r0 = rng.integers(0, 200_000, n)
    ql = rng.integers(1, 6000, n); rl = rng.integers(1, 6000, n)
    sc = rng.integers(45, 90, n); na = rng.integers(3, 6, n)
    return [iv(int(sc[i]), int(na[i]), int(q0[i]), int(q0[i] + ql[i]), int(r0[i]), int(r0[i] + rl[i]), int(rng.integers(0, 3)),
               int(rng.integers(0, 3)), int(rng.integers(0, n_chunks)), int(rng.integers(0, 2))) for i in range(n)]


def padded(lst, n, seed):
    """lst followed by lower-scoring intervals far away from it and from each other, n in all (the shared-memory vs global
    path of select_kernel is chosen by the list length)"""
    rng = np.random.default_rng(seed)
    out = list(lst)
    t = 0
    while len(out) < n:
        q = 10**9 + 4000 * t
        out.append(iv(int(rng.integers(1, 9)), 3, q, q + 1000, q, q + 1000, 50 + t % 7, 60 + t % 5, 0, t % 2))
        t += 1
    return out
