"""The chain back end's banded DP (dp_group_kernel / dp_warp_kernel) and interval selection (select_kernel) on constructed
anchor and interval lists, against the oracle, edge by edge (tests/dp_select_cases.py).

a. sk_debug_chain_anchors under every DP instantiation sk_chain_pairs can choose (group 4x5, 4x6, 8x3 with and without
   FULLBAND, the register cap lifted, warp NB 2 / 4 / 8 / 16): score and pointer of every anchor, every field of every sorted
   interval with its kept flag, the five per-chunk sums of the selection and the pair's summed chain length and chain count
   equal the oracle's (chain_anchors_ani, get_chain_intervals, get_nonoverlapping_chains on the same chunks).
b. sk_debug_select_intervals on given interval lists: ties of the primary key decided by each later field, overlaps of
   exactly half an interval, dependency lists of 4 and 5, bitmap spans of 32 / 33 cells, colliding cells, positions near 2^32,
   in lists of 1 to 3,000 intervals (select_kernel's shared-memory and global-memory paths), switched on and off.
A mismatch names the case, the anchor / interval / chunk and the field."""
import numpy as np
import pytest

import dp_select_cases as D
import oracle_py as O

pytestmark = pytest.mark.gpu
K = 15
IV_FIELDS = ("score", "num_anchors", "q0", "q1", "r0", "r1", "ref_contig", "query_contig", "chunk", "reverse", "kept")
ACC_FIELDS = ("total_anchors", "rq0", "rq1", "tbcq", "n_int")

# (c, environment hooks, band, instantiation sk_chain_pairs picks)
CONFIGS = [
    (125, {}, 20, "group 4x5 FULLBAND"),
    (150, {}, 16, "group 4x5"),
    (104, {}, 24, "group 4x6 FULLBAND"),
    (110, {}, 22, "group 4x6"),
    (104, {"SK_DP_GL": "8"}, 24, "group 8x3 FULLBAND"),
    (125, {"SK_DP_GL": "8"}, 20, "group 8x3"),
    (125, {"SK_DP_MINB": "1"}, 20, "group 4x5 FULLBAND uncapped"),
    (125, {"SK_DP_WARP": "1"}, 20, "warp NB 2"),
    (80, {}, 31, "warp NB 2"),
    (78, {}, 32, "warp NB 4"),
    (27, {}, 92, "warp NB 4"),
    (26, {}, 96, "warp NB 8"),
    (12, {}, 208, "warp NB 8"),
    (11, {}, 227, "warp NB 16"),
    (6, {}, 416, "warp NB 16"),
]


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def first_diff(got, exp, what, names):
    """message naming the first row / column where two 2-D tables differ"""
    got = np.asarray(got, np.int64).reshape(len(exp), -1) if len(exp) else np.asarray(got, np.int64)
    exp = np.asarray(exp, np.int64)
    if got.shape != exp.shape:
        return "%s: %s rows on the device, %s in the oracle" % (what, got.shape, exp.shape)
    bad = np.argwhere(got != exp)
    if len(bad) == 0:
        return None
    i, f = bad[0]
    return "%s %d, field %s: device %d, oracle %d" % (what, i, names[f], got[i, f], exp[i, f])


def compare_selection(tag, g, o):
    msg = (first_diff(g["intervals"], o["intervals"], "interval", IV_FIELDS) or
           first_diff(g["chunk_stats"][:, :5], o["chunk_acc"], "chunk", ACC_FIELDS))
    assert msg is None, "%s: %s" % (tag, msg)
    assert (g["pair_sumlen"], g["pair_nchains"]) == (o["pair_sumlen"], o["pair_nchains"]), \
        "%s: pair_sumlen / pair_nchains: device %s, oracle %s" % (tag, (g["pair_sumlen"], g["pair_nchains"]),
                                                                   (o["pair_sumlen"], o["pair_nchains"]))


@pytest.mark.parametrize("c,hooks,band,kernel", CONFIGS, ids=["c%d_%s" % (c, k.replace(" ", "_")) for c, _, _, k in CONFIGS])
def test_dp_against_oracle(ctx, monkeypatch, c, hooks, band, kernel):
    import skani_b200 as sk
    assert 2500 // c == band
    for var in ("SK_DP_GL", "SK_DP_WARP", "SK_DP_MINB"):
        monkeypatch.delenv(var, raising=False)
    for var, v in hooks.items():
        monkeypatch.setenv(var, v)
    gl = 8 if hooks.get("SK_DP_GL") == "8" else 4
    edge = D.dp_cases(band, gl)
    lens = D.length_cases(gl, seed=c)
    # pair 0: every edge case, one chunk each; pair 1: chunks of very different lengths (they share warps after the size
    # sort); pair 2: the same, switched
    pairs = [list(edge.items()), list(lens.items()), list(lens.items())]
    switched = [0, 0, 1]
    got = sk.host.debug_chain_anchors(ctx, c, K, [[ch for _, ch in p] for p in pairs], switched)
    for pi, (p, g) in enumerate(zip(pairs, got)):
        o = O.chain_chunks([ch for _, ch in p], c, K, switched[pi])
        names = [nm for nm, ch in p for _ in range(len(ch))]
        assert np.array_equal(g["anchors"], np.concatenate([ch for _, ch in p])), "anchors round trip"
        for key in ("score", "pointer"):
            bad = np.nonzero(g[key].astype(np.int64) != o[key].astype(np.int64))[0]
            assert len(bad) == 0, "%s pair %d: anchor %d (case %s), field %s: device %d, oracle %d" % (
                kernel, pi, bad[0], names[bad[0]], key, g[key][bad[0]], o[key][bad[0]])
        compare_selection("%s pair %d" % (kernel, pi), g, o)
        assert len(o["intervals"]) > 0
    # the edges are reached: per case, the oracle's DP outcome is the one the case was built for
    o_by_case = {nm: O.chain_chunks([ch], c, K) for nm, ch in edge.items()}
    D.check_dp_edges(edge, o_by_case, band)


def select_pairs():
    """(name, intervals, n_chunks) of every selection case, alone and embedded in lists of 1,023 to 2,100 intervals, and
    random crowded lists of 1 to 3,000"""
    out = []
    for name, (lst, nc) in D.select_cases().items():
        out.append((name, lst, nc))
        for n in (1023, 1024, 1025, 2100):
            out.append(("%s_in_%d" % (name, n), D.padded(lst, n, seed=n), nc))
    for n in (1, 2, 31, 1023, 1024, 1025, 3000):
        out.append(("random_%d" % n, D.random_intervals(n, seed=n), 50))
    return out


@pytest.mark.parametrize("switched", [0, 1])
def test_select_against_oracle(ctx, switched):
    import skani_b200 as sk
    cases = select_pairs()
    got = sk.host.debug_select_intervals(ctx, 125, K, [lst for _, lst, _ in cases], [nc for _, _, nc in cases], switched)
    kept_by_case, hits_by_case = {}, {}
    for (name, lst, nc), g in zip(cases, got):
        o = O.select_intervals(lst, nc, 125, K, switched)
        compare_selection("select %s switched=%d" % (name, switched), g, o)
        kept_by_case[name] = o["intervals"][:, 10].tolist()
        hits_by_case[name] = o["hits"].tolist()
    # the edges are reached
    for L in (1000, 1001):
        for axis in ("ref", "query", "both", "sum"):
            full = kept_by_case["half_%s_%d_%d" % (axis, L, L // 2)]
            assert full[-1] == (1 if L % 2 else 0) and kept_by_case["half_%s_%d_%d" % (axis, L, L // 2 - 1)][-1] == 1, (axis, L)
    assert kept_by_case["deps_4"] == [1, 0, 0, 0, 1] and kept_by_case["deps_5"] == [1, 0, 0, 0, 0, 1]
    assert kept_by_case["deps_kept_4"][-1] == 1 and kept_by_case["deps_kept_5"][-1] == 0
    assert kept_by_case["rejected_overlap"] == [1, 1, 0] and kept_by_case["touching"] == [1, 1]
    assert all(kept_by_case["tie_" + f] == [1, 0] for f in ("q0", "q1", "r0", "r1", "rctg", "qctg", "chunk", "rev"))
    # the 32 / 33-cell candidates overlap the accepted interval in their last ref cell only (the overlap is too small to reject
    # them; tests/emu/emu_dp_select.cpp checks that the bitmap sends them to the scan)
    for nc in (32, 33):
        assert kept_by_case["cells_%d" % nc] == [1, 1] and hits_by_case["cells_%d" % nc] == [[0, 0], [1, 0]], nc


def test_refuses_invalid_input(ctx):
    import skani_b200 as sk
    a = D.chunk([(100, 0, 100, 0), (200, 0, 200, 0)])
    bad = [a[::-1].copy(),                                           # unsorted
           np.array([[0, 100, 0, 100, 0], [1, 200, 0, 200, 0]], np.uint32),   # two query contigs in one chunk
           np.array([[0, 100, 2**30, 100, 0]], np.uint32),            # ref contig 2^30
           np.array([[0, 2**32 - 65536, 0, 100, 0]], np.uint32)]      # position past the sketch bound
    for x in bad:
        with pytest.raises(sk.host.SkaniError):
            sk.host.debug_chain_anchors(ctx, 125, K, [[x]])
    with pytest.raises(sk.host.SkaniError):
        sk.host.debug_select_intervals(ctx, 125, K, [[D.iv(50, 3, 10, 10, 0, 5)]], 1)     # q0 == q1
    with pytest.raises(sk.host.SkaniError):
        sk.host.debug_select_intervals(ctx, 125, K, [[D.iv(50, 3, 0, 10, 5, 5)]], 1)      # r0 == r1
