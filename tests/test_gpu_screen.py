"""GPU marker screen (screen.cu) against the CPU oracle, pair list by pair list, on fabricated markers-only sketch sets whose
shared-marker counts are known by construction.  Every entry point is compared: sk_screen_triangle, sk_screen_triangle_rows
(row_mod 3), sk_screen_triangle_block over several cuts (the incremental table and the one-shot screen of SK_FULL_RESCREEN),
sk_screen_query_ref in modes 0-3 with rescue on and off, and sk_screen_query_ref_multi with 2 and 3 contexts on one device.

Families: shared counts at thr - 1, thr and thr + 1 for every step of thr = max(floor(0.8^21 * mn), 1) and at screen_val 0.95
and 0.99; genomes with 0, 1, 19, 20 and 21 markers on either side (rescue); 100,000 genomes, i.e. three 49,152-column tiles of
screen_rows_kernel / ts_rows_kernel, with planned pairs on each side of every tile boundary, a rescued row and a marker shared by
thousands of genomes; more passing pairs than the first pair buffer holds (max(2^20, 64 * rows)); markers at both ends of the
42-bit range (prefix buckets 0 and 65,535 of the incremental table); empty genomes and sets.  The largest sets are also checked
against a scipy.sparse incidence product A * A^T with the predicate of src/screen.rs written out in numpy.  Each test asserts
that it reached the edge it is named for.  Import refuses markers >= 2^42 and seed k-mers >= 4^k, which would alias another
genome's entries."""
import os

import numpy as np
import pytest
import scipy.sparse as sps

import oracle_py as O

pytestmark = pytest.mark.gpu

TILE = 48 * 1024                 # columns per shared-memory tile of screen_rows_kernel / ts_rows_kernel
CAP0 = 1 << 20                   # first pair-buffer capacity: max(2^20, 64 * rows)
SMALL = 20                       # SCREEN_MINIMUM_KMERS (src/params.rs:49)
SHARED_BASE = 1 << 30            # marker values of planned shared markers ...
BG_BASE = 1 << 36                # ... and of every genome's own background markers (all < 2^42)
U64 = np.uint64


@pytest.fixture(scope="module")
def ctxs():
    import skani_b200 as sk
    cs = [sk.Context(0) for _ in range(3)]
    yield cs
    for c in cs:
        c.close()


# ---------------------------------------------------------------------------------------------------------------------
# fabricated marker sets
# ---------------------------------------------------------------------------------------------------------------------
def powi21(x):
    """f64::powi(x, 21) as __powidf2 evaluates it (square-and-multiply from the low bit)"""
    r, a, b = 1.0, float(x), 21
    while True:
        if b & 1:
            r *= a
        b //= 2
        if b == 0:
            break
        a *= a
    return r


def cutoff_of(sv):
    return powi21(0.80 if sv == 0 else sv)


def thr_of(sv, mn):
    return max(int(cutoff_of(sv) * mn), 1)


def plan(cards, groups, bg_base=BG_BASE):
    """Markers-only genomes: genome g has exactly cards[g] markers.  groups[k] lists the genomes holding planned shared marker
    SHARED_BASE + k; every other marker of a genome is its own.  Returns (mk_off, markers), genome-major."""
    cards = np.asarray(cards, np.int64)
    n = len(cards)
    gs = [np.asarray(g, np.int64) for g in groups]
    for g in gs:
        assert len(np.unique(g)) == len(g)
    sg = np.concatenate(gs) if gs else np.zeros(0, np.int64)
    sm = np.repeat(SHARED_BASE + np.arange(len(gs), dtype=np.int64), [len(g) for g in gs])
    bg = cards - np.bincount(sg, minlength=n)
    assert bg.min() >= 0, "a genome holds more shared markers than its card"
    bgg = np.repeat(np.arange(n, dtype=np.int64), bg)
    g_all = np.concatenate([sg, bgg])
    m_all = np.concatenate([sm, bg_base + np.arange(len(bgg), dtype=np.int64)])
    order = np.argsort(g_all, kind="stable")
    off = np.concatenate([[0], np.cumsum(cards)]).astype(U64)
    return off, m_all[order].astype(U64)


def share(groups, a, b, s):
    """a and b share s planned markers"""
    groups.extend([[a, b]] * s)


def subset(off, mk, genomes):
    genomes = np.asarray(genomes, np.int64)
    cards = (off[genomes + 1] - off[genomes]).astype(np.int64)
    parts = [mk[int(off[g]):int(off[g + 1])] for g in genomes]
    return np.concatenate([[0], np.cumsum(cards)]).astype(U64), (np.concatenate(parts) if parts else np.zeros(0, U64)).astype(U64)


def cards_of(off):
    return np.diff(off.astype(np.int64))


def device_set(ctx, off, mk):
    import skani_b200 as sk
    return sk.import_sketches(ctx, [dict(markers=mk[int(off[g]):int(off[g + 1])], total_len=0) for g in range(len(off) - 1)], seeds=False)


def oracle_set(off, mk):
    return O.sketches_from_markers(off, mk)


def pid(a, b):
    return (int(a) << 32) | int(b)


def as_set(pairs):
    return set(pairs.tolist())


def all_pairs_triangle(n):
    i, j = np.triu_indices(n, 1)
    return (i.astype(U64) << U64(32)) | j.astype(U64)


# ---- independent reference: incidence product with the predicate of src/screen.rs ---------------------------------------
def incidence(off, mk, universe):
    cards = cards_of(off)
    g = np.repeat(np.arange(len(cards)), cards)
    col = np.searchsorted(universe, mk)
    return sps.csr_matrix((np.ones(len(mk), np.int64), (g, col)), shape=(len(cards), len(universe)))


def sparse_triangle(off, mk, sv, rescue):
    cards = cards_of(off)
    universe = np.unique(mk)
    a = incidence(off, mk, universe)
    c = sps.triu(a @ a.T, k=1).tocoo()
    i, j, cnt = c.row.astype(np.int64), c.col.astype(np.int64), c.data
    mn = np.minimum(cards[i], cards[j]).astype(np.float64)
    thr = np.maximum((cutoff_of(sv) * mn).astype(np.int64), 1)                 # screen_refs, src/screen.rs:177-187
    keep = cnt > thr
    parts = [(i[keep].astype(U64) << U64(32)) | j[keep].astype(U64)]
    if rescue:                                                                   # src/screen.rs:158-160: the row decides
        for r in np.nonzero(cards < SMALL)[0]:
            parts.append((U64(r) << U64(32)) | np.arange(r + 1, len(cards), dtype=U64))
    return np.unique(np.concatenate(parts))


def sparse_query_ref(r_off, r_mk, q_off, q_mk, sv, mode, rescue):
    rc, qc = cards_of(r_off), cards_of(q_off)
    universe = np.unique(np.concatenate([r_mk, q_mk]))
    cnt = (incidence(q_off, q_mk, universe) @ incidence(r_off, r_mk, universe).T).toarray()    # [query, ref]
    mn = np.minimum(qc[:, None], rc[None, :])
    v = (cutoff_of(sv) * mn.astype(np.float64)).astype(np.int64)
    if mode >= 2:                                                                # screen_refs / screen_refs_indices
        ok = cnt > np.maximum(v, 1)
        if mode == 2 and rescue:
            ok[qc < SMALL, :] = True
    else:                                                                        # check_markers_quickly
        rs = mode == 0 and rescue
        ok = cnt >= np.maximum(v, 1)
        ok[mn == 0] = rs
        if rs:
            ok[mn < SMALL] = True
    q, r = np.nonzero(ok)
    return np.sort((r.astype(U64) << U64(32)) | q.astype(U64))


# ---- comparisons ----------------------------------------------------------------------------------------------------
def assert_same(got, want, what):
    assert got.dtype == U64, what
    assert len(got) < 2 or bool(np.all(got[1:] > got[:-1])), "%s: not sorted or duplicated" % what
    if not np.array_equal(got, want):
        g, w = as_set(got), as_set(want)
        miss, extra = sorted(w - g), sorted(g - w)
        raise AssertionError("%s: %d pairs, want %d; missing %s, extra %s" % (
            what, len(got), len(want), [(p >> 32, p & 0xFFFFFFFF) for p in miss[:8]], [(p >> 32, p & 0xFFFFFFFF) for p in extra[:8]]))


def check_triangle(ctx, s, want, mp, cuts):
    """every triangle entry point on set s against the full pair list `want`"""
    import skani_b200 as sk
    assert_same(sk.screen_triangle(ctx, s, mp), want, "sk_screen_triangle")
    rows, cols = want >> U64(32), want & U64(0xFFFFFFFF)
    for rem in range(3):
        assert_same(sk.screen_triangle_rows(ctx, s, 3, rem, mp), want[rows % U64(3) == U64(rem)], "sk_screen_triangle_rows(3, %d)" % rem)
    for g0, g1 in zip(cuts[:-1], cuts[1:]):
        w = want[(cols >= U64(g0)) & (cols < U64(g1))]
        assert_same(sk.screen_triangle_block(ctx, s, g0, g1, mp), w, "sk_screen_triangle_block(%d, %d)" % (g0, g1))
        os.environ["SK_FULL_RESCREEN"] = "1"
        try:
            assert_same(sk.screen_triangle_block(ctx, s, g0, g1, mp), w, "sk_screen_triangle_block(%d, %d), one-shot" % (g0, g1))
        finally:
            del os.environ["SK_FULL_RESCREEN"]


def triangle_case(ctx, off, mk, sv, rescue, cuts, sparse=False):
    """oracle list (and the incidence product's) == every GPU entry point; returns the list"""
    import skani_b200 as sk
    want = O.screen_triangle_pairs(oracle_set(off, mk), sv, rescue)
    if sparse:
        assert_same(sparse_triangle(off, mk, sv, rescue), want, "incidence product")
    s = device_set(ctx, off, mk)
    check_triangle(ctx, s, want, sk.map_params(screen_val=sv, rescue_small=rescue), cuts)
    s.free()
    return want


def query_ref_case(ctx, r_off, r_mk, q_off, q_mk, sv, rescues=(True, False), sparse=False, rset=None, qset=None):
    """sk_screen_query_ref in modes 0-3 == the oracle's list; returns {(mode, rescue): list}"""
    import skani_b200 as sk
    ro, qo = oracle_set(r_off, r_mk), oracle_set(q_off, q_mk)
    rs = rset or device_set(ctx, r_off, r_mk)
    qs = qset or device_set(ctx, q_off, q_mk)
    out = {}
    for rescue in rescues:
        for mode in range(4):
            want = O.screen_query_ref(ro, qo, sv, mode, rescue)
            if sparse:
                assert_same(sparse_query_ref(r_off, r_mk, q_off, q_mk, sv, mode, rescue), want, "incidence product, mode %d" % mode)
            got = sk.screen_query_ref(ctx, rs, qs, sk.map_params(screen_val=sv, rescue_small=rescue), mode)
            assert_same(got, want, "sk_screen_query_ref mode %d rescue %d" % (mode, rescue))
            out[(mode, rescue)] = want
    return out


# ---------------------------------------------------------------------------------------------------------------------
# 1. threshold edges
# ---------------------------------------------------------------------------------------------------------------------
MNS = (20, 108, 109, 216, 217, 325, 326, 1000, 5000)


def threshold_plan(sv):
    """pair p = genomes (2p, 2p + 1): the smaller one has mn markers, the other mn + 37; they share `count` markers"""
    cards, groups, meta = [], [], []
    for mn in MNS:
        t = thr_of(sv, mn)
        for count in sorted({0, 1, t - 1, t, t + 1, mn}):
            for small_first in (True, False):
                a, b = len(cards), len(cards) + 1
                cards += [mn, mn + 37] if small_first else [mn + 37, mn]
                share(groups, a, b, count)
                meta.append((mn, t, count, small_first))
    return cards, groups, meta


@pytest.mark.parametrize("sv", [0.0, 0.95, 0.99])
def test_threshold_edges(ctxs, sv):
    ctx = ctxs[0]
    cards, groups, meta = threshold_plan(sv)
    off, mk = plan(cards, groups)
    n = len(cards)
    tri = as_set(triangle_case(ctx, off, mk, sv, True, [0, 1, n // 2, n - 1, n]))
    roff, rmk = subset(off, mk, range(0, n, 2))                 # pair p: ref p, query p
    qoff, qmk = subset(off, mk, range(1, n, 2))
    qr = {k: as_set(v) for k, v in query_ref_case(ctx, roff, rmk, qoff, qmk, sv).items()}
    on_thr = below = 0
    for p, (mn, t, count, small_first) in enumerate(meta):
        in_tri, key = pid(2 * p, 2 * p + 1) in tri, pid(p, p)
        assert in_tri == (count > t), (mn, count, small_first)
        for rescue in (True, False):
            assert (key in qr[(2, rescue)]) == (key in qr[(3, rescue)]) == (count > t), (mn, count, rescue)
            assert (key in qr[(0, rescue)]) == (key in qr[(1, rescue)]) == (count >= t), (mn, count, rescue)
        if count == t:            # the quick screen passes, screen_refs does not
            on_thr += 1
            assert key in qr[(0, False)] and key not in qr[(2, False)] and not in_tri
        below += count == t - 1 and count >= 1
    assert on_thr >= 2 * len(MNS) and below > 0
    if sv == 0.95:
        assert thr_of(sv, 20) == 6 and thr_of(sv, 100) == 34
    if sv == 0.0:
        assert [thr_of(sv, m) for m in MNS] == [1, 1, 1, 1, 2, 2, 3, 9, 46]


# ---------------------------------------------------------------------------------------------------------------------
# 2. rescue of genomes with < 20 markers
# ---------------------------------------------------------------------------------------------------------------------
RESCUE_CARDS = [21, 0, 19, 20, 1, 21, 19, 0, 20, 1, 21, 19, 20, 0]


def rescue_plan():
    cards = RESCUE_CARDS
    groups = []
    share(groups, 0, 2, 1)        # large row, small column, one shared marker (= thr): fails, the column does not rescue it
    share(groups, 3, 5, 2)        # 20 / 21 with two shared markers: passes without any rescue
    share(groups, 4, 6, 1)        # 1 / 19 sharing their only marker
    share(groups, 8, 10, 1)
    share(groups, 2, 11, 3)       # 19 / 19: count 3 passes without rescue
    share(groups, 9, 12, 1)
    return plan(cards, groups)


def test_rescue_small_genomes(ctxs):
    ctx = ctxs[0]
    off, mk = rescue_plan()
    cards = np.array(RESCUE_CARDS)
    n = len(cards)
    small = [g for g in range(n) if cards[g] < SMALL]
    for rescue in (True, False):
        tri = as_set(triangle_case(ctx, off, mk, 0.0, rescue, [0, 1, 5, 13, n], sparse=True))
        for i in small[:-1] if small[-1] == n - 1 else small:   # a small row passes every later column only with rescue
            later = {pid(i, j) for j in range(i + 1, n)}
            assert (later <= tri) == rescue, (i, rescue)
        # a small column never rescues its row: (0, 1), (0, 7): row 21 markers, column 0 markers; (0, 2): column 19, count 1
        assert not {pid(0, 1), pid(0, 7), pid(0, 2), pid(3, 13), pid(5, 6)} & tri
        assert pid(3, 5) in tri and pid(2, 11) in tri
    # query x ref: every genome as ref and as query
    qr = {k: as_set(v) for k, v in query_ref_case(ctx, off, mk, off, mk, 0.0, sparse=True).items()}
    for r in range(n):
        for q in range(n):
            mn, key = min(cards[r], cards[q]), pid(r, q)
            # mode 0: min(|Mi|, |Mj|) < 20 passes with rescue; 0 markers passes only with rescue
            if mn < SMALL:
                assert key in qr[(0, True)], (r, q)
            if mn == 0:
                assert key not in qr[(0, False)] and key not in qr[(1, True)] and key not in qr[(1, False)]
                assert key not in qr[(3, True)] and key not in qr[(3, False)]
            # mode 2: the query (row) decides; a small ref does not rescue a large query
            assert (key in qr[(2, True)]) == (cards[q] < SMALL or key in qr[(2, False)]), (r, q)
    assert qr[(1, True)] == qr[(1, False)] and qr[(3, True)] == qr[(3, False)]      # modes 1 and 3 never rescue
    assert pid(1, 0) in qr[(0, True)] and pid(0, 1) in qr[(0, True)] and pid(0, 1) in qr[(2, True)] and pid(1, 0) not in qr[(2, True)]


# ---------------------------------------------------------------------------------------------------------------------
# 3. three column tiles: 100,000 genomes
# ---------------------------------------------------------------------------------------------------------------------
N_TILE = 100_000
RESCUE_ROW = 3
ROW_TILE_ROWS = (0, 5, 1000)                                     # screen_rows_kernel rows: tiles start at i + 1
TS_COLS = (0, 49_151, 49_152, 98_303, 98_304)                    # ts_rows_kernel / query x ref tiles start at 0
LAST = N_TILE - 1
N_Q, N_SMALL_Q = 6, 20


def tile_plan():
    """genomes [0, N_TILE): the triangle / ref set; then N_Q queries; then N_SMALL_Q queries with 5 markers each"""
    n = N_TILE + N_Q + N_SMALL_Q
    cards = np.full(n, 30, np.int64)
    cards[RESCUE_ROW] = 10
    groups = []
    planned = []
    for i in ROW_TILE_ROWS:
        for d in (TILE - 1, TILE, 2 * TILE):
            planned.append((i, i + 1 + d))
    for c in TS_COLS:
        planned += [(c, LAST), (c, 98_305)]
    planned += [(LAST - 1, LAST), (49_150, 49_151)]
    planned = sorted(set(planned))
    for a, b in planned:
        share(groups, a, b, 2)
    fail_pairs = [(1, 1 + TILE), (49_151, 98_304), (2, LAST)]    # one shared marker: count == thr, screen_refs fails
    for a, b in fail_pairs:
        share(groups, a, b, 1)
    busy = {g for p in planned + fail_pairs for g in p} | {RESCUE_ROW}
    hub = [g for g in range(11, N_TILE, 37) if g not in busy]    # ~2,700 genomes in all three tiles share one marker ...
    q = N_TILE
    groups.append(hub + [q + 3])                                 # ... and so does query 3
    for r in (0, 49_151, 49_152, 98_303, 98_304, LAST):
        share(groups, q, r, 2)                                   # query 0: two shared markers on both sides of each boundary
    for r in (1, 49_153, 98_305):
        share(groups, q, r, 1)                                   # ... and one (= thr) next to them
    cards[q + 1] = 10                                            # query 1: small (rescued in modes 0 and 2)
    share(groups, q + 1, 49_152, 1)
    cards[q + 2] = 0                                             # query 2: no markers
    share(groups, q + 4, LAST, 3)                                # query 4
    share(groups, q + 4, 0, 2)
    cards[N_TILE + N_Q:] = 5                                     # 20 small queries, nothing shared
    off, mk = plan(cards, groups)
    return off, mk, planned, fail_pairs, hub


@pytest.fixture(scope="module")
def tiles(ctxs):
    off, mk, planned, fail_pairs, hub = tile_plan()
    t_off, t_mk = subset(off, mk, range(N_TILE))
    q_off, q_mk = subset(off, mk, range(N_TILE, N_TILE + N_Q))
    s_off, s_mk = subset(off, mk, range(N_TILE + N_Q, N_TILE + N_Q + N_SMALL_Q))
    ctx = ctxs[0]
    d = dict(t=(t_off, t_mk), q=(q_off, q_mk), small=(s_off, s_mk), planned=planned, fail_pairs=fail_pairs, hub=hub,
             tset=device_set(ctx, t_off, t_mk), qset=device_set(ctx, q_off, q_mk))
    yield d
    d["tset"].free(); d["qset"].free()


def test_triangle_column_tiles(ctxs, tiles):
    ctx = ctxs[0]
    import skani_b200 as sk
    t_off, t_mk = tiles["t"]
    assert N_TILE > 2 * TILE and len(tiles["hub"]) > 2000
    hub = np.array(tiles["hub"])
    assert hub.min() < TILE and ((hub >= TILE) & (hub < 2 * TILE)).any() and hub.max() >= 2 * TILE
    want = O.screen_triangle_pairs(oracle_set(t_off, t_mk), 0.0, True)
    assert_same(sparse_triangle(t_off, t_mk, 0.0, True), want, "incidence product")
    check_triangle(ctx, tiles["tset"], want, sk.map_params(), [0, TILE, TILE + 1, 2 * TILE + 1, N_TILE])
    got = as_set(want)
    for a, b in tiles["planned"]:
        assert pid(a, b) in got, (a, b)
    for a, b in tiles["fail_pairs"]:
        assert pid(a, b) not in got, (a, b)
    for i in ROW_TILE_ROWS:       # screen_rows_kernel: last column of tile 0, first of tile 1, first of tile 2
        assert {pid(i, i + 1 + TILE - 1), pid(i, i + 1 + TILE), pid(i, i + 1 + 2 * TILE)} <= got
    for c in TS_COLS:             # ts_rows_kernel: first / last column of every tile, the last genome as row
        assert pid(c, LAST) in got
    rescued = want[(want >> U64(32)) == U64(RESCUE_ROW)]
    assert np.array_equal(rescued & U64(0xFFFFFFFF), np.arange(RESCUE_ROW + 1, N_TILE, dtype=U64))   # spans all three tiles


def test_query_ref_column_tiles(ctxs, tiles):
    import skani_b200 as sk
    t_off, t_mk = tiles["t"]
    q_off, q_mk = tiles["q"]
    qr = query_ref_case(ctxs[0], t_off, t_mk, q_off, q_mk, 0.0, sparse=True, rset=tiles["tset"], qset=tiles["qset"])
    s2 = {k: as_set(v) for k, v in qr.items()}
    for r in (0, 49_151, 49_152, 98_303, 98_304, LAST):
        assert all(pid(r, 0) in s2[(m, False)] for m in range(4)), r
    for r in (1, 49_153, 98_305):                                # count == thr: modes 0 / 1 only
        assert pid(r, 0) in s2[(1, False)] and pid(r, 0) not in s2[(3, False)], r
    assert len(qr[(0, True)][(qr[(0, True)] & U64(0xFFFFFFFF)) == U64(1)]) == N_TILE      # small query: rescued everywhere
    assert len(qr[(2, True)][(qr[(2, True)] & U64(0xFFFFFFFF)) == U64(2)]) == N_TILE      # 0 markers: rescued by mode 2
    assert len(qr[(1, True)][(qr[(1, True)] & U64(0xFFFFFFFF)) == U64(3)]) == len(tiles["hub"])   # hub query, all tiles
    # the same lists over 2 and 3 contexts on one device, blocks cut on and next to tile boundaries
    qcopies = [tiles["qset"]] + [tiles["qset"].copy_to(c) for c in ctxs[1:]]
    for cuts in ([0, TILE], [0, TILE - 1, 60_000], [0, TILE + 1, 2 * TILE]):
        cs = ctxs[:len(cuts)]
        b = cuts + [N_TILE]
        sets = [device_set(cs[d], *subset(t_off, t_mk, range(b[d], b[d + 1]))) for d in range(len(cuts))]
        for (mode, rescue), want in qr.items():
            got = sk.screen_query_ref_multi(cs, sets, cuts, qcopies[:len(cuts)], sk.map_params(rescue_small=rescue), mode)
            assert_same(got, want, "sk_screen_query_ref_multi %s mode %d rescue %d" % (cuts, mode, rescue))
        for s in sets:
            s.free()
    for q in qcopies[1:]:
        q.free()


# ---------------------------------------------------------------------------------------------------------------------
# 4. more passing pairs than the first pair buffer holds
# ---------------------------------------------------------------------------------------------------------------------
def test_pair_buffer_retry_triangle(ctxs):
    n = 2600                                                     # every genome < 20 markers: with rescue every pair passes
    groups = []
    for g in range(0, n - 1, 7):
        share(groups, g, g + 1, 2)
    off, mk = plan(np.full(n, 5), groups)
    want = triangle_case(ctxs[0], off, mk, 0.0, True, [0, 1500, n])
    assert_same(want, all_pairs_triangle(n), "oracle vs every pair")
    cap = max(CAP0, 64 * n)
    rows, cols = want >> U64(32), want & U64(0xFFFFFFFF)
    assert len(want) > cap                                                         # sk_screen_triangle
    assert all(int(np.sum(rows % U64(3) == U64(r))) > cap for r in range(3))       # every row_mod-3 share
    assert int(np.sum(cols < U64(1500))) > max(CAP0, 64 * 1500)                    # both blocks
    assert int(np.sum(cols >= U64(1500))) > max(CAP0, 64 * 1100)


def test_pair_buffer_retry_query_ref(ctxs, tiles):
    t_off, t_mk = tiles["t"]
    s_off, s_mk = tiles["small"]
    qr = query_ref_case(ctxs[0], t_off, t_mk, s_off, s_mk, 0.0, rescues=(True,), rset=tiles["tset"])
    full = np.sort((np.repeat(np.arange(N_TILE, dtype=U64), N_SMALL_Q) << U64(32)) | np.tile(np.arange(N_SMALL_Q, dtype=U64), N_TILE))
    for mode in (0, 2):
        assert len(qr[(mode, True)]) > max(CAP0, 64 * N_SMALL_Q)
        assert_same(qr[(mode, True)], full, "mode %d: every pair" % mode)


# ---------------------------------------------------------------------------------------------------------------------
# 5. both ends of the 42-bit marker range
# ---------------------------------------------------------------------------------------------------------------------
def test_marker_range_extremes(ctxs):
    ctx = ctxs[0]
    top = (1 << 42) - 1
    rng = np.random.default_rng(42)
    low = np.arange(2, 3000, dtype=np.int64)                     # prefix bucket 0 of the incremental table (marker < 2^26)
    high = np.arange(top - 3000, top - 1, dtype=np.int64)        # prefix bucket 65,535 (marker >= 2^42 - 2^26)
    pool = np.concatenate([low, high])
    lists = []
    for g in range(40):
        m = rng.choice(pool, 90, replace=False)
        if g % 4 == 0:
            m = np.concatenate([m, [0, 1]])
        if g % 4 in (0, 1):
            m = np.concatenate([m, [top, top - 1]])
        lists.append(np.unique(m).astype(U64))
    off = np.concatenate([[0], np.cumsum([len(m) for m in lists])]).astype(U64)
    mk = np.concatenate(lists)
    assert (mk < U64(1 << 26)).sum() > 1000 and (mk >= U64((1 << 42) - (1 << 26))).sum() > 1000
    want = triangle_case(ctx, off, mk, 0.0, True, [0, 1, 20, 39, 40], sparse=True)
    assert pid(0, 4) in as_set(want)                             # 0, 1, 2^42 - 1 and 2^42 - 2 shared, among others
    s = device_set(ctx, off, mk)
    assert np.array_equal(s.export(0)["markers"], lists[0]) and int(s.export(0)["markers"][-1]) == top
    s.free()
    roff, rmk = subset(off, mk, range(0, 40, 2))
    qoff, qmk = subset(off, mk, range(1, 40, 2))
    query_ref_case(ctx, roff, rmk, qoff, qmk, 0.0, sparse=True)


# ---------------------------------------------------------------------------------------------------------------------
# 6. empty and degenerate sets
# ---------------------------------------------------------------------------------------------------------------------
def test_empty_and_degenerate(ctxs):
    import skani_b200 as sk
    ctx = ctxs[0]
    # one genome
    off, mk = plan([30], [])
    for rescue in (True, False):
        assert len(triangle_case(ctx, off, mk, 0.0, rescue, [0, 1])) == 0
    # every genome empty: only a rescued row passes (all of them, with rescue)
    off, mk = plan([0] * 6, [])
    assert_same(triangle_case(ctx, off, mk, 0.0, True, [0, 3, 6]), all_pairs_triangle(6), "all empty, rescue")
    assert len(triangle_case(ctx, off, mk, 0.0, False, [0, 3, 6])) == 0
    # an empty genome as first, middle and last row and column
    cards = [0, 30, 25, 0, 30, 40, 0]
    groups = []
    share(groups, 1, 2, 2); share(groups, 2, 4, 3); share(groups, 4, 5, 1); share(groups, 1, 5, 2)
    off, mk = plan(cards, groups)
    for rescue in (True, False):
        want = as_set(triangle_case(ctx, off, mk, 0.0, rescue, [0, 1, 3, 4, 6, 7]))
        assert {pid(1, 2), pid(2, 4), pid(1, 5)} <= want and pid(4, 5) not in want
        assert ({pid(0, j) for j in range(1, 7)} <= want) == rescue and ({pid(3, 6)} <= want) == rescue
        assert pid(1, 3) not in want and pid(5, 6) not in want
    query_ref_case(ctx, off, mk, off, mk, 0.0)
    # refs with no markers at all / queries with no markers at all
    e_off, e_mk = plan([0] * 4, [])
    qr = query_ref_case(ctx, e_off, e_mk, off, mk, 0.0)
    assert len(qr[(0, True)]) == 4 * 7 and len(qr[(0, False)]) == 0 and len(qr[(3, True)]) == 0
    qr = query_ref_case(ctx, off, mk, e_off, e_mk, 0.0)
    assert len(qr[(2, True)]) == 7 * 4 and len(qr[(2, False)]) == 0 and len(qr[(1, True)]) == 0


# ---------------------------------------------------------------------------------------------------------------------
# 7. import refuses keys that would alias another genome
# ---------------------------------------------------------------------------------------------------------------------
def test_import_refuses_out_of_range_keys(ctxs):
    import skani_b200 as sk
    ctx = ctxs[0]
    top = (1 << 42) - 1
    with pytest.raises(sk.host.SkaniError, match="marker out of range"):
        sk.import_sketches(ctx, [dict(markers=np.array([5], U64), total_len=0), dict(markers=np.array([7, 1 << 42], U64), total_len=0)],
                           seeds=False)
    rec = lambda k: dict(kmer=np.array([3, k], np.uint32), pos=np.array([10, 20], np.uint32), cc=np.array([0, 1], np.uint32),
                         markers=np.array([9], U64), contig_lengths=np.array([1000], np.uint32))
    with pytest.raises(sk.host.SkaniError, match="k-mer out of range"):
        sk.import_sketches(ctx, [rec(4 ** 15)], sk.sketch_params(k=15))
    with pytest.raises(sk.host.SkaniError, match="k-mer out of range"):
        sk.import_sketches(ctx, [rec(4 ** 13)], sk.sketch_params(k=13))
    # the largest legal values import, and the context still imports and screens
    ok = sk.import_sketches(ctx, [rec(4 ** 15 - 1)], sk.sketch_params(k=15))
    assert int(ok.export(0)["kmer"].max()) == 4 ** 15 - 1
    s = sk.import_sketches(ctx, [dict(markers=np.array([top, 1, 2, 3], U64), total_len=0),
                                 dict(markers=np.arange(100, 130, dtype=U64), total_len=0),
                                 dict(markers=np.array([top, 1, 2, 4], U64), total_len=0)], seeds=False)
    assert int(s.export(0)["markers"][-1]) == top
    assert_same(sk.screen_triangle(ctx, s, sk.map_params(rescue_small=False)), np.array([pid(0, 2)], U64), "after a refused import")
    for x in (ok, s):
        x.free()
