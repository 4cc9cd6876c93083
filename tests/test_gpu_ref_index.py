"""Persistent reference marker index (sk_ref_index_create / sk_ref_index_screen, screen.cu) against sk_screen_query_ref, pair
list by pair list, on the marker sets test_gpu_screen.py fabricates: counts at thr - 1, thr and thr + 1, genomes of 19, 20 and
21 markers with rescue on and off, 100,000 references (three 49,152-column tiles of screen_rows_kernel), queries and
references without markers, markers 0 and 2^42 - 1, and more passing pairs than the first pair buffer holds.  Every case is
checked in modes 0-3, with the index in one part and cut into several (SK_REF_INDEX_PART_MARKERS), and with the queries
screened in several groups whose lists, offset and concatenated, must equal the one call's."""
import numpy as np
import pytest

from test_gpu_screen import (CAP0, N_SMALL_Q, N_TILE, TILE, U64, assert_same, device_set, pid, plan, rescue_plan, share,
                             subset, thr_of, threshold_plan, tile_plan)

pytestmark = pytest.mark.gpu
MASK = U64(0xFFFFFFFF)


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def grouped(ctx, idx, q_off, q_mk, cuts, mp, mode):
    """the queries screened in groups [cuts[k], cuts[k + 1]), query ids offset back, lists concatenated and sorted"""
    parts = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        qs = device_set(ctx, *subset(q_off, q_mk, range(a, b)))
        p = idx.screen(qs, mp, mode)
        qs.free()
        parts.append((p & ~MASK) | ((p & MASK) + U64(a)))
    return np.sort(np.concatenate(parts)) if parts else np.zeros(0, U64)


def check(ctx, monkeypatch, r_off, r_mk, q_off, q_mk, sv=0.0, rescues=(True, False), part_markers=(), qcuts=None, rset=None, qset=None):
    """sk_ref_index_screen == sk_screen_query_ref for modes 0-3, with one index part and with the forced part sizes listed;
    qcuts: query groups screened separately.  Returns {(mode, rescue): list}."""
    import skani_b200 as sk
    rs = rset or device_set(ctx, r_off, r_mk)
    qs = qset or device_set(ctx, q_off, q_mk)
    want = {}
    for rescue in rescues:
        for mode in range(4):
            mp = sk.map_params(screen_val=sv, rescue_small=rescue)
            want[(mode, rescue)] = sk.screen_query_ref(ctx, rs, qs, mp, mode)
    n_refs = len(r_off) - 1
    for pm in (None,) + tuple(part_markers):
        if pm is None:
            monkeypatch.delenv("SK_REF_INDEX_PART_MARKERS", raising=False)
        else:
            monkeypatch.setenv("SK_REF_INDEX_PART_MARKERS", str(pm))
        idx = sk.RefIndex(ctx, rs)
        g, parts, nbytes = idx.info()
        assert g == n_refs and nbytes >= 12 * int(r_off[-1])
        if pm is None:
            assert parts == min(n_refs, 1)
        elif int(r_off[-1]) > pm:
            assert parts > 1, (pm, parts)
        for (mode, rescue), w in want.items():
            mp = sk.map_params(screen_val=sv, rescue_small=rescue)
            assert_same(idx.screen(qs, mp, mode), w, "ref index mode %d rescue %d parts %d" % (mode, rescue, parts))
            if qcuts is not None:
                assert_same(grouped(ctx, idx, q_off, q_mk, qcuts, mp, mode), w, "groups %s mode %d rescue %d" % (qcuts, mode, rescue))
        idx.free()
    monkeypatch.delenv("SK_REF_INDEX_PART_MARKERS", raising=False)
    if rset is None:
        rs.free()
    if qset is None:
        qs.free()
    return want


@pytest.mark.parametrize("sv", [0.0, 0.95])
def test_threshold_edges(ctx, monkeypatch, sv):
    cards, groups, meta = threshold_plan(sv)
    off, mk = plan(cards, groups)
    n = len(cards)
    roff, rmk = subset(off, mk, range(0, n, 2))                 # pair p: ref p, query p
    qoff, qmk = subset(off, mk, range(1, n, 2))
    nq = n // 2
    qr = check(ctx, monkeypatch, roff, rmk, qoff, qmk, sv, part_markers=(1000, 5000), qcuts=[0, 1, nq // 3, nq // 2 + 1, nq])
    s0, s2 = set(qr[(0, False)].tolist()), set(qr[(2, False)].tolist())
    reached = {"thr - 1": 0, "thr": 0, "thr + 1": 0}
    for p, (mn, t, count, _) in enumerate(meta):
        key = pid(p, p)
        assert (key in s0) == (count >= t) and (key in s2) == (count > t), (mn, count)
        reached["thr - 1"] += count == t - 1
        reached["thr"] += count == t
        reached["thr + 1"] += count == t + 1
    assert all(v > 0 for v in reached.values()), reached
    assert thr_of(sv, 1000) > 1


def test_rescue_small_genomes(ctx, monkeypatch):
    off, mk = rescue_plan()
    cards = np.diff(off.astype(np.int64))
    assert {19, 20, 21} <= set(cards.tolist())
    qr = check(ctx, monkeypatch, off, mk, off, mk, part_markers=(1, 40), qcuts=[0, 3, 4, 9, len(cards)])
    assert len(qr[(0, True)]) > len(qr[(0, False)]) and len(qr[(2, True)]) > len(qr[(2, False)])


@pytest.fixture(scope="module")
def tiles(ctx):
    off, mk, planned, fail_pairs, hub = tile_plan()
    t_off, t_mk = subset(off, mk, range(N_TILE))
    q_off, q_mk = subset(off, mk, range(N_TILE, N_TILE + 6))
    s_off, s_mk = subset(off, mk, range(N_TILE + 6, N_TILE + 6 + N_SMALL_Q))
    d = dict(t=(t_off, t_mk), q=(q_off, q_mk), small=(s_off, s_mk), tset=device_set(ctx, t_off, t_mk))
    yield d
    d["tset"].free()


def test_column_tiles(ctx, monkeypatch, tiles):
    t_off, t_mk = tiles["t"]
    q_off, q_mk = tiles["q"]
    assert N_TILE > 2 * TILE
    # parts cut inside the first tile, on no tile boundary, and about one tile each
    qr = check(ctx, monkeypatch, t_off, t_mk, q_off, q_mk, part_markers=(30 * 20_000 + 7, 30 * TILE), qcuts=[0, 2, 3, 6], rset=tiles["tset"])
    s = set(qr[(1, False)].tolist())
    for r in (0, 49_151, 49_152, 98_303, 98_304, N_TILE - 1):   # query 0 passes on both sides of every tile boundary
        assert pid(r, 0) in s, r
    assert len(qr[(2, True)][(qr[(2, True)] & MASK) == U64(2)]) == N_TILE      # the query without markers: rescued by mode 2


def test_pair_buffer_retry(ctx, monkeypatch, tiles):
    t_off, t_mk = tiles["t"]
    s_off, s_mk = tiles["small"]
    qr = check(ctx, monkeypatch, t_off, t_mk, s_off, s_mk, rescues=(True,), part_markers=(30 * 60_000,), qcuts=[0, 7, N_SMALL_Q],
               rset=tiles["tset"])
    for mode in (0, 2):
        assert len(qr[(mode, True)]) == N_TILE * N_SMALL_Q > max(CAP0, 64 * N_SMALL_Q)


def test_marker_range_extremes(ctx, monkeypatch):
    top = (1 << 42) - 1
    rng = np.random.default_rng(43)
    pool = np.concatenate([np.arange(2, 3000), np.arange(top - 3000, top - 1)])
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
    roff, rmk = subset(off, mk, range(0, 40, 2))
    qoff, qmk = subset(off, mk, range(1, 40, 2))
    assert int(rmk.min()) == 0 and int(rmk.max()) == top and int(qmk.max()) == top
    qr = check(ctx, monkeypatch, roff, rmk, qoff, qmk, part_markers=(200, 1000), qcuts=[0, 5, 20])
    assert pid(0, 0) in set(qr[(1, False)].tolist())            # ref 0 and query 0 share 2^42 - 1 and 2^42 - 2


def test_empty_sets(ctx, monkeypatch):
    cards = [0, 30, 25, 0, 30, 40, 0]
    groups = []
    share(groups, 1, 2, 2); share(groups, 2, 4, 3); share(groups, 4, 5, 1); share(groups, 1, 5, 2)
    off, mk = plan(cards, groups)
    check(ctx, monkeypatch, off, mk, off, mk, part_markers=(1, 30), qcuts=[0, 1, 4, 7])
    e_off, e_mk = plan([0] * 4, [])
    qr = check(ctx, monkeypatch, e_off, e_mk, off, mk, part_markers=(1,))             # references without markers
    assert len(qr[(0, True)]) == 4 * 7 and len(qr[(3, True)]) == 0
    qr = check(ctx, monkeypatch, off, mk, e_off, e_mk, part_markers=(1,))             # queries without markers
    assert len(qr[(2, True)]) == 7 * 4 and len(qr[(1, True)]) == 0
