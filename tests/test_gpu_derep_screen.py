"""dereplicate's marker index and row screen (derep.cu: index_add, dr_keys_kernel, dr_bucket_kernel, dr_rows_kernel, Run::screen)
through sk_debug_derep_screen, pair list by pair list against the triangle screen restricted to the call: without `upper`, the
triangle's pairs with one genome among the rows and the other among the slots; with `upper`, its pairs inside the slot list.
The small sets take the triangle from the CPU oracle, the sets of 100,000 genomes from test_gpu_screen's scipy incidence
product.  Every call also checks the index itself: keys == sorted(marker << 22 | slot), buckets == their prefix search.

Markers-only sets fabricated with test_gpu_screen's planner: shared counts thr - 1, thr, thr + 1 at screen_val 0.8, 0.95 and
0.99 with the row's genome index below and above the slot's; cards 0, 1, 19, 20, 21 with the rescue on and off; 100,000
slots in a shuffled order (three 49,152-slot tiles) with pairs on both sides of every tile boundary in both modes, a rescued
row and two markers held by 2,000 slots; one slot list indexed in several batchings (one batch, the default wave growth, a
markerless first batch, one-genome batches, a marker run extended by many merges); markers 0, 1, 2^42 - 1 and the first and
last marker of prefix buckets; more passing pairs than the first pair buffer; empty lists; the index limits and the entry's
own refusals.  Each test asserts that it reached the edge it is named for.  test_past_first_slot_tile runs sk_dereplicate
with more than 49,152 representatives against sk_cluster on the triangle's rows."""
import ctypes as C
import time

import numpy as np
import pytest

import oracle_py as O
import test_gpu_screen as S

pytestmark = pytest.mark.gpu

U64 = np.uint64
TILE = 48 * 1024                 # slots counted per shared-memory tile of dr_rows_kernel
CAP0 = 1 << 20                   # first pair-buffer capacity of Run::screen: max(2^20, 64 * rows)
PREFIX_SHIFT = 48                # a key's 16-bit bucket prefix: key >> (42 + 22 - 16)
MAX_SLOTS = (1 << 22) - 1
LO32 = U64(0xFFFFFFFF)


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def pid(a, b):
    return S.pid(min(a, b), max(a, b))


def wave_batches(n):
    """the default wave sizes of sk_dereplicate (64, 128, ... 4,096) over n slots"""
    out, size = [], 64
    while sum(out) < n:
        out.append(min(size, n - sum(out)))
        size = min(2 * size, 4096)
    return out


def index_keys(off, mk, slots):
    slots = np.asarray(slots, np.int64)
    cards = (off[slots + 1] - off[slots]).astype(np.int64)
    first = np.concatenate([[0], np.cumsum(cards)[:-1]]).astype(np.int64)
    at = np.repeat(off[slots].astype(np.int64) - first, cards) + np.arange(int(cards.sum()), dtype=np.int64)
    slot = np.repeat(np.arange(len(slots), dtype=U64), cards)
    return np.sort((mk[at] << U64(22)) | slot)


def restrict(tri, rows, slots, upper):
    """the triangle's pairs that the call screens"""
    a, b = tri >> U64(32), tri & LO32
    sl = np.asarray(slots, U64)
    if upper:
        return tri[np.isin(a, sl) & np.isin(b, sl)]
    rw = np.asarray(rows, U64)
    assert not np.isin(rw, sl).any(), "rows and slots must be disjoint without upper"
    return tri[(np.isin(a, rw) & np.isin(b, sl)) | (np.isin(b, rw) & np.isin(a, sl))]


def dscreen(ctx, s, off, mk, slots, rows, upper, mp, tri, batches=None, what=""):
    """sk_debug_derep_screen == the restricted triangle, its keys and buckets == the plain ones; returns (pairs, keys, bucket)"""
    import skani_b200 as sk
    pairs, keys, bucket = sk.host.debug_derep_screen(ctx, s, slots, rows, upper, batches, mp)
    want_keys = index_keys(off, mk, slots)
    assert np.array_equal(keys, want_keys), what + ": index keys"
    assert np.array_equal(bucket, np.searchsorted(keys >> U64(PREFIX_SHIFT), np.arange((1 << 16) + 1, dtype=U64), "left")), what + ": buckets"
    S.assert_same(pairs, restrict(tri, rows, slots, upper), "%s (upper %d, %d rows, %d slots)" % (what, upper, len(rows), len(slots)))
    return pairs, keys, bucket


def oracle_tri(off, mk, sv, rescue):
    return O.screen_triangle_pairs(S.oracle_set(off, mk), sv, rescue)


# ---------------------------------------------------------------------------------------------------------------------
# a. threshold edges
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sv", [0.0, 0.95, 0.99])
def test_threshold_edges(ctx, sv):
    import skani_b200 as sk
    cards, groups, meta = S.threshold_plan(sv)             # pair p = genomes (2p, 2p + 1) sharing `count` markers
    off, mk = S.plan(cards, groups)
    n = len(cards)
    tri = oracle_tri(off, mk, sv, True)
    s = S.device_set(ctx, off, mk)
    mp = sk.map_params(screen_val=sv)
    rng = np.random.default_rng(11)
    ev, od = np.arange(0, n, 2), np.arange(1, n, 2)
    # rows below their slots' genome indices, then above; slots shuffled, indexed in waves
    for rows, slots in ((ev, rng.permutation(od)), (od, rng.permutation(ev))):
        dscreen(ctx, s, off, mk, slots, rows, False, mp, tri, wave_batches(len(slots)), "thresholds sv %g" % sv)
    perm = rng.permutation(n)
    dscreen(ctx, s, off, mk, perm, perm, True, mp, tri, None, "thresholds sv %g" % sv)
    s.free()
    got, pos = S.as_set(tri), np.argsort(perm)
    on_thr = below = row_lo = row_hi = 0
    for p, (mn, t, count, small_first) in enumerate(meta):
        assert (S.pid(2 * p, 2 * p + 1) in got) == (count > t), (mn, count, small_first)
        on_thr += count == t
        below += count == t - 1 and count >= 1
        if count in (t, t + 1):                            # upper: is the row (earlier slot) the smaller genome index?
            row_lo += pos[2 * p] < pos[2 * p + 1]
            row_hi += pos[2 * p] > pos[2 * p + 1]
    assert on_thr >= 2 * len(S.MNS) and below > 0 and row_lo > 5 and row_hi > 5


# ---------------------------------------------------------------------------------------------------------------------
# b. rescue of genomes with < 20 markers
# ---------------------------------------------------------------------------------------------------------------------
def test_rescue_small_genomes(ctx):
    import skani_b200 as sk
    off, mk = S.rescue_plan()
    cards = np.array(S.RESCUE_CARDS)
    n = len(cards)
    assert {0, 1, 19, 20, 21} <= set(cards.tolist())
    s = S.device_set(ctx, off, mk)
    rng = np.random.default_rng(5)
    for rescue in (True, False):
        mp = sk.map_params(rescue_small=rescue)
        tri = oracle_tri(off, mk, 0.0, rescue)
        assert S.as_set(tri) == S.as_set(S.sparse_triangle(off, mk, 0.0, rescue))
        for g in range(n):                                 # every genome as the only row, every other one a slot
            others = rng.permutation(np.delete(np.arange(n), g))
            pairs, _, _ = dscreen(ctx, s, off, mk, others, [g], False, mp, tri, [3, 1, n - 5], "rescue %d, row %d" % (rescue, g))
            got = S.as_set(pairs)
            if g == 4:                                     # 1 marker: rescued as the smaller index only
                assert ({pid(4, 5), pid(4, 7), pid(4, 13)} <= got) == rescue   # 21 markers, none shared; 0 markers
                assert pid(0, 4) not in got and pid(3, 4) not in got          # the larger index: never rescued
            if g == 1:                                     # 0 markers: rescued against every later genome
                assert ({pid(1, j) for j in range(2, n)} <= got) == rescue and pid(0, 1) not in got
        perm = rng.permutation(n)
        got = S.as_set(dscreen(ctx, s, off, mk, perm, perm, True, mp, tri, [1, 6, n - 7], "rescue %d, upper" % rescue)[0])
        small = [g for g in range(n - 1) if cards[g] < S.SMALL]
        assert all(({pid(g, j) for j in range(g + 1, n)} <= got) == rescue for g in small)
        assert not {pid(0, 1), pid(0, 7), pid(0, 2), pid(3, 13), pid(5, 6)} & got
    s.free()


# ---------------------------------------------------------------------------------------------------------------------
# c. three slot tiles: 100,000 slots, slot != genome
# ---------------------------------------------------------------------------------------------------------------------
N_SLOTS = 100_000
R_SMALL, R_POS, R_HUB, R_POS2, R_EMPTY = 0, 40_000, 70_001, 100_003, 100_005   # row genomes (R_SMALL: 10 markers, rescued)
ROW_GENOMES = (R_SMALL, 2, R_POS, R_HUB, R_POS2, R_EMPTY, 100_006, 100_007)
N_GEN = N_SLOTS + len(ROW_GENOMES)
TILE_POS = (0, TILE - 1, TILE, 2 * TILE - 1, 2 * TILE, N_SLOTS - 1)             # first / last slot of every tile (from 0)
FAIL_POS = (1, TILE + 1, 2 * TILE + 1)                                          # one shared marker (= thr): fails
UPPER_K = (0, 5, 1000)                                                          # tiles from k + 1
UPPER_D = (TILE, TILE + 1, 1 + 2 * TILE)
RESCUED_SLOT = 3                                                                # holds genome 1 (10 markers)


def tile_plan():
    rng = np.random.default_rng(2024)
    slot_genome = rng.permutation(np.setdiff1d(np.arange(N_GEN), ROW_GENOMES))
    j = int(np.nonzero(slot_genome == 1)[0][0])
    slot_genome[[j, RESCUED_SLOT]] = slot_genome[[RESCUED_SLOT, j]]
    cards = np.full(N_GEN, 30, np.int64)
    cards[[R_SMALL, 1]] = 10
    cards[R_EMPTY] = 0
    groups = []
    for r in (R_POS, R_POS2):
        for p in TILE_POS:
            S.share(groups, r, slot_genome[p], 2)
        for p in FAIL_POS:
            S.share(groups, r, slot_genome[p], 1)
    for k in UPPER_K:
        for d in UPPER_D:
            S.share(groups, slot_genome[k], slot_genome[k + d], 2)
    busy = set(TILE_POS) | set(FAIL_POS) | {RESCUED_SLOT} | {k for k in UPPER_K} | {k + d for k in UPPER_K for d in UPPER_D}
    hub_pos = np.array([p for p in range(11, N_SLOTS, 50) if p not in busy])
    hub = [int(g) for g in slot_genome[hub_pos]] + [R_HUB]
    groups += [hub, hub]                                   # two markers: count 2 passes
    off, mk = S.plan(cards, groups)
    return off, mk, slot_genome, hub_pos


@pytest.fixture(scope="module")
def tiles(ctx):
    off, mk, slot_genome, hub_pos = tile_plan()
    tri = S.sparse_triangle(off, mk, 0.0, True)
    s = S.device_set(ctx, off, mk)
    yield dict(off=off, mk=mk, slots=slot_genome, hub_pos=hub_pos, tri=tri, s=s)
    s.free()


def test_slot_tiles(ctx, tiles):
    import skani_b200 as sk
    off, mk, sg, tri = tiles["off"], tiles["mk"], tiles["slots"], tiles["tri"]
    assert N_SLOTS > 2 * TILE and (sg != np.arange(N_SLOTS)).mean() > 0.99
    mp = sk.map_params()
    rows = np.array(ROW_GENOMES)
    pairs, keys, _ = dscreen(ctx, tiles["s"], off, mk, sg, rows, False, mp, tri, wave_batches(N_SLOTS), "tiles")
    got = S.as_set(pairs)
    for r in (R_POS, R_POS2):                              # tiles start at 0: both sides of every boundary
        assert all(pid(r, sg[p]) in got for p in TILE_POS), r
        assert not any(pid(r, sg[p]) in got for p in FAIL_POS), r
    rescued = pairs[(pairs >> U64(32)) == U64(R_SMALL)] & LO32
    assert np.array_equal(np.sort(rescued), np.sort(sg.astype(U64)))            # every slot of all three tiles
    hp = tiles["hub_pos"]
    assert len(hp) >= 1900 and hp.min() < TILE and ((hp >= TILE) & (hp < 2 * TILE)).any() and hp.max() >= 2 * TILE
    hub = {pid(R_HUB, g) for g in sg[hp]}
    assert hub <= got and len([p for p in got if R_HUB in (p >> 32, p & 0xFFFFFFFF)]) == len(hp) + 1   # + genome 1 (rescued)
    # upper: row k against slots k + 1 ..
    pu, _, _ = dscreen(ctx, tiles["s"], off, mk, sg, sg, True, mp, tri, None, "tiles, upper")
    gu = S.as_set(pu)
    for k in UPPER_K:                                      # last slot of tile 0, first of tile 1, first of tile 2
        assert all(pid(sg[k], sg[k + d]) in gu for d in UPPER_D), k
    assert {pid(1, g) for g in sg[RESCUED_SLOT + 1:]} <= gu                       # a rescued row over all three tiles
    assert len({pid(a, b) for a in sg[hp[:40]] for b in sg[hp[-40:]]} - gu) == 0


# ---------------------------------------------------------------------------------------------------------------------
# d. the index built in several batchings
# ---------------------------------------------------------------------------------------------------------------------
def test_index_batchings(ctx):
    import skani_b200 as sk
    rng = np.random.default_rng(9)
    n_slot, n_row, n_empty = 6000, 40, 10
    n = n_slot + n_row
    cards = rng.integers(22, 45, n)
    slots = rng.permutation(n_slot)                        # genomes [0, n_slot) are slots, the rest rows
    cards[slots[:n_empty]] = 0                             # a first batch without markers
    groups = []
    run_pos = np.arange(n_empty, n_slot, 97)               # one marker held by a slot of every batch
    groups.append([int(g) for g in slots[run_pos]])
    groups.append([int(g) for g in slots[run_pos[::3]]])   # ... and a second one for a third of them: count 2 passes
    for i in range(3000):                                  # random pairs of slots and of rows x slots around the threshold
        a = int(slots[rng.integers(n_empty, n_slot)]) if i % 2 else int(rng.integers(n_slot, n))
        b = int(slots[rng.integers(n_empty, n_slot)])
        if a != b:
            S.share(groups, a, b, int(rng.integers(5, 15)))
    cards = np.maximum(cards, np.bincount(np.concatenate([np.asarray(g) for g in groups]), minlength=n))
    cards[slots[:n_empty]] = 0
    off, mk = S.plan(cards, groups)
    tri = S.sparse_triangle(off, mk, 0.0, True)
    assert S.as_set(tri) == S.as_set(oracle_tri(off, mk, 0.0, True))
    s = S.device_set(ctx, off, mk)
    mp = sk.map_params()
    waves = wave_batches(n_slot)
    batchings = {"one": [n_slot], "waves": waves, "empty first": [n_empty, n_slot - n_empty],
                 "one-genome": [n_empty, 1, 1, 500, 1, n_slot - n_empty - 503], "hundreds": [n_empty] + [142] * 42 + [n_slot - n_empty - 142 * 42]}
    rows = np.arange(n_slot, n)
    out = {}
    for name, b in batchings.items():
        assert sum(b) == n_slot
        for upper in (False, True):
            out[(name, upper)] = dscreen(ctx, s, off, mk, slots, slots if upper else rows, upper, mp, tri, b, "batching " + name)
    for upper in (False, True):
        base = out[("one", upper)]
        for name in batchings:
            for x, y in zip(out[(name, upper)], base):
                assert x.tobytes() == y.tobytes(), (name, upper)
        assert len(base[0]) > 300
    # the markerless first batch leaves ix.n = 0, so the second batch copies instead of merging
    assert (off[slots[:n_empty] + 1] == off[slots[:n_empty]]).all()
    # the shared marker's run is extended by every wave after the first
    cum = np.cumsum([0] + waves)
    assert len(np.unique(np.searchsorted(cum, run_pos, "right"))) == len(waves) >= 6
    s.free()


# ---------------------------------------------------------------------------------------------------------------------
# e. markers at both ends of the 42-bit range and on prefix-bucket edges
# ---------------------------------------------------------------------------------------------------------------------
def test_marker_extremes(ctx):
    import skani_b200 as sk
    top = (1 << 42) - 1
    edge = [0, 1, top, top - 1]
    for b in (1, 2, 777, 32_768, 65_535):
        edge += [b * (1 << 26) - 1, b * (1 << 26)]         # the last marker of prefix bucket b - 1, the first of bucket b
    n = 3 * len(edge) + 6
    rng = np.random.default_rng(3)
    lists = [set((S.BG_BASE + 100 * g + np.arange(4)).tolist()) for g in range(n)]   # 4 own markers each
    plans = []
    owner = rng.permutation(n)
    for j, v in enumerate(edge):                           # v and one planned marker shared by 3 genomes of 6 markers: count
        grp = owner[3 * j:3 * j + 3]                       # 2 passes (thr 1), count 1 (v missed) fails
        for g in grp:
            lists[g] |= {v, S.SHARED_BASE + j}
        plans.append((v, grp))
    lists = [np.array(sorted(x), U64) for x in lists]
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(U64)
    mk = np.concatenate(lists)
    tri = oracle_tri(off, mk, 0.0, False)                  # every genome has 4 or 6 markers: no rescue
    assert S.as_set(tri) == S.as_set(S.sparse_triangle(off, mk, 0.0, False))
    s = S.device_set(ctx, off, mk)
    mp = sk.map_params(rescue_small=False)
    perm = rng.permutation(n)
    _, keys, bucket = dscreen(ctx, s, off, mk, perm, perm, True, mp, tri, [7, 20, n - 27], "extremes, upper")
    got = S.as_set(tri)
    for v, grp in plans:
        assert all(pid(a, b) in got for a in grp for b in grp if a < b), v
    assert len(got) == 3 * len(edge)
    half = rng.permutation(n)
    for slots, rows in ((half[:30], half[30:]), (half[30:], half[:30])):
        assert len(restrict(tri, rows, slots, False)) > 5
        dscreen(ctx, s, off, mk, slots, rows, False, mp, tri, [1, len(slots) - 1], "extremes")
    km = keys >> U64(22)
    assert int(km[0]) == 0 and int(km[-1]) == top and bucket[1] > 0 and bucket[65_535] < len(keys)
    for b in (1, 2, 777, 32_768, 65_535):                  # the bucket's first key is marker b * 2^26, the previous one's last b * 2^26 - 1
        assert int(km[bucket[b]]) == b << 26 and int(km[bucket[b] - 1]) == (b << 26) - 1, b
    s.free()


# ---------------------------------------------------------------------------------------------------------------------
# f. more passing pairs than the first pair buffer holds
# ---------------------------------------------------------------------------------------------------------------------
def test_pair_buffer_retry(ctx):
    import skani_b200 as sk
    mp = sk.map_params()
    rng = np.random.default_rng(8)
    # upper: 1,500 rescued genomes -> every pair
    n = 1500
    groups = []
    for g in range(0, n - 1, 7):
        S.share(groups, g, g + 1, 2)
    off, mk = S.plan(np.full(n, 5), groups)
    s = S.device_set(ctx, off, mk)
    every = S.all_pairs_triangle(n)
    S.assert_same(S.sparse_triangle(off, mk, 0.0, True), every, "incidence product")
    perm = rng.permutation(n)
    pairs = dscreen(ctx, s, off, mk, perm, perm, True, mp, every, None, "retry, upper")[0]
    assert len(pairs) == 1_124_250 > max(CAP0, 64 * n)
    s.free()
    # rows x slots: 50 rescued rows (the smaller indices) x 25,000 slots
    nr, ns = 50, 25_000
    cards = np.full(nr + ns, 30)
    cards[:nr] = 5
    groups = []
    for g in range(nr, nr + ns - 1, 11):
        S.share(groups, g, g + 1, 3)
    off, mk = S.plan(cards, groups)
    tri = S.sparse_triangle(off, mk, 0.0, True)
    s = S.device_set(ctx, off, mk)
    slots = rng.permutation(np.arange(nr, nr + ns))
    pairs = dscreen(ctx, s, off, mk, slots, np.arange(nr), False, mp, tri, wave_batches(ns), "retry")[0]
    assert len(pairs) == nr * ns > max(CAP0, 64 * nr)
    s.free()


# ---------------------------------------------------------------------------------------------------------------------
# g. degenerate inputs
# ---------------------------------------------------------------------------------------------------------------------
def test_degenerate(ctx):
    import skani_b200 as sk
    mp = sk.map_params()
    cards = [0, 30, 25, 0, 30, 40, 0, 5, 0]
    groups = []
    S.share(groups, 1, 2, 2); S.share(groups, 2, 4, 3); S.share(groups, 4, 5, 1); S.share(groups, 1, 5, 2)
    off, mk = S.plan(cards, groups)
    tri = oracle_tri(off, mk, 0.0, True)
    s = S.device_set(ctx, off, mk)
    # no rows; no slots
    p, k, b = dscreen(ctx, s, off, mk, [5, 1, 2], [], False, mp, tri, None, "no rows")
    assert len(p) == 0 and len(k) == 95
    p, k, b = dscreen(ctx, s, off, mk, [], [1, 4], False, mp, tri, [], "no slots")
    assert len(p) == len(k) == 0 and not b.any()
    p, k, b = dscreen(ctx, s, off, mk, [], [], True, mp, tri, [], "no slots, upper")
    assert len(p) == len(k) == 0
    # every slot markerless: the buckets stay zero, and only the rescue passes pairs
    for rows in ([1, 2, 4, 5], [7], [1, 7]):
        for batches in (None, [1, 1, 1, 1]):
            p, k, b = dscreen(ctx, s, off, mk, [6, 0, 8, 3], rows, False, mp, tri, batches, "markerless slots")
            assert len(k) == 0 and not b.any()
    assert len(p) > 0
    p, k, b = dscreen(ctx, s, off, mk, [6, 0, 8, 3], [6, 0, 8, 3], True, mp, tri, [2, 2], "markerless slots, upper")
    assert not b.any() and len(p) == 6                     # 0 markers each: every pair rescued
    # rows without markers
    p = dscreen(ctx, s, off, mk, [5, 2, 4, 1, 7], [0, 3, 6, 8], False, mp, tri, [2, 3], "markerless rows")[0]
    assert len(p) > 0
    # a single slot
    for g in range(len(cards)):
        others = [x for x in range(len(cards)) if x != g]
        dscreen(ctx, s, off, mk, [g], others, False, mp, tri, None, "single slot %d" % g)
        p = dscreen(ctx, s, off, mk, [g], [g], True, mp, tri, None, "single slot %d, upper" % g)[0]
        assert len(p) == 0
    s.free()


# ---------------------------------------------------------------------------------------------------------------------
# h. refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_refusals(ctx):
    import skani_b200 as sk
    mp = sk.map_params()
    off, mk = S.plan([1000, 30, 30, 10, 0], [[1, 2], [1, 2]])
    tri = oracle_tri(off, mk, 0.0, True)
    s = S.device_set(ctx, off, mk)
    Err = sk.host.SkaniError

    def still_screens():
        dscreen(ctx, s, off, mk, [2, 0, 3], [1], False, mp, tri, [1, 2], "after a refusal")
        dscreen(ctx, s, off, mk, [3, 1, 2, 0], [3, 1, 2, 0], True, mp, tri, None, "after a refusal, upper")

    # more than 2^22 - 1 slots: one genome repeated
    big = np.ones(MAX_SLOTS + 1, np.uint32)
    with pytest.raises(Err, match=r"more than 2\^22 - 1 genomes \(4194304\) in one marker index"):
        sk.host.debug_derep_screen(ctx, s, big, [2], False, None, mp)
    big[:] = 4                                             # markerless: the first batch adds no key, the second is refused
    with pytest.raises(Err, match=r"more than 2\^22 - 1 genomes \(4194304\)"):
        sk.host.debug_derep_screen(ctx, s, big, [2], False, [MAX_SLOTS, 1], mp)
    still_screens()
    # 2^31 keys or more: the 1,000-marker genome repeated (checked from mk_off before any key is built)
    rep = 2_200_000
    assert rep * 1000 >= 1 << 31 and rep < MAX_SLOTS
    many = np.zeros(rep, np.uint32)
    with pytest.raises(Err, match=r"2200000000 markers in one marker index \(at most 2\^31 - 1\)"):
        sk.host.debug_derep_screen(ctx, s, many, [1], False, None, mp)
    with pytest.raises(Err, match=r"2200000000 markers in one marker index"):
        sk.host.debug_derep_screen(ctx, s, many, [1], False, [1000, rep - 1000], mp)       # 10^6 keys, then the rest
    still_screens()
    # the entry's own refusals
    with pytest.raises(Err, match="holds genome 5 >= 5"):
        sk.host.debug_derep_screen(ctx, s, [0, 5], [1], False, None, mp)
    with pytest.raises(Err, match="is genome 7 >= 5"):
        sk.host.debug_derep_screen(ctx, s, [0, 2], [1, 7], False, None, mp)
    with pytest.raises(Err, match="batch sizes sum to 1, not n_slots = 2"):
        sk.host.debug_derep_screen(ctx, s, [0, 2], [1], False, [1], mp)
    with pytest.raises(Err, match="batch sizes sum to 3"):
        sk.host.debug_derep_screen(ctx, s, [0, 2], [1], False, [1, 2], mp)
    for rows in ([2, 0], [0], [0, 2, 1]):
        with pytest.raises(Err, match="upper needs rows equal to slot_genome"):
            sk.host.debug_derep_screen(ctx, s, [0, 2], rows, True, None, mp)
    sg, rw, bs = np.array([0, 2], np.uint32), np.array([1], np.uint32), np.array([2], np.uint32)
    pp, kp, n, nk = C.POINTER(C.c_uint64)(), C.POINTER(C.c_uint64)(), C.c_uint64(), C.c_uint64()
    bucket = np.zeros((1 << 16) + 1, np.uint32)
    args = [ctx.h, s.h, C.byref(mp), sg.ctypes.data, 2, bs.ctypes.data, 1, rw.ctypes.data, 1, 0, C.byref(pp), C.byref(n),
            C.byref(kp), C.byref(nk), bucket.ctypes.data]
    for i in (1, 2, 3, 5, 7, 10, 11, 12, 13):
        bad = list(args)
        bad[i] = None
        assert ctx.L.sk_debug_derep_screen(*bad) == -2, i
        assert "NULL" in ctx.L.sk_last_error(ctx.h).decode(), i
    assert ctx.L.sk_debug_derep_screen(None, *args[1:]) == -2
    assert ctx.L.sk_debug_derep_screen(*args[:12], None, None, None) == 0          # keys and buckets are optional
    assert n.value == 1 and pp[0] == S.pid(1, 2)
    ctx.L.sk_free(pp)
    still_screens()
    s.free()


# ---------------------------------------------------------------------------------------------------------------------
# sk_dereplicate with more than one slot tile of representatives
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.slow
def test_past_first_slot_tile(ctx):
    """60,000 two-genome families of 8 kbp: the first genome of every family ranks first (shuffled), so 60,000
    representatives fill the index before any member is screened, in the waves and in the final screen"""
    import skani_b200 as sk
    from bench_support import synth
    fam, L = 60_000, 8_000
    n = 2 * fam
    t0 = time.time()
    bases, off, goc = synth.generate(0, n, L, G=2)
    s = sk.sketch_contigs(ctx, bases, off, goc, n, sk.sketch_params(c=100, marker_c=100))
    del bases
    cards = np.array([s.info(g)["n_markers"] for g in range(n)])
    assert cards.min() >= 20, cards.min()                  # no genome is rescued
    firsts, members = np.arange(0, n, 2), np.arange(1, n, 2)   # family f: genomes 2f, 2f + 1
    rng = np.random.default_rng(17)
    order = np.concatenate([rng.permutation(firsts), rng.permutation(members)])
    rank = np.empty(n, np.uint32)
    rank[order] = np.arange(n)
    mp = sk.map_params()
    min_ani = 0.9
    t1 = time.time()
    pairs = sk.screen_triangle(ctx, s, mp)
    tri = sk.chain_pairs(ctx, s, s, pairs, mp, as_array=True)
    erep, ecl, eedge, _ = sk.cluster(ctx, n, tri, rank, min_ani=min_ani)
    t2 = time.time()
    rep, cl, join, st = sk.dereplicate(ctx, s, rank, min_ani=min_ani, mp=mp)
    t3 = time.time()
    print("dereplicate of %d genomes in %d families: %.1f s (triangle + cluster %.1f s, sketch %.1f s); %d clusters, %d pairs "
          "screened, %d chained, %d waves" % (n, fam, t3 - t2, t2 - t1, t1 - t0, st.n_clusters, st.pairs_screened, st.pairs_chained, st.waves))
    assert np.array_equal(rep, erep) and np.array_equal(cl, ecl), np.nonzero((rep != erep) | (cl != ecl))[0][:5]
    g = np.arange(n)
    mem = erep != g
    assert join[mem].tobytes() == tri[eedge[mem].astype(np.int64)].tobytes()
    # every family's first genome is a representative; a representative's slot is its place among them in rank order
    assert (erep[firsts] == firsts).all() and st.n_clusters >= fam
    rep_ranks = np.sort(rank[erep[~mem]])
    slot = np.searchsorted(rep_ranks, rank[erep[mem]])
    assert np.array_equal(slot[erep[mem] % 2 == 0], rank[erep[mem]][erep[mem] % 2 == 0])
    print("%d members, %d of them with a representative in slot >= %d" % (mem.sum(), (slot >= TILE).sum(), TILE))
    assert mem.sum() > fam // 4 and (slot >= TILE).sum() > 1000 and (slot < TILE).sum() > 1000
    s.free()
