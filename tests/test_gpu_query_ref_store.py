"""dist over host sketch stores (sk_query_ref_store), every context on GPU 0 unless a case says otherwise.

query_ref_store must equal, byte for byte after sorting, the in-memory screen_query_ref + chain_pairs (kept ani > 0.1) on sets
holding the same genomes with the same name ranks: modes 0-3 with rescue on and off; one working set, many working sets and
components cut into chunk pairs (asserted through sk_store_stats); one and two contexts; contiguous and shuffled genome
order; stores filled in several adds; --qi style shared ranks; one store as both sides; a genome of >= 2^20 records, one with
fewer than 20 markers and one without contigs on both sides; and no passing pair.  Small n is checked against the oracle;
bad arguments fail cleanly and leave the context usable."""
import numpy as np
import pytest

import oracle_py as O
from bench_support import synth
from chain_testlib import rand_seq

pytestmark = pytest.mark.gpu
TOL = 1e-4
L = 200_000


def key_sort(r):
    return r[np.lexsort((r["query_id"], r["ref_id"]))]


def layout(gs):
    contigs = [c for g in gs for c in g]
    off = np.concatenate([[0], np.cumsum([len(c) for c in contigs])]).astype(np.uint64)
    goc = np.concatenate([np.full(len(g), i, np.uint32) for i, g in enumerate(gs)]) if contigs else np.zeros(0, np.uint32)
    return (np.concatenate(contigs) if contigs else np.zeros(1, np.uint8)), off, goc


def split_genomes(bases, off, goc, n):
    return [[bases[int(off[i]):int(off[i + 1])] for i in np.nonzero(goc == g)[0]] for g in range(n)]


@pytest.fixture(scope="module")
def ctxs():
    import skani_b200 as sk
    cs = [sk.Context(0), sk.Context(0)]
    yield cs
    for c in cs:
        c.close()


def sketch(sk, ctx, gs, sp=None):
    bases, off, goc = layout(gs)
    return sk.sketch_contigs(ctx, bases, off, goc, len(gs), sp)


def store_of(sk, ctx, gs, ranks, groups=3, sp=None):
    """gs sketched in `groups` consecutive groups, each added to the store and freed; then the ranks."""
    st = sk.SketchStore(sp or sk.sketch_params())
    bounds = np.linspace(0, len(gs), groups + 1).astype(int)
    for a, b in zip(bounds[:-1], bounds[1:]):
        if b > a:
            s = sketch(sk, ctx, gs[a:b], sp)
            st.add(s)
            s.free()
    st.set_name_ranks(ranks)
    return st


def in_memory(sk, ctx, R, Q, mp, mode):
    pairs = sk.screen_query_ref(ctx, R, Q, mp, mode=mode)
    res = sk.chain_pairs(ctx, R, Q, pairs, mp, as_array=True)
    return key_sort(res[res["ani"] > np.float32(0.1)])


def ranks_in_one_order(nr, nq, shared=False):
    """refs and queries ranked in one file-name order; shared: --qi style, queries in files of three that share a rank, some
    of them equal to a reference's."""
    rr = 2 * np.arange(nr, dtype=np.uint64)
    qr = (2 * (np.arange(nq) // 3) + 1).astype(np.uint64) if shared else (2 * np.arange(nq) + 1).astype(np.uint64)
    if shared:
        qr[::5] = rr[np.arange(0, nq, 5) % nr]
    return rr, qr


def run_case(sk, ctxs, rg, qg, budget_of, n_ctx=1, mode=2, rescue=True, shared=False, sp=None):
    """budget_of(rbytes, qbytes) -> device_budget; returns (results, stats) after checking them against in-memory."""
    ctx = ctxs[0]
    mp = sk.map_params(rescue_small=rescue)
    rr, qr = ranks_in_one_order(len(rg), len(qg), shared)
    R, Q = sketch(sk, ctx, rg, sp), sketch(sk, ctx, qg, sp)
    R.set_name_ranks(rr); Q.set_name_ranks(qr)
    want = in_memory(sk, ctx, R, Q, mp, mode)
    R.free(); Q.free()
    rs, qs = store_of(sk, ctx, rg, rr, sp=sp), store_of(sk, ctx, qg, qr, groups=2, sp=sp)
    budget = budget_of(np.array([rs.genome_bytes(g) for g in range(len(rg))]), np.array([qs.genome_bytes(g) for g in range(len(qg))]))
    got, stats = sk.query_ref_store(ctxs[:n_ctx], rs, qs, mp, mode=mode, device_budget=budget)
    assert got.tobytes() == want.tobytes()
    assert budget == 0 or stats.max_working_set_bytes <= budget
    rs.free(); qs.free()
    return got, stats


# ---- clustered references and queries held back from the same clusters ---------------------------------------------------
N, G = 48, 8          # 6 clusters of 8; genome 8c + 3 and 8c + 6 of each cluster are queries


def clustered(ids="contiguous"):
    if ids == "contiguous":
        gen = split_genomes(*synth.generate(0, N, L, G=G), N)
    else:
        order = synth.shuffled_ids(N, 11)
        gen = split_genomes(*synth.generate_ids(order, L, G=G), N)
    qmask = np.array([g % G in (3, 6) for g in range(N)])
    return [gen[g] for g in range(N) if not qmask[g]], [gen[g] for g in range(N) if qmask[g]]


def cluster_bytes(rb, qb):
    # 6 refs and 2 queries per cluster in the contiguous order
    return max(rb[6 * c:6 * c + 6].sum() + qb[2 * c:2 * c + 2].sum() for c in range(N // G))


BUDGETS = {   # device_budget from the genome sizes, and the plan shape it must produce
    "single_set": (lambda rb, qb: 0, "single"),
    "many_sets": (lambda rb, qb: int(max(1.05 * cluster_bytes(rb, qb), 2 * max(rb.max(), qb.max()) + 1)), "many"),
    "chunk_pairs": (lambda rb, qb: int(max(0.45 * cluster_bytes(rb, qb), 2 * max(rb.max(), qb.max()) + 1)), "chunks"),
}


def check_shape(stats, expect):
    assert stats.gathered_bytes > 0
    if expect == "single":
        assert stats.n_working_sets == 1 and stats.n_split_components == 0
    elif expect == "many":
        assert stats.n_working_sets >= N // G // 2 and stats.n_split_components == 0
    else:
        assert stats.n_split_components > 0 and stats.n_working_sets > N // G


@pytest.mark.parametrize("n_ctx", [1, 2])
@pytest.mark.parametrize("ids", ["contiguous", "shuffled"])
@pytest.mark.parametrize("case", sorted(BUDGETS))
def test_store_equals_in_memory(ctxs, case, ids, n_ctx):
    import skani_b200 as sk
    rg, qg = clustered(ids)
    budget_of, expect = BUDGETS[case]
    if ids == "shuffled" and expect != "single":      # clusters are scattered: size the budget by the whole set instead
        budget_of = (lambda rb, qb: int(max(0.3 * (rb.sum() + qb.sum()), 2 * max(rb.max(), qb.max()) + 1))) if expect == "many" else \
            (lambda rb, qb: int(2.2 * max(rb.max(), qb.max())))
    got, stats = run_case(sk, ctxs, rg, qg, budget_of, n_ctx=n_ctx)
    assert len(got) >= len(qg) * 3
    if ids == "contiguous":
        check_shape(stats, expect)
    else:
        assert (stats.n_working_sets == 1) == (expect == "single")


@pytest.mark.parametrize("rescue", [True, False], ids=["rescue", "no_rescue"])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_modes(ctxs, mode, rescue):
    """Small pieces (< 20 markers) on both sides make the rescue matter."""
    import skani_b200 as sk
    rg, qg = clustered()
    rg = rg + [[rg[0][0][:3_000]], [rg[7][0][:6_000]]]
    qg = qg + [[rg[0][0][:4_000]], [qg[3][0][:5_000]]]
    got, stats = run_case(sk, ctxs, rg, qg, BUDGETS["many_sets"][0], n_ctx=2, mode=mode, rescue=rescue)
    assert len(got) >= len(qg) * 2 and stats.n_working_sets > 1


def test_shared_ranks_and_identical_genomes(ctxs):
    """--qi style ranks: identical genomes on both sides tie on everything but the rank (switch_qr's file-name tie-break)."""
    import skani_b200 as sk
    rg, qg = clustered()
    qg = qg + [rg[0], rg[5], rg[0], rg[20]]
    got, stats = run_case(sk, ctxs, rg, qg, BUDGETS["chunk_pairs"][0], n_ctx=2, shared=True)
    assert stats.n_split_components > 0 and len(got) > len(qg)


def test_dense_cluster_chunk_pairs(ctxs):
    """One cluster, few queries against many references: chunk pairs, each reference gathered about once."""
    import skani_b200 as sk
    n = 20
    gen = split_genomes(*synth.generate(0, n, L, G=n), n)
    rg, qg = gen[:18], gen[18:]
    got, stats = run_case(sk, ctxs, rg, qg, lambda rb, qb: int(4.5 * max(rb.max(), qb.max())), n_ctx=2)
    assert len(got) >= len(rg)
    assert stats.n_split_components == 1 and stats.n_working_sets >= 4


def test_same_store_both_sides(ctxs):
    import skani_b200 as sk
    ctx = ctxs[0]
    rg, qg = clustered()
    gs = rg[:18] + qg[:6]
    ranks = np.arange(len(gs), dtype=np.uint64)
    S = sketch(sk, ctx, gs)
    S.set_name_ranks(ranks)
    mp = sk.map_params()
    want = in_memory(sk, ctx, S, S, mp, 2)
    S.free()
    st = store_of(sk, ctx, gs, ranks)
    gb = max(st.genome_bytes(g) for g in range(len(gs)))
    for budget in (0, int(2.5 * gb)):
        got, stats = sk.query_ref_store(ctxs, st, st, mp, mode=2, device_budget=budget)
        assert got.tobytes() == want.tobytes() and len(got) > len(gs)
        assert (stats.n_working_sets == 1) == (budget == 0)
    st.free()


def test_edge_genomes_both_sides(ctxs):
    """c = 10: a 12 Mbp genome (>= 2^20 records, no k-mer table), a 2 kb piece (< 20 markers) and a genome without contigs,
    on the reference and on the query side."""
    import skani_b200 as sk
    sp = sk.sketch_params(c=10, k=15, marker_c=200)
    gen = split_genomes(*synth.generate(0, 12, L, G=3), 12)
    big = [rand_seq(np.random.default_rng(5), 12_000_000)]
    rg = gen[:8] + [big, [gen[0][0][:2_000]], []]
    qg = gen[8:] + [[big[0][:6_000_000]], [gen[9][0][:2_000]], []]
    ctx = ctxs[0]
    probe = sketch(sk, ctx, rg, sp)
    assert probe.info(8)["n_records"] >= 1 << 20 and probe.info(9)["n_markers"] < 20 and probe.info(10)["n_contigs"] == 0
    probe.free()
    for budget_of in (lambda rb, qb: 0, lambda rb, qb: int(2.2 * max(rb.max(), qb.max()))):
        got, stats = run_case(sk, ctxs, rg, qg, budget_of, n_ctx=2, mode=0, sp=sp)
        assert len(got) >= 3                                                   # queries 8 against refs 6, 7 of its cluster
        assert ((got["ref_id"] == 8) & (got["query_id"] == 4)).any()      # the big genome against its half


def test_no_passing_pair(ctxs):
    import skani_b200 as sk
    rng = np.random.default_rng(9)
    rg = [[rand_seq(rng, L)] for _ in range(4)]
    qg = [[rand_seq(rng, L)] for _ in range(3)]
    got, stats = run_case(sk, ctxs, rg, qg, lambda rb, qb: 0, n_ctx=2, mode=0)
    assert len(got) == 0 and stats.n_working_sets == 0 and stats.gathered_bytes == 0


def test_oracle_small_n(ctxs):
    import skani_b200 as sk
    n = 14
    bases, off, goc = synth.generate_ids(synth.shuffled_ids(n, 3), L, G=4)
    gen = split_genomes(bases, off, goc, n)
    rsel, qsel = [g for g in range(n) if g % 3], [g for g in range(n) if g % 3 == 0]
    rg, qg = [gen[g] for g in rsel], [gen[g] for g in qsel]
    ctx = ctxs[0]
    rr, qr = ranks_in_one_order(len(rg), len(qg))
    rs, qs = store_of(sk, ctx, rg, rr, groups=2), store_of(sk, ctx, qg, qr, groups=2)
    gb = max(max(rs.genome_bytes(g) for g in range(len(rg))), max(qs.genome_bytes(g) for g in range(len(qg))))
    got, stats = sk.query_ref_store(ctxs, rs, qs, mode=0, device_budget=int(2.2 * gb))
    assert stats.n_working_sets > 1
    osk = O.sketch_many(bases, off, goc, n)
    ores = O.dist([osk[g] for g in rsel], [osk[g] for g in qsel], O.cmd())
    exp = {(r.ref_id, r.query_id): r for r in ores}
    assert sorted(exp) == [(int(r["ref_id"]), int(r["query_id"])) for r in got] and len(exp) >= len(qg)
    for r in got:
        o = exp[(int(r["ref_id"]), int(r["query_id"]))]
        for f in ("ani", "af_query", "af_ref"):
            assert abs(float(r[f]) - getattr(o, f)) <= TOL, (r, f)
    rs.free(); qs.free()


# ---- errors -------------------------------------------------------------------------------------------------------------
def test_errors_fail_cleanly(ctxs):
    import ctypes as C
    import skani_b200 as sk
    ctx = ctxs[0]
    rg, qg = clustered()
    rg, qg = rg[:12], qg[:4]
    rr, qr = ranks_in_one_order(len(rg), len(qg))
    rs, qs = store_of(sk, ctx, rg, rr), store_of(sk, ctx, qg, qr, groups=1)
    other = store_of(sk, ctx, qg, qr, groups=1, sp=sk.sketch_params(c=200))
    gb = max(rs.genome_bytes(g) for g in range(len(rg)))
    with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*parameters differ"):
        sk.query_ref_store(ctxs, rs, other)
    for mode in (-1, 4):
        with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*mode"):
            sk.query_ref_store(ctxs, rs, qs, mode=mode)
    with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*NULL argument"):
        sk.query_ref_store(ctxs, None, qs)
    with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*NULL argument"):
        sk.query_ref_store(ctxs, rs, None)
    with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*NULL context"):
        sk.query_ref_store([ctx, None], rs, qs)
    out = C.POINTER(sk.host.AniResult)(); n = C.c_uint64()
    hs = (C.c_void_p * 1)(ctx.h)
    assert ctx.L.sk_query_ref_store(hs, 1, rs.h, qs.h, None, 0, 0, C.byref(out), C.byref(n), None) == -2      # NULL map params
    assert "NULL argument" in ctx.L.sk_last_error(ctx.h).decode()
    with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*appears twice"):
        sk.query_ref_store([ctx, ctxs[1], ctx], rs, qs)
    with pytest.raises(sk.host.SkaniError, match=r"rc=-3.*reference \d+ needs .* more than half"):
        sk.query_ref_store(ctxs, rs, qs, device_budget=gb)
    qbig = store_of(sk, ctx, [rg[0] + rg[1] + rg[2]], [1], groups=1)
    with pytest.raises(sk.host.SkaniError, match=r"rc=-3.*query 0 needs .* more than half"):
        sk.query_ref_store(ctxs, rs, qbig, device_budget=int(2.2 * gb))
    # the contexts and the stores still work
    R, Q = sketch(sk, ctx, rg), sketch(sk, ctx, qg)
    R.set_name_ranks(rr); Q.set_name_ranks(qr)
    want = in_memory(sk, ctx, R, Q, sk.map_params(), 0)
    got, stats = sk.query_ref_store(ctxs, rs, qs, mode=0)
    assert got.tobytes() == want.tobytes() and len(got) > 0 and stats.n_working_sets == 1
    for s in (rs, qs, other, qbig):
        s.free()


def test_two_devices():
    import skani_b200 as sk
    L_ = sk.host._lib.load()
    if L_.sk_device_count() < 2:
        pytest.skip("needs two GPUs")
    cs = [sk.Context(0), sk.Context(0), sk.Context(1), sk.Context(1)]
    try:
        rg, qg = clustered()
        got, stats = run_case(sk, cs, rg, qg, BUDGETS["many_sets"][0], n_ctx=4)
        assert stats.n_working_sets > 1 and len(got) > len(qg)
    finally:
        for c in cs:
            c.close()
