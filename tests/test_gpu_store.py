"""Host sketch store and the triangle over it (sk_sketch_store_*, sk_triangle_store), every context on GPU 0.

Round trip: sets added to a store and gathered back in scattered subsets export bit-exact, chain byte-identical and screen
identically (markers only) to the sources, including a genome of >= 2^20 records (no k-mer table: bucket index rebuilt), a
genome without contigs, a genome with fewer than 20 markers and -i style name ranks.  Triangle: sk_triangle_store equals
sk_triangle byte for byte (sorted) for contiguous and shuffled ids, one and two contexts, one working set, many working sets
and components cut into chunk pairs, and matches the oracle within 1e-4 at small n.  Every triangle test asserts through
sk_store_stats that it reached the case it is named for."""
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
    goc = np.concatenate([np.full(len(g), i, np.uint32) for i, g in enumerate(gs)])
    return np.concatenate(contigs), off, goc


def split_genomes(bases, off, goc, n):
    return [[bases[int(off[i]):int(off[i + 1])] for i in np.nonzero(goc == g)[0]] for g in range(n)]


@pytest.fixture(scope="module")
def ctxs():
    import skani_b200 as sk
    cs = [sk.Context(0), sk.Context(0)]
    yield cs
    for c in cs:
        c.close()


# ---- round trip ---------------------------------------------------------------------------------------------------------
KW = dict(c=10, k=15, marker_c=200)


@pytest.fixture(scope="module")
def two_sets(ctxs):
    """Set A: 6 clustered genomes, a 12 Mbp random genome (>= 2^20 records at c = 10), a 2 kb piece (< 20 markers) and a
    genome without contigs (last); -i style ranks.  Set B: 6 more clustered genomes, default ranks."""
    import skani_b200 as sk
    ctx = ctxs[0]
    sp = sk.sketch_params(**KW)
    gen = split_genomes(*synth.generate(0, 12, L, G=3), 12)
    big = [rand_seq(np.random.default_rng(5), 12_000_000)]
    a_gen = gen[:6] + [big, [gen[0][0][:2_000]]]
    bases, off, goc = layout(a_gen)
    A = sk.sketch_contigs(ctx, bases, off, goc, len(a_gen) + 1, sp)
    A.set_name_ranks([0, 0, 1, 1, 2, 3, 4, 5, 5])
    B = sk.sketch_contigs(ctx, *layout(gen[6:]), 6, sp)
    assert A.info(6)["n_records"] >= 1 << 20 and A.info(7)["n_markers"] < 20 and A.info(8)["n_contigs"] == 0
    both = A.copy_to(ctx)
    both.append(B)          # one set holding A then B, ranks continued as the store continues them
    return sk, sp, A, B, both


@pytest.mark.parametrize("slab_mb", [1, 0], ids=["1MiB_slabs", "default_slabs"])
def test_round_trip(ctxs, two_sets, monkeypatch, slab_mb):
    sk, sp, A, B, both = two_sets
    ctx = ctxs[slab_mb == 1]          # gather on another context of the device too
    if slab_mb:
        monkeypatch.setenv("SK_STORE_SLAB_MB", str(slab_mb))
    st = sk.SketchStore(sp)
    st.add(A)
    st.add(B)
    nA = len(A)
    assert st.n_genomes() == nA + len(B) == len(both)
    assert st.genome_bytes(6) > 20 * (1 << 20) > st.genome_bytes(0) > st.genome_bytes(7) > st.genome_bytes(8) > 0
    for sub in ([1, 3, 6, 7, 8, nA + 0, nA + 4], list(range(len(both))), [8, nA + 5], [6]):
        g = st.gather(ctx, sub)
        assert len(g) == len(sub)
        for i, s in enumerate(sub):
            e, w = g.export(i), both.export(s)
            for k in w:
                assert np.array_equal(e[k], w[k]), (sub, s, k)
            assert g.info(i) == both.info(s)
        pairs = np.array([(x << 32) | y for x in range(len(sub)) for y in range(len(sub)) if x != y], np.uint64)
        gp = np.array([(sub[x] << 32) | sub[y] for x in range(len(sub)) for y in range(len(sub)) if x != y], np.uint64)
        got = sk.chain_pairs(ctx, g, g, pairs, as_array=True)
        want = sk.chain_pairs(ctxs[0], both, both, gp, as_array=True)
        want["ref_id"] = (pairs >> np.uint64(32)).astype(np.uint32)          # ids are indices into the set chained
        want["query_id"] = (pairs & np.uint64(0xFFFFFFFF)).astype(np.uint32)
        assert got.tobytes() == want.tobytes(), sub
        if len(sub) == len(both):
            assert np.isfinite(got["ani"]).sum() > 20
        g.free()
    # the ranks decide switch_qr between the identical-rank genomes 0/1 exactly as in the source
    g = st.gather(ctx, [0, 1, 2])
    assert [d["switched"] for d in sk.chain_pairs_debug(ctx, g, g, [1, 1 << 32])] == \
        [d["switched"] for d in sk.chain_pairs_debug(ctxs[0], both, both, [1, 1 << 32])]
    # markers only: screens like the source, chains to "no anchors"
    mk = st.gather(ctx, None, markers_only=True)
    assert sk.screen_triangle(ctx, mk).tobytes() == sk.screen_triangle(ctxs[0], both).tobytes()
    assert len(sk.screen_triangle(ctx, mk)) > 10
    for mode in range(4):
        assert sk.screen_query_ref(ctx, mk, mk, mode=mode).tobytes() == sk.screen_query_ref(ctxs[0], both, both, mode=mode).tobytes()
    assert np.isnan(sk.chain_pairs(ctx, mk, mk, [1], as_array=True)["ani"]).all()
    st.free()


# ---- triangle -----------------------------------------------------------------------------------------------------------
def make_store(sk, ctx, bases, off, goc, n, groups=3, sp=None, ranks=None):
    """The genomes sketched in `groups` consecutive groups, each added to the store and freed."""
    sp = sp or sk.sketch_params()
    st = sk.SketchStore(sp)
    bounds = np.linspace(0, n, groups + 1).astype(int)
    for a, b in zip(bounds[:-1], bounds[1:]):
        idx = np.nonzero((goc >= a) & (goc < b))[0]
        lo, hi = int(off[idx[0]]), int(off[idx[-1] + 1])
        s = sk.sketch_contigs(ctx, bases[lo:hi], off[idx[0]:idx[-1] + 2] - off[idx[0]], goc[idx] - a, b - a, sp)
        st.add(s)
        s.free()
    if ranks is not None:
        st.set_name_ranks(ranks)
    return st


def in_memory(sk, ctx, bases, off, goc, n, ranks=None):
    if ranks is None:
        res, _ = sk.triangle(ctx, bases, off, goc, n, as_array=True)
    else:
        res, s, _ = sk.triangle_local(ctx, bases, off, goc, n, name_ranks=ranks)
        s.free()
    return key_sort(res)


N, G = 40, 5
CASES = {   # budget as a multiple of the largest cluster's bytes (None = derived from free memory), expected case
    "single_set": (None, "single"),
    "many_sets": (1.05, "many"),
    "chunk_pairs": (0.45, "chunks"),
}


@pytest.mark.parametrize("n_ctx", [1, 2])
@pytest.mark.parametrize("ids", ["contiguous", "shuffled"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_triangle_store_equals_triangle(ctxs, case, ids, n_ctx):
    import skani_b200 as sk
    ctx = ctxs[0]
    if ids == "contiguous":
        bases, off, goc = synth.generate(0, N, L, G=G)
    else:
        bases, off, goc = synth.generate_ids(synth.shuffled_ids(N, 11), L, G=G)
    want = in_memory(sk, ctx, bases, off, goc, N)
    st = make_store(sk, ctx, bases, off, goc, N)
    gb = np.array([st.genome_bytes(g) for g in range(N)])
    mult, expect = CASES[case]
    cluster = max(gb[i:i + G].sum() for i in range(0, N, G))
    budget = 0 if mult is None else int(max(mult * cluster, 2 * gb.max() + 1))
    got, stats = sk.triangle_store(ctxs[:n_ctx], st, device_budget=budget)
    assert len(want) > N and got.tobytes() == want.tobytes()
    assert stats.gathered_bytes > 0 and (budget == 0 or stats.max_working_set_bytes <= budget)
    if expect == "single":
        assert stats.n_working_sets == 1 and stats.n_split_components == 0
    elif expect == "many":
        assert stats.n_working_sets >= N // G // 2 and stats.n_split_components == 0
    else:
        assert stats.n_split_components > 0 and stats.n_working_sets > N // G
    st.free()


def test_triangle_store_oracle_small_n(ctxs):
    import skani_b200 as sk
    n = 12
    bases, off, goc = synth.generate_ids(synth.shuffled_ids(n, 3), L, G=4)
    st = make_store(sk, ctxs[0], bases, off, goc, n, groups=2)
    gb = max(st.genome_bytes(g) for g in range(n))
    got, stats = sk.triangle_store(ctxs, st, device_budget=int(2.2 * gb))
    assert stats.n_split_components > 0
    osk = O.sketch_many(bases, off, goc, n)
    ores, _ = O.triangle(osk, O.cmd())
    exp = {(r.ref_id, r.query_id): r for r in ores}
    assert sorted(exp) == [(int(r["ref_id"]), int(r["query_id"])) for r in got] and len(exp) >= n
    for r in got:
        o = exp[(int(r["ref_id"]), int(r["query_id"]))]
        for f in ("ani", "af_query", "af_ref"):
            assert abs(float(r[f]) - getattr(o, f)) <= TOL, (r, f)
    st.free()


def test_triangle_store_individual_ranks(ctxs):
    """-i style ranks: records of one file share a rank; identical genomes tie on everything but the rank."""
    import skani_b200 as sk
    gen = split_genomes(*synth.generate(0, 12, L, G=4), 12)
    gen = gen + [gen[0], gen[5], gen[0]]                      # exact copies: switch_qr falls back to the ranks
    bases, off, goc = layout(gen)
    n = len(gen)
    ranks = np.array([g // 3 for g in range(n)], np.uint64)
    ranks[12], ranks[14] = 0, 0
    want = in_memory(sk, ctxs[0], bases, off, goc, n, ranks=ranks)
    st = make_store(sk, ctxs[0], bases, off, goc, n, ranks=ranks)
    gb = max(st.genome_bytes(g) for g in range(n))
    for budget in (0, int(2.5 * gb)):
        got, stats = sk.triangle_store(ctxs, st, device_budget=budget)
        assert got.tobytes() == want.tobytes()
        assert (stats.n_working_sets == 1) == (budget == 0)
    st.free()


def test_triangle_store_dense_cluster_chunk_pairs(ctxs):
    import skani_b200 as sk
    n = 16
    bases, off, goc = synth.generate(0, n, L, G=n)            # one cluster: every pair related
    want = in_memory(sk, ctxs[0], bases, off, goc, n)
    st = make_store(sk, ctxs[0], bases, off, goc, n)
    gb = max(st.genome_bytes(g) for g in range(n))
    got, stats = sk.triangle_store(ctxs, st, device_budget=int(4.5 * gb))
    assert len(want) >= 2 * n and got.tobytes() == want.tobytes()
    assert stats.n_split_components == 1 and stats.n_working_sets >= 10
    st.free()


# ---- errors -------------------------------------------------------------------------------------------------------------
def test_errors_fail_cleanly(ctxs):
    import skani_b200 as sk
    ctx = ctxs[0]
    n = 10
    bases, off, goc = synth.generate(0, n, L, G=5)
    st = make_store(sk, ctx, bases, off, goc, n, groups=1)
    gb = max(st.genome_bytes(g) for g in range(n))
    with pytest.raises(sk.host.SkaniError, match=r"rc=-3.*more than half"):
        sk.triangle_store(ctxs, st, device_budget=gb)
    with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*out of range"):
        st.gather(ctx, [0, n])
    with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*ascending"):
        st.gather(ctx, [3, 2])
    with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*ascending"):
        st.gather(ctx, [2, 2])
    other = sk.sketch_contigs(ctx, bases, off, goc, n, sk.sketch_params(c=200))
    with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*parameters"):
        st.add(other)
    assert st.n_genomes() == n
    # the context and the store still work
    s = sk.sketch_contigs(ctx, bases, off, goc, n)
    pairs = sk.screen_triangle(ctx, s)
    want = sk.chain_pairs(ctx, s, s, pairs, as_array=True)
    g = st.gather(ctx)
    assert sk.chain_pairs(ctx, g, g, pairs, as_array=True).tobytes() == want.tobytes()
    got, stats = sk.triangle_store(ctxs, st)
    assert got.tobytes() == key_sort(want[want["ani"] > np.float32(0.1)]).tobytes() and stats.n_working_sets == 1
    st.free()
