"""dist / search over several contexts (sk_sketch_set_copy, sk_screen_query_ref_multi, sk_chain_pairs_multi) with every
context on GPU 0: the references are split into contiguous blocks, one per context, and the query set is copied to every
context.  Screen pair lists and chain results must equal the single-context calls on one set of all refs byte for byte,
and a sample of pairs the oracle within 1e-4."""
import numpy as np
import pytest

import oracle_py as O
from bench_support import synth

pytestmark = pytest.mark.gpu
TOL = 1e-4
L, G, N = 200_000, 6, 24      # 4 clusters of 6 related genomes


def genomes():
    """Refs: members 0-3 of every cluster, a 15 kb piece of genome 1 and a 12 kb piece of genome 7 (< 20 markers each),
    and an exact copy of genome 4.  Queries: members 4-5 of every cluster and a 14 kb piece of genome 13."""
    bases, off, goc = synth.generate(0, N, L, G=G)
    gen = [[bases[int(off[i]):int(off[i + 1])] for i in np.nonzero(goc == g)[0]] for g in range(N)]
    refs = [gen[g] for g in range(N) if g % G < 4] + [[gen[1][0][:15_000]], [gen[7][0][:12_000]], gen[4]]
    queries = [gen[g] for g in range(N) if g % G >= 4] + [[gen[13][0][:14_000]]]
    return refs, queries


def layout(gs):
    contigs = [c for g in gs for c in g]
    off = np.concatenate([[0], np.cumsum([len(c) for c in contigs])]).astype(np.uint64)
    goc = np.concatenate([np.full(len(g), i, np.uint32) for i, g in enumerate(gs)])
    return np.concatenate(contigs), off, goc


def sketch(sk, ctx, gs):
    if not gs:
        return None
    bases, off, goc = layout(gs)
    return sk.sketch_contigs(ctx, bases, off, goc, len(gs))


@pytest.fixture(scope="module")
def env():
    import skani_b200 as sk
    refs, queries = genomes()
    ctxs = [sk.Context(0) for _ in range(4)]
    e = dict(sk=sk, ctxs=ctxs, refs=refs, queries=queries, rset=sketch(sk, ctxs[0], refs), qset=sketch(sk, ctxs[0], queries))
    e["qcopies"] = [e["qset"]] + [e["qset"].copy_to(c) for c in ctxs[1:]]
    yield e
    for c in ctxs:
        c.close()


def blocks(e, bounds, n_refs=None):
    """Ref blocks [bounds[d], bounds[d + 1]) sketched on context d (None for an empty block)."""
    n_refs = len(e["refs"]) if n_refs is None else n_refs
    b = list(bounds) + [n_refs]
    sets = [sketch(e["sk"], e["ctxs"][d], e["refs"][b[d]:b[d + 1]]) for d in range(len(bounds))]
    return e["ctxs"][:len(bounds)], sets, list(bounds), e["qcopies"][:len(bounds)]


def test_copy_is_identical(env):
    sk, ctxs, rset = env["sk"], env["ctxs"], env["rset"]
    assert [info["n_markers"] < 20 for info in (rset.info(g) for g in (16, 17))] == [True, True]
    pairs = np.array([(r << 32) | q for r in range(len(rset)) for q in range(0, len(env["queries"]), 3)], np.uint64)
    want = sk.chain_pairs(ctxs[0], rset, env["qset"], pairs, as_array=True)
    assert np.isfinite(want["ani"]).sum() > 5
    for dst in (ctxs[0], ctxs[1]):        # same context, and another context on the device
        cp = rset.copy_to(dst)
        assert len(cp) == len(rset)
        for g in range(len(rset)):
            a, b = rset.export(g), cp.export(g)
            for k in a:
                assert np.array_equal(a[k], b[k]), (g, k)
            assert rset.info(g) == cp.info(g)
        q = env["qcopies"][1] if dst is ctxs[1] else env["qset"]
        got = sk.chain_pairs(dst, cp, q, pairs, as_array=True)
        assert got.tobytes() == want.tobytes()
        assert sk.screen_query_ref(dst, cp, q, mode=0).tobytes() == sk.screen_query_ref(ctxs[0], rset, env["qset"], mode=0).tobytes()
        cp.free()


def test_copy_carries_name_ranks(env):
    """-i style ranks (records of one file share a rank) decide switch_qr's tie between identical genomes; the copy keeps them."""
    sk, ctxs, refs = env["sk"], env["ctxs"], env["refs"]
    s = sketch(sk, ctxs[0], [refs[0], refs[0], refs[5], refs[5]])
    pairs = [(0 << 32) | 1, (1 << 32) | 0, (2 << 32) | 3, (3 << 32) | 2]
    default = [d["switched"] for d in sk.chain_pairs_debug(ctxs[0], s, s, pairs)]
    assert default == [True, False, True, False]          # default rank = index: query index > ref index switches
    s.set_name_ranks([1, 0, 0, 0])
    want = [d["switched"] for d in sk.chain_pairs_debug(ctxs[0], s, s, pairs)]
    assert want == [False, True, False, False]
    cp = s.copy_to(ctxs[2])
    assert [d["switched"] for d in sk.chain_pairs_debug(ctxs[2], cp, cp, pairs)] == want
    assert sk.chain_pairs(ctxs[2], cp, cp, pairs, as_array=True).tobytes() == sk.chain_pairs(ctxs[0], s, s, pairs, as_array=True).tobytes()


SPLITS = {"2 uneven": [0, 3], "3 empty middle": [0, 8, 8], "3 uneven": [0, 11, 12], "4 uneven": [0, 1, 9, 10]}


@pytest.mark.parametrize("split", sorted(SPLITS))
def test_screen_multi_equals_single(env, split):
    sk, ctxs = env["sk"], env["ctxs"]
    cs, sets, rf, qs = blocks(env, SPLITS[split])
    n = 0
    for mode in range(4):
        for rescue in (True, False):
            mp = sk.map_params(rescue_small=rescue)
            want = sk.screen_query_ref(ctxs[0], env["rset"], env["qset"], mp, mode)
            got = sk.screen_query_ref_multi(cs, sets, rf, qs, mp, mode)
            assert got.dtype == np.uint64 and got.tobytes() == want.tobytes(), (mode, rescue)
            n += len(want)
            # the small genomes take part: rescued in modes 0 / 2 with rescue_small, never in 1 / 3
            small = set(range(16, 18))
            got_small = {int(p >> 32) for p in got} & small
            if mode in (0, 2) and rescue:
                assert got_small == small, mode
    assert n > 0


def test_screen_more_contexts_than_refs(env):
    sk, ctxs = env["sk"], env["ctxs"]
    sub = sketch(sk, ctxs[0], env["refs"][:3])
    cs, sets, rf, qs = blocks(env, [0, 1, 2, 3], n_refs=3)
    assert sets[3] is None
    n = 0
    for mode in range(4):
        want = sk.screen_query_ref(ctxs[0], sub, env["qset"], mode=mode)
        assert sk.screen_query_ref_multi(cs, sets, rf, qs, mode=mode).tobytes() == want.tobytes()
        n += len(want)
    assert n > 0
    pairs = sk.screen_query_ref(ctxs[0], sub, env["qset"])
    want = sk.chain_pairs(ctxs[0], sub, env["qset"], pairs, as_array=True)
    assert sk.chain_pairs_multi(cs, sets, rf, qs, pairs[::-1], as_array=True).tobytes() == want[::-1].tobytes()


@pytest.mark.parametrize("user_ranks", [False, True])
def test_chain_multi_equals_single_and_oracle(env, user_ranks):
    sk, ctxs = env["sk"], env["ctxs"]
    rset, qset = env["rset"], env["qset"]
    cs, sets, rf, qs = blocks(env, [0, 5, 5, 13])
    if user_ranks:      # -i style: refs 0-3 share one file name, the exact copy (ref 18) shares query 0's name
        rset, qset = sketch(sk, ctxs[0], env["refs"]), sketch(sk, ctxs[0], env["queries"])
        rr = np.array([0, 0, 0, 0] + list(range(1, 16)), np.uint64)
        rr[18] = 100
        rset.set_name_ranks(rr)
        for d, s in enumerate(sets):
            if s is not None:
                s.set_name_ranks(rr[rf[d]:rf[d] + len(s)])
        qset.set_name_ranks(np.arange(100, 100 + len(qset), dtype=np.uint64))
        qs = [qset] + [qset.copy_to(c) for c in cs[1:]]
    pairs = sk.screen_query_ref(ctxs[0], rset, qset, mode=0)
    extra = np.array([(18 << 32) | 0, (16 << 32) | 0, (17 << 32) | 8, (0 << 32) | 8], np.uint64)
    pairs = np.concatenate([pairs, extra])
    pairs = pairs[np.random.default_rng(7).permutation(len(pairs))]
    want = sk.chain_pairs(ctxs[0], rset, qset, pairs, as_array=True)
    got = sk.chain_pairs_multi(cs, sets, rf, qs, pairs, as_array=True)
    assert len(got) == len(pairs) > 40
    assert got.tobytes() == want.tobytes()
    assert np.array_equal(got["ref_id"].astype(np.uint64), pairs >> np.uint64(32))
    if user_ranks:
        return
    # oracle: refs are named before queries, as the default ranks order them
    refs, queries = env["refs"], env["queries"]
    ro = {}
    qo = {}
    pick = np.sort(np.random.default_rng(3).choice(len(pairs), 16, replace=False))
    for i in pick:
        r, q = int(pairs[i] >> np.uint64(32)), int(pairs[i] & np.uint64(0xFFFFFFFF))
        if r not in ro:
            ro[r] = O.sketch_from_contigs("r%03d" % r, refs[r])
        if q not in qo:
            qo[q] = O.sketch_from_contigs("q%03d" % q, queries[q])
        o = O.chain(ro[r], qo[q], O.cmd())
        for f in ("ani", "af_ref", "af_query"):
            a, b = float(got[i][f]), float(getattr(o, f))
            assert (np.isnan(a) and np.isnan(b)) or abs(a - b) <= TOL, (r, q, f, a, b)


def test_invalid_arguments_fail_cleanly(env):
    sk, ctxs = env["sk"], env["ctxs"]
    cs, sets, rf, qs = blocks(env, [0, 10])
    pairs = np.array([(3 << 32) | 1, (12 << 32) | 2], np.uint64)
    with pytest.raises(sk.host.SkaniError, match="ascending"):
        sk.screen_query_ref_multi(cs, sets, [0, 5], qs)              # blocks overlap
    with pytest.raises(sk.host.SkaniError, match="ascending"):
        sk.chain_pairs_multi(cs, sets, [10, 0], qs, pairs)
    with pytest.raises(sk.host.SkaniError, match="no block"):
        sk.chain_pairs_multi(cs, sets, rf, qs, np.array([(19 << 32) | 0], np.uint64))
    with pytest.raises(sk.host.SkaniError, match="query index"):
        sk.chain_pairs_multi(cs, sets, rf, qs, np.array([(1 << 32) | 99], np.uint64))
    with pytest.raises(sk.host.SkaniError, match="ctxs"):
        sk.chain_pairs_multi(cs, sets, rf, [qs[0], qs[0]], pairs)     # the query set of context 0 handed to context 1
    other = sk.sketch_contigs(ctxs[1], *layout(env["refs"][10:12]), 2, sk.sketch_params(c=200))
    with pytest.raises(sk.host.SkaniError, match="parameters"):
        sk.chain_pairs_multi(cs, [sets[0], other], rf, qs, pairs)
    # the contexts still work
    want = sk.chain_pairs(ctxs[0], env["rset"], env["qset"], pairs, as_array=True)
    assert sk.chain_pairs_multi(cs, sets, rf, qs, pairs, as_array=True).tobytes() == want.tobytes()
