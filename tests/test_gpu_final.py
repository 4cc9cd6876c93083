"""final_kernel (trimmed mean, std, bootstrap CI, AF cutoffs, learned ANI) bit for bit against the oracle's final_estimate.

The oracle is applied to the device's own debug tap (sorted est / weight, total_bases_covered, avg_chain_int_len, contig
quantiles), so the pow() ulp drift of the chunk estimates stays out of the comparison and every f32 field must match
exactly.  Where the device's estimates equal the oracle's bit for bit, the end-to-end result must too.  The branch tests
assert that their inputs reached the edge they are named for: 9 / 10 estimates, power-of-two lists, pools below and
above the guide table's 1,024 buckets, 1,024 / 1,025 chunks, more than 1,024 chunks with at most 1,024 estimates, more
than 65,535 estimates, and learned ANI applied and gated off by either condition.  SK_FINAL_FORCE_REDO=1 takes
the sequential bootstrap redo for every pair; the results must not change."""
import numpy as np
import pytest

import oracle_py as O
from chain_testlib import make_sets, mutate, rand_seq, synth_genomes

pytestmark = pytest.mark.gpu
F32 = ("ani", "af_query", "af_ref", "ci_lower", "ci_upper", "std", "q90_q", "q90_r", "q50_q", "q50_r", "q10_q", "q10_r")
U32 = ("avg_chain_int_len", "total_bases_covered")
GUIDE_BUCKETS = 1024
FIN_SMEM_MAX = 1024
GUIDE_MAX_N = 0xFFFF


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def pair_ids(pairs):
    return np.array([(r << 32) | q for r, q in pairs], np.uint64)


def bits(x):
    return np.float32(x).view(np.uint32)


def assert_bits(g, o, what, fields=F32):
    for f in fields:
        assert bits(getattr(g, f)) == bits(getattr(o, f)), (what, f, getattr(g, f), getattr(o, f))
    for f in U32:
        assert getattr(g, f) == getattr(o, f), (what, f, getattr(g, f), getattr(o, f))


def from_tap(gd, qlen, rlen, cp, model):
    """the oracle's final estimate of the device's own (est, weight) list and pair statistics"""
    g = gd["result"]
    return O.final_estimate(gd["est"], gd["weight"], g.total_bases_covered, g.avg_chain_int_len, qlen, rlen,
                            (g.q10_q, g.q50_q, g.q90_q), (g.q10_r, g.q50_r, g.q90_r), cp, model)


def check_taps(gs, pairs, gds, cp, model):
    """every pair with estimates: device result == final_estimate(tap), f32 bit for bit.  Returns the checked pairs."""
    checked = []
    for (r, q), gd in zip(pairs, gds):
        if len(gd["est"]) == 0:
            assert np.isnan(gd["result"].ani)
            continue
        o = from_tap(gd, gs.info(q)["total_len"], gs.info(r)["total_len"], cp, model)
        assert_bits(gd["result"], o, (r, q))
        checked.append((r, q))
    return checked


# ---------------------------------------------------------------------------------------------------------------------
# a. bit-exact from the device's own estimates, and end to end where the estimates agree
# ---------------------------------------------------------------------------------------------------------------------
SETS = {"c125": (125, 1000, 0, True), "c200": (200, 1000, 1, True), "c30_no_model": (30, 200, -1, False)}
PARAMS = ["default", "robust", "median", "learned_off", "min_af_near", "both_min_af_near"]


@pytest.fixture(scope="module")
def cluster_sets(ctx):
    out = {}
    genomes = synth_genomes(6, 400_000, 3)
    rng = np.random.default_rng(7)
    genomes.append([np.asarray(c, np.uint8).copy() for c in genomes[0]])            # an exact copy: ani 1.0
    genomes.append([mutate(rng, np.concatenate(genomes[1]), 0.11)])               # a divergent one: ani below 0.9
    genomes.append([np.concatenate(genomes[2])[50_000:160_000].copy()])           # a 110 kb piece: few bases covered
    for name, (c, mc, model, learned) in SETS.items():
        gs, osk = make_sets(ctx, genomes, dict(c=c, k=15, marker_c=mc))
        out[name] = (gs, osk)
    return out


def run(ctx, gs, pairs, mp):
    import skani_b200 as sk
    gds = sk.chain_pairs_debug(ctx, gs, gs, pair_ids(pairs), mp)
    res = sk.chain_pairs(ctx, gs, gs, pair_ids(pairs), mp, as_array=True)
    assert np.frombuffer(b"".join(bytes(gd["result"]) for gd in gds), res.dtype).tobytes() == res.tobytes()
    return gds


@pytest.mark.parametrize("param", PARAMS)
@pytest.mark.parametrize("set_name", list(SETS))
def test_final_estimate_bit_exact_from_device_estimates(ctx, cluster_sets, set_name, param):
    import skani_b200 as sk
    c, mc, model, learned = SETS[set_name]
    gs, osk = cluster_sets[set_name]
    n = len(osk)
    pairs = [(r, q) for r in range(n) for q in range(n) if r != q]
    kw = dict(learned_ani=learned and param != "learned_off", robust=param == "robust", median=param == "median")
    if param in ("min_af_near", "both_min_af_near"):
        # a cutoff on one pair's AF (its f32 value: the f64 AF lies within half an f32 ulp, on either side), so pairs
        # fall on both sides of it
        base = run(ctx, gs, pairs, sk.map_params(**kw))
        afs = sorted(float(min(gd["result"].af_query, gd["result"].af_ref)) for gd in base if len(gd["est"]))
        cut = afs[len(afs) // 2]
        kw.update(min_af=cut) if param == "min_af_near" else kw.update(both_min_af=cut)
    mp = sk.map_params(**kw)
    cp = O.cmd(**kw)
    mdl = model if kw["learned_ani"] else -1
    gds = run(ctx, gs, pairs, mp)
    checked = check_taps(gs, pairs, gds, cp, mdl)
    assert len(checked) >= len(pairs) // 3
    if param in ("min_af_near", "both_min_af_near"):
        assert any(gd["result"].ani == -1 for gd in gds) and any(gd["result"].ani > 0 for gd in gds)
    # end to end: where the device's estimates equal the oracle's bit for bit, so does the whole result (the CPU oracle
    # chains every pair: checked for the trims, once each)
    if param not in ("default", "robust", "median"):
        return
    same_est = 0
    for (r, q), gd in zip(pairs, gds):
        if len(gd["est"]) == 0:
            continue
        od = O.chain_debug(osk[r], osk[q], cp)
        if len(od["est"]) == len(gd["est"]) and od["est"].tobytes() == gd["est"].tobytes() and np.array_equal(od["weight"], gd["weight"]):
            same_est += 1
            assert_bits(gd["result"], od["result"], (r, q, "end to end"))
    assert same_est >= len(checked) // 2, (same_est, len(checked))


# ---------------------------------------------------------------------------------------------------------------------
# b. every branch of final_kernel reached
# ---------------------------------------------------------------------------------------------------------------------
def stats(gd):
    return len(gd["est"]), len(gd["chunk_first"]) - 1, int(np.sum(gd["weight"], dtype=np.uint64))


def regression_branch(gd, qlen, rlen, cp, model):
    """'applied', 'gate_ani', 'gate_bases' or 'clamped' (prediction >= 100): from the estimate without the model"""
    pre = from_tap(gd, qlen, rlen, cp, -1)
    if not np.float32(pre.ani) > np.float32(0.9):
        return "gate_ani"
    if not pre.total_bases_covered > 150_000:
        return "gate_bases"
    return "clamped" if bits(gd["result"].ani) == bits(pre.ani) else "applied"


def test_branches_list_sizes_pools_and_learned_ani(ctx):
    import skani_b200 as sk
    kw = dict(c=125, k=15, marker_c=1000)
    rng = np.random.default_rng(41)
    R = rand_seq(rng, 3_000_000)
    genomes = [[R]]
    for m in range(7, 13):                                           # m x 20 kb related end to end: 9 / 10 estimates
        a = 100_000 * m
        genomes.append([R[a:a + m * 20_000].copy()])
    for m in (16, 32):                                               # power-of-two lists
        genomes.append([R[1_300_000:1_300_000 + m * 20_000].copy()])
    genomes.append([R[2_000_000 + 3_000 * i:2_000_000 + 3_000 * i + 1_600].copy() for i in range(24)])   # pool < 1024
    genomes.append([mutate(rng, R[2_200_000:2_500_000], 0.01)])      # learned ANI applied
    genomes.append([mutate(rng, R[2_500_000:2_800_000], 0.11)])      # ani below 0.9
    genomes.append([R[2_800_000:2_900_000].copy()])                  # 100 kb: total_bases_covered <= 150,000
    genomes.append([R[0:400_000].copy()])                            # exact copy: ani 1.0 before the model
    gs, osk = make_sets(ctx, genomes, kw)
    pairs = [(0, g) for g in range(1, len(genomes))] + [(g, 0) for g in range(1, len(genomes))]
    gds = run(ctx, gs, pairs, sk.map_params())
    ns = [stats(gd)[0] for gd in gds]
    pools = [stats(gd)[2] for gd in gds if len(gd["est"]) >= 10]
    assert 9 in ns and 10 in ns, ns
    assert any(n >= 16 and n & (n - 1) == 0 for n in ns), ns
    assert min(pools) < GUIDE_BUCKETS <= max(pools), pools
    # learned ANI: the default run and a both-AF cutoff of 0.5 (partial copies get ani = -1).  These inputs do not reach a
    # prediction of 100 or more (exact copies give ani 1.0 but chain intervals of ~20 kb, and the models then predict just
    # below 100); tests/emu/emu_final.cpp covers the clamp on constructed inputs.
    kinds = set()
    for kw in ({}, dict(both_min_af=0.5)):
        mp, cp = sk.map_params(**kw), O.cmd(**kw)
        gds = gds if not kw else run(ctx, gs, pairs, mp)
        check_taps(gs, pairs, gds, cp, 0)
        kinds |= {regression_branch(gd, gs.info(q)["total_len"], gs.info(r)["total_len"], cp, 0)
                  for (r, q), gd in zip(pairs, gds) if len(gd["est"])}
    assert {"applied", "gate_ani", "gate_bases"} <= kinds, kinds


def test_branches_1024_chunks_and_global_memory_lists(ctx):
    import skani_b200 as sk
    kw = dict(c=125, k=15, marker_c=1000)
    rng = np.random.default_rng(43)
    R = rand_seq(rng, 25_000_000)
    genomes = [[R]]
    for extra in (-10_000, -2_000, 0, 5_000, 12_000, 19_000, 25_000):  # 1,024 x 20 kb related end to end, +- a chunk
        genomes.append([mutate(rng, R[:1024 * 20_000 + extra], 0.002)])
    # 25 Mbp, 8 Mbp of it related: chance anchors in the unrelated part make chunks without estimates
    genomes.append([np.concatenate([mutate(rng, R[10_000_000:18_000_000], 0.01), rand_seq(rng, 17_000_000)])])
    gs, _ = make_sets(ctx, genomes, kw)
    pairs = [(0, g) for g in range(1, len(genomes))]
    gds = run(ctx, gs, pairs, sk.map_params(robust=True))
    check_taps(gs, pairs, gds, O.cmd(robust=True), 0)
    st = [stats(gd) for gd in gds]
    ncs = [s[1] for s in st]
    assert 1024 in ncs and 1025 in ncs, ncs
    assert any(n <= FIN_SMEM_MAX < nc for n, nc, _ in st), st


def test_branch_more_than_65535_estimates(ctx):
    """~70,000 related contigs of 2.5 kb: more than 65,535 estimates (binary-search lookups, no guide table)"""
    import skani_b200 as sk
    rng = np.random.default_rng(47)
    R = rand_seq(rng, 70_000 * 2_600)
    contigs = [mutate(rng, R[2_600 * i:2_600 * i + 2_500], 0.01) for i in range(70_000)]
    gs = sk.sketch_sequences(ctx, [[R], contigs], sk.sketch_params(c=125, k=15, marker_c=1000))
    pairs = [(0, 1)]
    gds = run(ctx, gs, pairs, sk.map_params())
    assert check_taps(gs, pairs, gds, O.cmd(), 0) == pairs
    assert stats(gds[0])[0] > GUIDE_MAX_N, stats(gds[0])


# ---------------------------------------------------------------------------------------------------------------------
# c. the sequential bootstrap redo on the device
# ---------------------------------------------------------------------------------------------------------------------
def test_forced_redo_gives_identical_results(ctx, cluster_sets, monkeypatch):
    import skani_b200 as sk
    gs, osk = cluster_sets["c125"]
    n = len(osk)
    pairs = [(r, q) for r in range(n) for q in range(n) if r != q]
    rng = np.random.default_rng(53)                                   # and a pair of more than 1,024 estimates
    R = rand_seq(rng, 22_000_000)
    bs = sk.sketch_sequences(ctx, [[R], [mutate(rng, R[:21_500_000], 0.002)]], sk.sketch_params(c=125, k=15, marker_c=1000))
    big = run(ctx, bs, [(0, 1)], sk.map_params())[0]
    assert len(big["est"]) > FIN_SMEM_MAX
    assert sum(len(gd["est"]) >= 10 for gd in run(ctx, gs, pairs, sk.map_params())) > 10
    for s, p in ((gs, pairs), (bs, [(0, 1), (1, 0)])):
        for mp in (sk.map_params(), sk.map_params(robust=True)):
            a = sk.chain_pairs(ctx, s, s, pair_ids(p), mp, as_array=True)
            monkeypatch.setenv("SK_FINAL_FORCE_REDO", "1")
            b = sk.chain_pairs(ctx, s, s, pair_ids(p), mp, as_array=True)
            monkeypatch.delenv("SK_FINAL_FORCE_REDO")
            assert a.tobytes() == b.tobytes()
