"""chunkstat_kernel and chunk_estimate on the device against the oracle.

a. The device's chunk_estimate (sk_debug_chunk_estimate) against the oracle's over every a <= m <= 4096 and every k the
   sketch parameters accept, a random sample up to m = 20,000, and the ratios nearest 0.95^k: weights and filter decisions
   identical, estimates within EST_ULPS ulps (the largest difference is printed).
b. Synthetic pairs whose per-chunk tap (chunk_stats: sums, seed counts, filter decision) must equal the oracle's exactly,
   and which reach every branch of the kernel: more than 32 kept intervals in a chunk, chunks of about 1,024 seeds (the
   search cap), seeds on the padded interval ends, intervals starting below c, the filter applied and decided by each of its
   four conditions, chunks without intervals or shorter than 500 bp, and switched pairs.
c. Positions past 2^31: one contig of 2^31 + delta N bases and then sequence, in both roles; the padded start of an interval
   at q0 >= 2^31 + c is 0 (the reference's wrapping i32 arithmetic).  And a contig of 2^32 - 65537 bases seeds as the oracle
   does, while one base more is refused."""
import time

import numpy as np
import pytest

import oracle_py as O
from chain_testlib import (CHUNK_STAT_FIELDS, EST_ULPS, assert_debug_equal, make_sets, mutate, rand_seq, revcomp,
                           ulp_diff)

pytestmark = pytest.mark.gpu
F = {f: i for i, f in enumerate(CHUNK_STAT_FIELDS)}
KS = range(1, 17)        # sk_sketch_batch accepts 1 <= k <= 16


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# a. device pow / chunk_estimate against glibc
# ---------------------------------------------------------------------------------------------------------------------
def rows(a, m, n_seeds, ul, span=1000, tbcq=1_000_000):
    """chunk_estimate inputs: one interval, total_anchors a, num_in m"""
    n = len(a)
    x = np.zeros((n, 8), np.uint32)
    x[:, 0] = a; x[:, 1] = 100; x[:, 2] = 100 + span; x[:, 3] = tbcq; x[:, 4] = 1
    x[:, 5] = n_seeds; x[:, 6] = m; x[:, 7] = ul
    return x


def compare(ctx, x, c, k):
    import skani_b200 as sk
    ge, gw, gv = sk.host.debug_chunk_estimate(ctx, x, c, k)
    oe, ow, ov = O.chunk_estimate(x, c, k)
    bad = np.nonzero((gv != ov) | (gw != ow))[0]
    assert len(bad) == 0, ("decision / weight differ", k, x[bad[:5]].tolist(), gv[bad[:5]], ov[bad[:5]], gw[bad[:5]], ow[bad[:5]])
    u = ulp_diff(ge, oe)
    return int(u.max(initial=0)), int(np.count_nonzero(u)), len(x)


def test_device_chunk_estimate_against_glibc(ctx):
    t0 = time.time()
    worst, n_diff, n_all = 0, 0, 0
    rng = np.random.default_rng(5)
    # every a <= m <= 4096: n_seeds = 2m, upper_lower = m, so the filter decides between weight m and 2m
    m = np.repeat(np.arange(1, 4097, dtype=np.uint64), np.arange(1, 4097))
    a = np.concatenate([np.arange(1, j + 1, dtype=np.uint64) for j in range(1, 4097)])
    all_am = rows(a, m, 2 * m, m)
    for k in KS:
        sets = [all_am]
        # random sample up to m = 20,000 (a up to 1.2 m: the clamp), n_seeds up to 3 m
        m = rng.integers(1, 20_001, 2_000_000).astype(np.uint64)
        a = (rng.random(len(m)) * 1.2 * m).astype(np.uint64) + 1
        ns = m + (rng.random(len(m)) * 2 * m).astype(np.uint64)
        sets.append(rows(a, m, ns, m))
        # the ratios nearest 0.95^k for every num_in <= 2^16 (the putative-ANI filter's edge)
        m = np.arange(1, 65_537, dtype=np.uint64)
        t = np.floor(m * 0.95 ** k).astype(np.int64)
        for d in (-1, 0, 1, 2):
            a = np.maximum(t + d, 1).astype(np.uint64)
            sets.append(rows(a, m, 2 * m, m))
        for x in sets:
            w, nd, n = compare(ctx, x, 125, k)
            worst = max(worst, w); n_diff += nd; n_all += n
    print("device pow vs glibc: %d of %d estimates differ, at most %d ulp (%.1f s)" % (n_diff, n_all, worst, time.time() - t0))
    assert worst <= EST_ULPS, worst


# ---------------------------------------------------------------------------------------------------------------------
# b. synthetic pairs reaching every branch; chunk_stats equal to the oracle's
# ---------------------------------------------------------------------------------------------------------------------
def filter_conditions(cs, c, k):
    """per valid chunk: (putative > 0.95, tbcq > 4c, span < 18000, n_seeds > 1.05 upper_lower, filtered)"""
    out = []
    for r in cs:
        ta, rq0, rq1, tbcq, n_int, ns, num_in, ul, filt = (int(v) for v in r)
        if n_int == 0 or ta == 0 or rq1 - rq0 < 500:
            continue
        put = np.power(np.float64(ta) / np.float64(num_in), 1.0 / k) > 0.950
        out.append((bool(put), tbcq > 4 * c, rq1 - rq0 < 18_000, ns > 1.05 * ul, bool(filt)))
    return out


def padded_end_hits(gd, gs, qrole, c):
    """kept intervals with a query-role seed exactly on the padded start or stop"""
    e = gs.export(qrole)
    ctg = e["cc"] >> 1
    hits = 0
    for iv in gd["intervals"][gd["intervals"][:, 10] == 1]:
        q0, q1, qc = int(iv[2]), int(iv[3]), int(iv[7])
        p = set(e["pos"][ctg == qc].tolist())
        s0 = q0 - c if q0 - c > 0 else 0
        hits += (s0 in p and s0 != q0) + ((q1 + c) in p)
    return hits


def check_pairs(ctx, gs, osk, pairs, kw):
    import skani_b200 as sk
    ids = np.array([(r << 32) | q for r, q in pairs], np.uint64)
    gds = sk.chain_pairs_debug(ctx, gs, gs, ids, sk.map_params())
    for (r, q), gd in zip(pairs, gds):
        od = O.chain_debug(osk[r], osk[q], O.cmd())
        try:
            assert_debug_equal(gd, od)
        except AssertionError as ex:
            raise AssertionError("pair %s (c %d): %s" % ((r, q), kw["c"], ex))
    return gds


def test_branches_chunk_statistics(ctx):
    rng = np.random.default_rng(71)
    reach = dict(more32=0, seeds_1023=0, seeds_1024=0, seeds_1025=0, seeds_over_1024=0, pad_end_seed=0, q0_below_c=0,
                 no_intervals=0, short_chunk=0, switched_with_intervals=0, filtered=0)
    decided = {"putative": 0, "tbcq": 0, "span": 0, "considered": 0}
    cases = []
    # 1. more than 32 kept intervals in one chunk: a 21.6 kb query stretch of 48 shuffled 450 bp blocks of the reference, 6 kb
    #    apart there (too far for a chain to join two); then 400 bp pieces between 20 kb of unrelated sequence (chunks whose
    #    intervals span less than 500 bp)
    R = rand_seq(rng, 400_000)
    blocks = [R[6_000 * i:6_000 * i + 450] for i in range(48)]
    order = rng.permutation(48)
    Q = np.concatenate([blocks[i] for i in order] + [x for j in range(6) for x in (rand_seq(rng, 20_000), R[300_000 + 5_000 * j:300_400 + 5_000 * j])]
                       + [rand_seq(rng, 20_000), R[340_000:390_000]])
    cases.append((dict(c=30, k=15, marker_c=200), [[R], [Q]]))
    # 2. about 1,024 seeds per 20 kb chunk (c = 19, 20) on an 8 Mb mutated copy
    R = rand_seq(rng, 8_000_000)
    for c in (19, 20):
        cases.append((dict(c=c, k=15, marker_c=200), [[R], [mutate(rng, R, 0.01)]]))
    # 3. filter conditions: a copy with unrelated insertions (seeds outside the chunk's interval range); 20 kb periods of 3 kb
    #    unrelated + 17 kb diverged (putative below 0.95 decides); 20 kb periods of 1.5 kb unrelated + 18.5 kb related (span
    #    >= 18,000 decides); short related blocks at c = 1000 (one interval of 500 - 1,985 bp: tbcq <= 4c decides); an
    #    unrelated stretch and a 5 kb copy (a short chunk covered end to end: the seed count decides)
    R = rand_seq(rng, 3_000_000)
    ins = []
    for i in range(0, 1_000_000, 20_000):
        ins.append(mutate(rng, R[i:i + 20_000], 0.003))
        if (i // 20_000) % 3 == 0:
            ins.append(rand_seq(rng, int(rng.integers(1_000, 3_000))))
    per = [np.concatenate([rand_seq(rng, 1_500), R[1_000_000 + 20_000 * i:1_000_000 + 20_000 * i + 18_500]]) for i in range(40)]
    div = [np.concatenate([np.concatenate([rand_seq(rng, 3_000), mutate(rng, R[2_000_000 + 20_000 * i:2_000_000 + 20_000 * i + 17_000], 0.06)])
                           for i in range(20)])]
    short = [np.concatenate([np.concatenate([R[2_500_000 + 2_000 * i:2_500_000 + 2_000 * i + 2_000], rand_seq(rng, 18_000)])
                             for i in range(150)])]
    genomes = [[R], [np.concatenate(ins)], [np.concatenate(per)], div, short, [rand_seq(rng, 300_000), R[:5_000]]]
    for c in (30, 125, 1000):
        cases.append((dict(c=c, k=15, marker_c=1000), genomes))
    for kw, gen in cases:
        gs, osk = make_sets(ctx, gen, kw)
        n = len(osk)
        pairs = [(0, g) for g in range(1, n)] + [(g, 0) for g in range(1, n)]
        gds = check_pairs(ctx, gs, osk, pairs, kw)
        c = kw["c"]
        for (r, q), gd in zip(pairs, gds):
            cs = gd["chunk_stats"]
            qrole = r if gd["switched"] else q
            reach["more32"] += int(np.sum(cs[:, F["n_int"]] > 32))
            ns = cs[:, F["n_seeds"]]
            for v in (1023, 1024, 1025):
                reach["seeds_%d" % v] += int(np.sum(ns == v))
            reach["seeds_over_1024"] += int(np.sum(ns > 1024))
            kept = gd["intervals"][gd["intervals"][:, 10] == 1]
            reach["q0_below_c"] += int(np.sum((kept[:, 2] < c) & (kept[:, 2] > 0)))
            reach["no_intervals"] += int(np.sum(cs[:, F["n_int"]] == 0))
            reach["short_chunk"] += int(np.sum((cs[:, F["n_int"]] > 0) & (cs[:, F["rq1"]] - cs[:, F["rq0"]] < 500)))
            reach["switched_with_intervals"] += int(gd["switched"] and np.any(cs[:, F["n_int"]] > 0))
            reach["filtered"] += int(np.sum(cs[:, F["filtered"]]))
            if len(kept) and c <= 125:
                reach["pad_end_seed"] += padded_end_hits(gd, gs, qrole, c)
            for put, tb, sp, co, filt in filter_conditions(cs, c, 15):
                assert filt == (put and tb and sp and co)
                conds = dict(putative=put, tbcq=tb, span=sp, considered=co)
                for name in conds:
                    if not conds[name] and all(v for n2, v in conds.items() if n2 != name):
                        decided[name] += 1
    print("reached:", reach, "filter off by one condition alone:", decided)
    for name, v in reach.items():
        assert v > 0, (name, reach)
    for name, v in decided.items():
        assert v > 0, (name, decided)


# ---------------------------------------------------------------------------------------------------------------------
# c. positions past 2^31
# ---------------------------------------------------------------------------------------------------------------------
def oracle_sketch_of(buf, start, end, kw, name="g"):
    """the oracle's sketch of the one contig buf[start:end], without copying it"""
    off = np.array([0, end - start], np.uint64)
    h = O.lib().orc_sketch_from_contigs(name.encode(), buf.ctypes.data + int(start), off.ctypes.data, 1, kw["c"], kw["k"],
                                        kw["marker_c"], 1)
    return O.Sketch(h)


def test_positions_past_2_31(ctx):
    import skani_b200 as sk
    rng = np.random.default_rng(2031)
    kw = dict(c=125, k=15, marker_c=1000)
    S = rand_seq(rng, 350_000)
    # the ref copy: 1 % substitutions, 1 - 3 kb insertions every ~25 kb, and a reverse-complemented 40 kb piece
    parts, i = [], 0
    while i < len(S):
        j = min(i + int(rng.integers(20_000, 30_000)), len(S))
        piece = S[i:j]
        parts.append(revcomp(piece) if 150_000 <= i < 190_000 else mutate(rng, piece, 0.01))
        parts.append(rand_seq(rng, int(rng.integers(1_000, 3_000))))
        i = j
    T = np.concatenate(parts)
    dq, dr = 1_000, 5_003
    nq, nr = (1 << 31) + dq + len(S), (1 << 31) + dr + len(T)
    buf = np.full(nq + nr, ord("N"), np.uint8)
    buf[nq - len(S):nq] = S
    buf[nq + nr - len(T):] = T
    off = np.array([0, nq, nq + nr], np.uint64)
    gs = sk.sketch_contigs(ctx, buf, off, np.array([0, 1], np.uint32), 2, sk.sketch_params(**kw))
    osk = [oracle_sketch_of(buf, 0, nq, kw, "g000000"), oracle_sketch_of(buf, nq, nq + nr, kw, "g000001")]
    for g in (0, 1):
        e, o = gs.export(g), osk[g].export()
        for key in ("kmer", "pos", "cc", "markers"):
            assert np.array_equal(e[key], o[key]), (g, key)
        assert int(e["pos"].min()) >= 1 << 31
    pairs = [(0, 1), (1, 0)]
    gds = check_pairs(ctx, gs, osk, pairs, kw)
    wrapped = 0
    for gd in gds:
        kept = gd["intervals"][gd["intervals"][:, 10] == 1]
        assert len(kept) > 10 and kept[:, 2].min() >= 1 << 31
        wrapped += int(np.sum(kept[:, 2] >= (1 << 31) + kw["c"]))
        cs = gd["chunk_stats"]
        valid = cs[:, F["n_int"]] > 0
        # padded to 0: every chunk seed up to the interval's end counts, insertion seeds before it included
        assert np.any(valid & (cs[:, F["num_in"]] > cs[:, F["upper_lower"]]))
        assert len(gd["est"]) > 5      # (the aligned fraction of a 2 Gbp genome is below the cutoff: ani = -1)
    assert wrapped > 0
    del gs, osk, buf


@pytest.mark.parametrize("host_pack", [None, "1"])
def test_longest_contig_seeds_and_one_more_is_refused(ctx, monkeypatch, host_pack):
    import skani_b200 as sk
    if host_pack is None:
        monkeypatch.delenv("SK_HOST_PACK", raising=False)
    else:
        monkeypatch.setenv("SK_HOST_PACK", host_pack)
    kw = dict(c=125, k=15, marker_c=1000)
    rng = np.random.default_rng(4294)
    n = (1 << 32) - 65537
    buf = np.full(n + 1, ord("N"), np.uint8)
    buf[n - 200_000:n] = rand_seq(rng, 200_000)
    gs = sk.sketch_contigs(ctx, buf, np.array([0, n], np.uint64), np.array([0], np.uint32), 1, sk.sketch_params(**kw))
    e, o = gs.export(0), oracle_sketch_of(buf, 0, n, kw).export()
    for key in ("kmer", "pos", "cc", "markers", "contig_lengths"):
        assert np.array_equal(e[key], o[key]), key
    assert len(e["pos"]) > 1000 and int(e["pos"].max()) > n - 1000
    del gs
    buf[n] = ord("A")
    with pytest.raises(sk.host.SkaniError, match="rc=-2"):
        sk.sketch_contigs(ctx, buf, np.array([0, n + 1], np.uint64), np.array([0], np.uint32), 1, sk.sketch_params(**kw))
