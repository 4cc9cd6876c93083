"""GPU: every genome's k-mer table (hash_build_kernel) checked slot by slot against the table contract (ktable_ref), and its
lookups (probe_kernel: staged in shared memory, global, and the bucket-index search) checked through whole chain batches,
bit-exact against the oracle, at the table's rare paths: spill chains of 1 to >= 4 buckets, the last bucket wrapping into
bucket 0, the capacity edges (no table, 16, 32, 2,048 = the largest staged table, 4,096), the smallest and largest seed
keys, saturated reference-role counts, saturated query-role multiplicities, the 2^20-record edge, and the tables the
pipelined triangle appends to its merged set (growth, the fall-back to a full rebuild with the bucket index, later waves).

Genomes are built by planting chosen seed k-mers: each k-mer sits in a unit (21 - k A's, the k-mer, a seed-free spacer)
whose windows yield that k-mer and nothing else, so a genome's distinct k-mers, their counts and their home buckets are
known before it is sketched (and asserted from info() / export() after).  Each partner holds every planted k-mer once,
in the same order, plus k-mers the planted genome lacks (homed on the same busy buckets); the planted genome is longer,
so it takes the reference (probed) role."""
import numpy as np
import pytest

import ktable_ref as T
import oracle_py as O
from chain_testlib import mutate, rand_seq
from test_gpu_blob_format import layout
from test_gpu_chain_batch import assert_pair_equal, check_batch, pair_ids, roles

pytestmark = pytest.mark.gpu
TABLES = 2                      # SK_PACK_TABLES
STAGE_ENTRIES = 2048            # probe_kernel stages tables of at most this many entries in shared memory
PROBES = [{}, {"SK_PROBE_TMA": "0"}, {"SK_FORCE_BUCKET_PROBE": "1"}]
PROBE_IDS = ["default", "no_tma", "bucket_probe"]
ACGT = np.frombuffer(b"ACGT", np.uint8)


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# planting
# ---------------------------------------------------------------------------------------------------------------------
def kmer_bases(key, k):
    return ACGT[(int(key) >> (2 * np.arange(k - 1, -1, -1))) & 3]


class Planter:
    """Units that yield exactly one chosen seed k-mer at (k, c)"""

    def __init__(self, k, c, seed):
        self.k, self.c = k, c
        self.rng = np.random.default_rng(seed)
        self.P = np.full(T.MARKER_K - k, ord("A"), np.uint8)
        for _ in range(10_000):             # an 8-periodic spacer without a seed window, also where it meets the A's
            p = rand_seq(self.rng, 8)
            if not T.window_seeds(np.concatenate([np.tile(p, 8), self.P]), k, c)[1].any():
                break
        else:
            raise AssertionError("no seed-free spacer")
        self.S = np.tile(p, 3)

    def unit(self, key):
        return np.concatenate([self.P, kmer_bases(key, self.k), self.S])

    def clean(self, keys):
        """which keys yield exactly one record, of themselves, in the unit context"""
        keys = np.asarray(keys, np.uint32)
        if len(keys) == 0:
            return np.zeros(0, bool)
        rows = np.stack([np.concatenate([self.S, self.unit(x), self.S]) for x in keys])
        wk, ok = T.window_seeds(rows, self.k, self.c)
        return (ok.sum(1) == 1) & (np.where(ok, wk, 0).max(1) == keys) & T.is_seed(keys, self.c)

    def pool(self, n):
        """n distinct clean seed keys, random"""
        out = np.zeros(0, np.uint32)
        for _ in range(1_000):
            if len(out) >= n:
                break
            cand = self.rng.integers(0, 4 ** self.k, 200_000 * 2, dtype=np.uint64)
            cand = np.unique(cand[T.is_seed(cand, self.c)]).astype(np.uint32)
            out = np.union1d(out, cand[self.clean(cand)])
        assert len(out) >= n, "too few clean keys"
        return self.rng.permutation(out)[:n]

    def extreme(self, largest):
        """the smallest (largest) clean seed key"""
        top = 4 ** self.k
        for b in range(256):
            lo = top - (b + 1) * (1 << 20) if largest else b << 20
            cand = np.arange(max(lo, 0), min(lo + (1 << 20), top), dtype=np.uint64)
            cand = cand[T.is_seed(cand, self.c)].astype(np.uint32)
            cand = cand[::-1] if largest else cand
            for i in range(0, len(cand), 4096):
                ok = self.clean(cand[i:i + 4096])
                if ok.any():
                    return int(cand[i:i + 4096][ok][0])
        raise AssertionError("no clean extreme key")

    def genome(self, keys, mult=None, pad=0):
        """spacer, then every key's unit mult[i] times (consecutively), then pad more spacers"""
        mult = np.ones(len(keys), np.int64) if mult is None else np.asarray(mult)
        parts = [self.S] + [np.tile(self.unit(x), int(m)) for x, m in zip(keys, mult)] + [np.tile(self.S, pad)]
        return np.concatenate(parts)


def homed(pool, cap, want, used):
    """take keys from pool (not yet in used) homed on the buckets of `want` ({bucket: number})"""
    h = T.home(pool, cap)
    out = []
    for b, n in want.items():
        got = [int(x) for x in pool[h == b] if int(x) not in used][:n]
        assert len(got) == n, (b, n)
        used.update(got)
        out += got
    return out


def take(pool, n, used):
    got = [int(x) for x in pool if int(x) not in used][:n]
    assert len(got) == n
    used.update(got)
    return got


# ---------------------------------------------------------------------------------------------------------------------
# 1. spills, wrap, capacity edges, extreme keys and reference-role counts: one batch per k and probe setting
# ---------------------------------------------------------------------------------------------------------------------
C_EDGE = 125
BAND = 2500 // C_EDGE
SPILL = {5: 5, 15: 9, 25: 13, 40: 17}                 # 5 / 9 / 13 / 17 keys homed on one bucket: spills of >= 1 / 2 / 3 / 4
WRAP = {62: 6, 63: 5, 0: 3, 1: 2}                     # 11 keys for buckets 62-63: >= 3 wrap into bucket 0, which has 3 own
FILL = {b: 1 for b in list(range(8, 13)) + list(range(32, 37)) + list(range(47, 57))}
COUNTS = [BAND, BAND + 1, 4094, 4095, 4096, 5000]
_EDGE_CACHE = {}


def edge_cases(k):
    """{name: (planted keys, their multiplicities, keys only the partner holds)}"""
    if k in _EDGE_CACHE:
        return _EDGE_CACHE[k]
    pl = Planter(k, C_EDGE, 1000 + k)
    pool = pl.pool(6000)
    used = set()
    lo, hi = pl.extreme(False), pl.extreme(True)
    used.update([lo, hi])
    cases = {}
    busy = {**SPILL, **WRAP}
    keys = homed(pool, 256, busy, used) + homed(pool, 256, FILL, used)
    cases["spill_wrap"] = (keys, None, homed(pool, 256, {b: 3 for b in busy}, used))
    cases["u0"] = ([], None, take(pool, 20, used))
    cases["u8"] = (homed(pool, 16, {b: 2 for b in range(4)}, used), None, homed(pool, 16, {b: 1 for b in range(4)}, used))
    cases["u9"] = (take(pool, 9, used), None, take(pool, 8, used))
    cases["u1024"] = (take(pool, 1024, used), None, take(pool, 40, used))
    cases["u1025"] = (take(pool, 1025, used), None, take(pool, 40, used))
    cases["extreme"] = ([lo, hi] + take(pool, 3, used), None, take(pool, 5, used))
    ck = take(pool, len(COUNTS) + 4, used)
    cases["counts"] = (ck, COUNTS + [1] * 4, take(pool, 5, used))
    genomes, names = [], []
    for name, (keys, mult, extra) in cases.items():
        partner_keys = list(keys) + list(extra)
        partner = pl.genome(partner_keys)
        partner = pl.genome(partner_keys, pad=max(0, (600 - len(partner)) // len(pl.S) + 1))    # records of >= 500 bp
        planted = pl.genome(keys, mult)
        pad = max(0, (len(partner) + 1_000 - len(planted)) // len(pl.S) + 1)
        genomes += [[pl.genome(keys, mult, pad)], [partner]]
        names.append(name)
    _EDGE_CACHE[k] = (cases, names, genomes, (lo, hi))
    return _EDGE_CACHE[k]


def sketch_both(ctx, genomes, kw):
    import skani_b200 as sk
    gs = sk.sketch_sequences(ctx, genomes, sk.sketch_params(**kw))
    assert len(gs) == len(genomes)
    return gs


def tables(gs):
    """[(table entries, capacity)] of every genome, read from a SK_PACK_TABLES blob sliced by its ht_off words"""
    import torch
    G = len(gs)
    nb, nw = gs.subset_blob_size(None, TABLES)
    t = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    meta = gs.pack_subset(None, TABLES, t.data_ptr(), nw)
    S, U, M, Cn, HT = (int(v) for v in meta[1:5].tolist() + [meta[8]])
    off = layout(G, S, U, M, Cn, HT)[0][11]
    htab = t.cpu().numpy()[off:off + HT * 8].view(np.uint64)
    ht_off = meta[len(meta) - (G + 1):].astype(np.int64)
    assert ht_off[-1] == HT
    return [(htab[ht_off[g]:ht_off[g + 1]], int(ht_off[g + 1] - ht_off[g])) for g in range(G)]


def check_genome_table(gs, g, tab, cap, absent):
    """check_table + probe of genome g; returns (keys, counts, spill distances or None)"""
    keys, starts, counts, want_cap = T.expected(gs.export(g))
    assert cap == want_cap, (g, cap, want_cap)
    if cap == 0:
        return keys, counts, None
    d = T.check_table(tab, keys, starts, counts)
    rng = np.random.default_rng(g)
    T.check_lookups(tab, keys, starts, counts, np.concatenate([np.asarray(absent, np.uint32),
                                                               rng.integers(0, 1 << 32, 5_000).astype(np.uint32)]))
    return keys, counts, d


def assert_edges_reached(k, gs, caps, cases, names, lo_hi):
    tabs = tables(gs)
    got = {}
    for i, name in enumerate(names):
        p, q = 2 * i, 2 * i + 1
        keys, mult, extra = cases[name]
        assert gs.info(p)["n_kmers"] == len(keys) and gs.info(q)["n_kmers"] == len(keys) + len(extra), name
        assert gs.info(p)["n_records"] == (sum(mult) if mult is not None else len(keys)), name
        got[name] = check_genome_table(gs, p, *tabs[p], absent=gs.export(q)["kmer"])
        check_genome_table(gs, q, *tabs[q], absent=gs.export(p)["kmer"])
    assert [caps[2 * names.index(n)] for n in ("u0", "u8", "u9", "u1024", "u1025")] == [0, 16, 32, 2048, 4096]
    # spill chains and the wrap
    keys, _, d = got["spill_wrap"]
    t = tabs[2 * names.index("spill_wrap")][0]
    h = T.home(keys, 256)
    for need, b in enumerate(SPILL, 1):
        assert d[h == b].max() >= need, (b, d[h == b])
    assert d.max() >= 4
    full = (t.reshape(-1, 4) != 0)[:, 3]
    assert full[62] and full[63] and full[0], "no full chain from bucket 62 across the end"
    wrapped = (h + d) >= 64
    assert wrapped.any(), "no key stored before its home"
    assert np.any(((h + d) % 64 == 0) & (h >= 62)), "no wrapped key in bucket 0"
    # extreme keys
    lo, hi = lo_hi
    ek = got["extreme"][0]
    assert ek.min() == lo and ek.max() == hi
    if k == 16:
        assert hi >= 1 << 31, hex(hi)                      # keys use all 32 bits
    # saturated reference-role counts: entry count 4095, start untouched (check_table compared both fields)
    ck, cc, _ = got["counts"]
    assert sorted(cc.tolist()) == sorted(COUNTS + [1] * 4)
    t = tabs[2 * names.index("counts")][0]
    f, s, c = T.probe(t, ck)
    assert f.all() and sorted(c.tolist()) == sorted([min(x, 4095) for x in COUNTS] + [1] * 4)


def edge_pairs(names):
    return [p for i in range(len(names)) for p in ((2 * i, 2 * i + 1), (2 * i + 1, 2 * i))]


@pytest.mark.parametrize("env", PROBES, ids=PROBE_IDS)
@pytest.mark.parametrize("k", [13, 15, 16])
def test_table_edges_and_lookups(ctx, monkeypatch, k, env):
    for name, v in env.items():
        monkeypatch.setenv(name, v)
    cases, names, genomes, lo_hi = edge_cases(k)
    kw = dict(c=C_EDGE, k=k, marker_c=1000)
    gs = sketch_both(ctx, genomes, kw)
    caps = [T.capacity(gs.info(g)["n_kmers"], gs.info(g)["n_records"]) for g in range(len(gs))]
    if "SK_FORCE_BUCKET_PROBE" not in env:
        assert_edges_reached(k, gs, caps, cases, names, lo_hi)
    else:
        assert all(cap == 0 for _, cap in tables(gs))          # no tables: every probe searches the bucket index
    osk = [O.sketch_from_contigs("g%06d" % g, cs, **kw) for g, cs in enumerate(genomes)]
    pairs = edge_pairs(names)
    gds = check_batch(ctx, gs, osk, pairs)
    n_small = 0
    for (r, q), gd in zip(pairs, gds):
        p = min(r, q)                                           # the planted genome of the pair
        assert len(genomes[p][0]) > len(genomes[p ^ 1][0])     # longer (< 100 kb or no markers): the reference role
        if len(gd["anchors"]):
            assert roles(gd, r, q)[1] == p, (r, q)
        n_small += 0 < caps[p] <= STAGE_ENTRIES
    with_anchors = {names[min(r, q) // 2] for (r, q), gd in zip(pairs, gds) if len(gd["anchors"])}
    assert with_anchors == set(names) - {"u0"}, with_anchors
    # probe_kernel<STAGED> (chain.cu: 2 * small tables >= pairs) with the 4,096-entry table taking its global branch
    assert 2 * n_small >= len(pairs) and caps[2 * names.index("u1025")] > STAGE_ENTRIES
    counts = gds[2 * names.index("counts")]
    assert len(counts["anchors"]) == BAND + 4                  # band copies hit, band + 1 and above dropped


@pytest.mark.parametrize("k", [13, 15, 16])
def test_query_ref_batch_probes_the_second_sets_tables(ctx, k):
    """pairs of a reference set and a query set in which the query-set genome is probed (switched): pd.rset = 1"""
    import skani_b200 as sk
    cases, names, genomes, _ = edge_cases(k)
    kw = dict(c=C_EDGE, k=k, marker_c=1000)
    refs = sketch_both(ctx, genomes[1::2], kw)                 # partners
    qs = sketch_both(ctx, genomes[0::2], kw)                   # planted genomes
    oref = [O.sketch_from_contigs("r%06d" % g, cs, **kw) for g, cs in enumerate(genomes[1::2])]
    oq = [O.sketch_from_contigs("q%06d" % g, cs, **kw) for g, cs in enumerate(genomes[0::2])]
    pairs = [(i, i) for i in range(len(names))] + [(0, 3), (4, 1)]
    gds = sk.chain_pairs_debug(ctx, refs, qs, pair_ids(pairs), sk.map_params())
    res = sk.chain_pairs(ctx, refs, qs, pair_ids(pairs), sk.map_params(), as_array=True)
    assert np.frombuffer(b"".join(bytes(gd["result"]) for gd in gds), res.dtype).tobytes() == res.tobytes()
    n_sw = 0
    for (r, q), gd in zip(pairs, gds):
        assert_pair_equal(gd, O.chain_debug(oref[r], oq[q]))
        n_sw += bool(len(gd["anchors"]) and gd["switched"])
    assert n_sw >= len(names) - 1


# ---------------------------------------------------------------------------------------------------------------------
# 2. query-role multiplicity saturating at 65,535
# ---------------------------------------------------------------------------------------------------------------------
MULTS = [65535, 65536, 65539]


_MULT_CACHE = {}


def mult_genomes(k):
    if k in _MULT_CACHE:
        return _MULT_CACHE[k]
    pl = Planter(k, C_EDGE, 77 + k)
    keys = [int(x) for x in pl.pool(3)]
    rng = np.random.default_rng(78)
    backbone = rand_seq(rng, 400_000)
    ref = np.concatenate([backbone, pl.genome(keys)])
    qry = np.concatenate([mutate(rng, backbone[:40_000], 0.005), pl.genome(keys, MULTS)])
    genomes = [[ref], [qry]]
    kw = dict(c=C_EDGE, k=k, marker_c=1000)
    _MULT_CACHE[k] = keys, genomes, kw, [O.sketch_from_contigs("g%06d" % g, cs, **kw) for g, cs in enumerate(genomes)]
    return _MULT_CACHE[k]


@pytest.mark.parametrize("env", PROBES, ids=PROBE_IDS)
@pytest.mark.parametrize("k", [13, 15, 16])
def test_query_role_multiplicity_saturates(ctx, monkeypatch, k, env):
    for name, v in env.items():
        monkeypatch.setenv(name, v)
    keys, genomes, kw, osk = mult_genomes(k)
    gs = sketch_both(ctx, genomes, kw)
    eq, er = gs.export(1), gs.export(0)
    uk, cnt = np.unique(eq["kmer"], return_counts=True)
    assert [int(cnt[np.searchsorted(uk, x)]) for x in keys] == MULTS
    assert np.isin(keys, er["kmer"]).all()
    gds = check_batch(ctx, gs, osk, [(0, 1), (1, 0)])
    for (r, q), gd in zip([(0, 1), (1, 0)], gds):
        assert roles(gd, r, q) == (1, 0)                       # the repeat-rich genome is iterated
        assert len(gd["anchors"]) > 100
        kpos = set(eq["pos"][np.isin(eq["kmer"], keys)].tolist())
        assert not any(int(a[1]) in kpos for a in gd["anchors"] if a[0] == 0)   # no anchor from a saturated k-mer


# ---------------------------------------------------------------------------------------------------------------------
# 3. the 2^20-record edge: a table whose largest start is at the top of the 20-bit field, and no table one record later
# ---------------------------------------------------------------------------------------------------------------------
C_REC = 6


def cut_contigs(rng, target, k):
    """one or two contigs of random sequence with exactly `target` records at (k, C_REC) (lengths multiples of 4: the
    4-lane seeder visits every window)"""
    seq = rand_seq(rng, int(target * C_REC * 1.08))
    pos, _ = T.contig_records(seq, k, C_REC)
    assert len(pos) > target
    n4 = np.arange(500, len(seq) + 1, 4)
    got = np.searchsorted(pos, n4)                              # records of the prefix of length n4
    hit = np.nonzero(got == target)[0]
    if len(hit):
        return [seq[:int(n4[hit[0]])]]
    i = int(np.nonzero(got <= target - 300)[0][-1])
    main, r = seq[:int(n4[i])], target - int(got[i])
    for _ in range(100):
        s = rand_seq(rng, 4_000)
        p, _ = T.contig_records(s, k, C_REC)
        m = np.arange(500, 4_001, 4)
        h = np.nonzero(np.searchsorted(p, m) == r)[0]
        if len(h):
            return [main, s[:int(m[h[0]])]]
    raise AssertionError("record count not reachable")


_RECORD_CACHE = {}


def record_edge(k):
    """genomes of 2^20 - 1 and 2^20 records at (k, C_REC), each followed by its partner"""
    if k in _RECORD_CACHE:
        return _RECORD_CACHE[k]
    rng = np.random.default_rng(2 ** 20 + k)
    genomes = []
    for target in ((1 << 20) - 1, 1 << 20):
        g = cut_contigs(rng, target, k)
        whole = np.concatenate(g)
        pos, keys = T.contig_records(g[0], k, C_REC)
        p = int(pos[np.argmax(keys)])                            # the query covers the largest k-mer's group
        a = max(0, p - 100_000)
        qs = mutate(rng, g[0][a:a + 200_000], 0.01)
        qs[p - a - 50:p - a + 50] = g[0][p - 50:p + 50]
        assert len(whole) > 1_000_000
        genomes += [g, [qs]]
    kw = dict(c=C_REC, k=k, marker_c=200)
    _RECORD_CACHE[k] = genomes, kw, [O.sketch_from_contigs("g%06d" % g, cs, **kw) for g, cs in enumerate(genomes)]
    return _RECORD_CACHE[k]


@pytest.mark.parametrize("env", PROBES, ids=PROBE_IDS)
@pytest.mark.parametrize("k", [13, 15, 16])
def test_record_count_edge(ctx, monkeypatch, k, env):
    for name, v in env.items():
        monkeypatch.setenv(name, v)
    genomes, kw, osk = record_edge(k)
    gs = sketch_both(ctx, genomes, kw)
    assert [gs.info(g)["n_records"] for g in (0, 2)] == [(1 << 20) - 1, 1 << 20]
    if "SK_FORCE_BUCKET_PROBE" not in env:
        tabs = tables(gs)
        keys, starts, counts, cap = T.expected(gs.export(0))
        assert tabs[2][1] == 0 and cap == tabs[0][1] > 0
        assert starts.max() == (1 << 20) - 1 - counts[-1] and starts.max() >= (1 << 20) - 16   # top of the 20-bit field
        check_genome_table(gs, 0, *tabs[0], absent=gs.export(1)["kmer"])
    gds = check_batch(ctx, gs, osk, [(0, 1), (1, 0), (2, 3), (3, 2)])
    for (r, q), gd in zip([(0, 1), (1, 0), (2, 3), (3, 2)], gds):
        big = min(r, q) & ~1
        assert roles(gd, r, q) == (big + 1, big) and len(gd["anchors"]) > 10_000
        assert gs.export(big)["kmer"].max() in set(gs.export(big + 1)["kmer"].tolist())


# ---------------------------------------------------------------------------------------------------------------------
# 4. tables grown in place: the pipelined triangle's merged set
# ---------------------------------------------------------------------------------------------------------------------
BIG_PATTERN = b"TGGCGTAAA"          # 9-periodic: 3 of its 9 windows are seeds at (k = 15, c = 125), one record per 3 bases
N_DENSE = 14
OLD = 8                 # genomes OLD and OLD + 1 have tables the growth copies; their shorter relatives probe the copies


def plantable_keys(rng, n, k, c):
    """n distinct seed keys that a window of (21 - k) A's followed by the key always yields, whatever surrounds it: the key
    starts with A and the reverse strand of the window starts with the complement of its base 2k - 21 (not T), so it is
    the larger strand"""
    out = np.zeros(0, np.uint32)
    while len(out) < n:
        x = rng.integers(0, 4 ** (k - 1), 4_000_000, dtype=np.uint64)
        x = x[((x >> np.uint64(2 * (21 - k) - 2)) & np.uint64(3)) != 3]
        out = np.union1d(out, x[T.is_seed(x, c)].astype(np.uint32))
    return rng.permutation(out)[:n]


def dense_genome(pl, keys):
    """every key's 21-base window back to back (a record per 21 bases), then a spacer"""
    P = pl.P
    return np.concatenate([np.concatenate([P, kmer_bases(x, pl.k)]) for x in keys] + [pl.S])


def dense_with_kmers(pl, keys, lo, hi):
    """the shortest prefix of `keys` whose dense genome has lo < distinct k-mers <= hi"""
    n = int(lo / 1.16)
    for _ in range(40):
        g = dense_genome(pl, keys[:n])
        u = len(np.unique(T.contig_records(g, pl.k, pl.c)[1]))
        if lo < u <= hi:
            return g, keys[n:]
        n += max(1, int((lo + hi) / 2 - u) * 6 // 7) if u <= lo else -max(1, int(u - (lo + hi) / 2) * 6 // 7)
    raise AssertionError("distinct k-mer count not reachable")


def ht_reserve(total_bytes, n, c):
    """table slots the pipelined triangle's merged set reserves up front (append_sets_inplace): 4 per expected record"""
    S = int(total_bytes / c * 1.06) + 64 * n + 1024
    return 4 * S + 16 * n


@pytest.fixture(scope="module")
def pipeline_genomes():
    k, c = 15, C_EDGE
    pl = Planter(k, c, 4242)
    rng = np.random.default_rng(4243)
    keys = plantable_keys(rng, 70_000, k, c)
    genomes = []
    for _ in range(N_DENSE // 2):                          # related pairs: the second copy has 5 % of its units replaced
        g, keys = dense_with_kmers(pl, keys, 4096, 4160)  # 4,097 - 4,160 distinct k-mers: 16,384-slot table
        n_units = (len(g) - len(pl.S)) // T.MARKER_K
        units = [g[i * T.MARKER_K:(i + 1) * T.MARKER_K] for i in range(n_units)]
        repl = rng.choice(n_units, n_units // 20, replace=False)
        for i, x in zip(repl, keys[:len(repl)]):
            units[i] = np.concatenate([pl.P, kmer_bases(x, k)])
        keys = keys[len(repl):]
        genomes += [[g], [np.concatenate(units + [pl.S])]]
    for g in (genomes[OLD][0], genomes[OLD + 1][0]):
        genomes.append([g[:(len(g) // T.MARKER_K) * 3 // 5 * T.MARKER_K]])   # the first 60 %: the original is probed
    backbone = rand_seq(rng, 200_000)
    block = np.tile(np.frombuffer(BIG_PATTERN, np.uint8), (1 << 20) // 3 + 2_000)
    genomes.append([np.concatenate([backbone, pl.S, block])])              # >= 2^20 records: no table, bucket index
    genomes.append([mutate(rng, backbone[20_000:170_000], 0.01)])         # probes it through the bucket index
    for lo, hi in ((1024, 1100), (600, 700)):                               # related pairs after it
        e, keys = dense_with_kmers(pl, keys, lo, hi)
        genomes += [[e], [mutate(rng, e, 0.002)]]
    return genomes


def test_pipelined_triangle_grows_tables_in_place(ctx, monkeypatch, capfd, pipeline_genomes):
    """sk_triangle's pipeline merges each wave into one set and appends the wave's k-mer tables to it (build_hash_range):
    the table array grows (1.5x, old tables copied) when a wave exceeds the slots reserved from the input size, a genome
    of >= 2^20 records makes it rebuild every table plus the bucket index, and every later wave is rebuilt in full.  That
    merged set is internal, so the results are what is compared: byte for byte with the unpipelined triangle, and every
    kept pair against the oracle within 1e-4.  The waves are read from the SK_TRACE lines; the growth is re-derived from
    the reserve rule and each genome's table size."""
    import re
    import skani_b200 as sk
    genomes = pipeline_genomes
    n = len(genomes)
    late, big = N_DENSE, N_DENSE + 2
    kw = dict(c=C_EDGE, k=15, marker_c=1000)
    sp = sk.sketch_params(**kw)
    bases = np.concatenate([g[0] for g in genomes])
    off = np.concatenate([[0], np.cumsum([len(g[0]) for g in genomes])]).astype(np.uint64)
    goc = np.arange(n, dtype=np.uint32)
    gs = sketch_both(ctx, genomes, kw)
    info = [gs.info(g) for g in range(n)]
    gs.free()
    caps = np.array([T.capacity(i["n_kmers"], i["n_records"]) for i in info])
    assert info[big]["n_records"] >= 1 << 20 and caps[big] == 0 and (caps[:big] > 0).all() and (caps[big + 1:] > 0).all()
    monkeypatch.setenv("SK_NO_PIPELINE", "1")
    r0, _ = sk.triangle(ctx, bases, off, goc, n, sp, as_array=True)
    monkeypatch.delenv("SK_NO_PIPELINE")
    monkeypatch.setenv("SK_FORCE_PIPELINE", "1")
    monkeypatch.setenv("SK_SUBBATCH_BYTES", "1")                   # one genome per sub-batch
    monkeypatch.setenv("SK_TRACE", "1")
    capfd.readouterr()
    r1, _ = sk.triangle(ctx, bases, off, goc, n, sp, as_array=True)
    trace = capfd.readouterr().err
    waves = [(int(a), int(b)) for a, b in re.findall(r"worker: genomes >= (\d+) \((\d+) new\)", trace)]
    assert [w[0] for w in waves] == np.cumsum([0] + [w[1] for w in waves[:-1]]).tolist() and sum(w[1] for w in waves) == n
    ends = np.cumsum([w[1] for w in waves])
    wave_of = lambda g: int(np.searchsorted(ends, g, side="right"))     # noqa: E731
    w_big = wave_of(big)
    assert len(waves) >= 4 and w_big >= 2 and w_big < len(waves) - 1, waves    # tabled waves before it, more after it
    grown = [w for w in range(w_big) if caps[:ends[w]].sum() > ht_reserve(int(off[-1]), n, C_EDGE)]
    assert grown, "no wave before the large genome outgrows the reserved table slots"
    # the first growth copies OLD's table (it arrived in an earlier wave); OLD's relative probes the copy before the
    # large genome's rebuild replaces every table
    assert wave_of(OLD + 1) < grown[0] < wave_of(late) <= wave_of(late + 1) < w_big, (waves, grown)
    k0 = np.sort(r0, order=["ref_id", "query_id"]); k1 = np.sort(r1, order=["ref_id", "query_id"])
    assert len(k0) == len(k1) and k0.tobytes() == k1.tobytes()
    got = {(int(r["ref_id"]), int(r["query_id"])): r for r in k1}
    pairs = {(i, i + 1) for i in range(0, N_DENSE, 2)} | {(OLD, late), (OLD + 1, late + 1)} | {(i, i + 1) for i in range(big, n, 2)}
    assert pairs <= set(got), sorted(got)                         # every planted pair, and the large genome's
    osk = [O.sketch_from_contigs("g%06d" % g, cs, **kw) for g, cs in enumerate(genomes)]
    for (r, q), x in got.items():
        o = O.chain(osk[r], osk[q])
        for f in ("ani", "af_ref", "af_query"):
            assert abs(float(x[f]) - getattr(o, f)) <= 1e-4, ((r, q), f)
