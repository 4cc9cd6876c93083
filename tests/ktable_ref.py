"""Plain reference of the per-genome k-mer table contract (hash_build_kernel builds it, probe_kernel reads it), and of
the FracMinHash seeding that decides which k-mers a planted sequence contributes.  TEST INFRASTRUCTURE ONLY.

Table of a genome with U distinct seed k-mers and R records: none when U == 0 or R >= 2^20 (the group start must fit 20
bits); otherwise `cap` = the smallest power of two >= 16 and >= 2U entries, in cap / 4 buckets of 4 slots.  A key's home
bucket is (key * 0x9E3779B1 mod 2^32) >> (32 - log2(buckets)).  Each bucket fills front to back; a full bucket spills into
the next one, the last bucket into bucket 0.  An entry is key << 32 | start << 12 | min(count, 4095), where start is the
key's group start in the genome's k-mer view (records sorted by k-mer) and count its number of records; 0 is an empty slot
(count >= 1, so no entry is 0, key 0 included).  A probe scans from the home bucket, front to back, and stops at the first
bucket whose last slot is empty."""
import numpy as np

import seed_ref
from seed_ref import MARKER_K, is_seed, mm_hash64  # noqa: F401  (the GPU table tests use them through this module)

GOLDEN = 0x9E3779B1
COUNT_MAX = 4095                  # 12-bit count field
START_BITS = 20                   # 20-bit start field: genomes of >= 2^20 records get no table
U64 = np.uint64


def capacity(n_kmers, n_records):
    if n_kmers == 0 or n_records >= 1 << START_BITS:
        return 0
    cap = 16
    while cap < 2 * n_kmers:
        cap <<= 1
    return cap


def home(keys, cap):
    """home bucket of every key in a table of `cap` entries"""
    nb = cap // 4
    bits = nb.bit_length() - 1
    h = (np.asarray(keys, np.uint64) * U64(GOLDEN)) & U64(0xFFFFFFFF)
    return (h >> U64(32 - bits)).astype(np.int64)


def entry(keys, starts, counts):
    k, s, c = (np.asarray(x, np.uint64) for x in (keys, starts, counts))
    return (k << U64(32)) | (s << U64(12)) | np.minimum(c, U64(COUNT_MAX))


def expected(export):
    """(distinct keys, group starts, counts, capacity) of a genome, from its export() (the k-mer view, sorted by k-mer)"""
    kmer = np.asarray(export["kmer"], np.uint32)
    assert np.all(kmer[1:] >= kmer[:-1]), "export()['kmer'] is not the sorted k-mer view"
    uk, first, cnt = np.unique(kmer, return_index=True, return_counts=True)
    return uk.astype(np.uint32), first.astype(np.int64), cnt.astype(np.int64), capacity(len(uk), len(kmer))


def check_table(table, keys, starts, counts):
    """Asserts that `table` is a valid table of exactly these keys (sorted, distinct) with these group starts and counts:
    every key once with its packed entry, no stray entry, no empty slot before a filled one inside a bucket, and every bucket
    from a key's home up to (cyclically, not including) its bucket full.  Returns each key's spill distance (buckets past its
    home, in key order)."""
    t = np.asarray(table, np.uint64)
    keys = np.asarray(keys, np.uint32)
    cap = len(t)
    assert cap >= 16 and cap & (cap - 1) == 0, "capacity %d is not a power of two >= 16" % cap
    assert cap >= 2 * len(keys), "capacity %d below twice the %d keys" % (cap, len(keys))
    nb = cap // 4
    filled = (t != 0).reshape(nb, 4)
    hole = ~filled[:, :-1] & filled[:, 1:]
    assert not hole.any(), "bucket %d has an empty slot before a filled one" % int(np.nonzero(hole.any(1))[0][0])
    slot = np.nonzero(t != 0)[0]
    ek = (t[slot] >> U64(32)).astype(np.uint32)
    order = np.argsort(ek, kind="stable")
    ek, slot = ek[order], slot[order]
    dup = ek[1:] == ek[:-1]
    assert not dup.any(), "key %d stored twice" % int(ek[1:][dup][0])
    assert len(ek) == len(keys), "%d entries for %d keys" % (len(ek), len(keys))
    bad = ek != keys
    assert not bad.any(), "stray key %d (or key %d missing)" % (int(ek[bad][0]), int(keys[bad][0]))
    want = entry(keys, starts, counts)
    bad = t[slot] != want
    assert not bad.any(), "key %d: entry %#x, expected %#x (start %d, count %d)" % (
        int(keys[bad][0]), int(t[slot][bad][0]), int(want[bad][0]), int(np.asarray(starts)[bad][0]), int(np.asarray(counts)[bad][0]))
    h = home(keys, cap)
    b = slot // 4
    dist = (b - h) % nb
    notfull = np.concatenate([[0], np.cumsum(np.tile(~filled[:, 3], 2))])
    gap = notfull[h + dist] - notfull[h]          # buckets h .. h + dist - 1 (cyclic) that are not full
    bad = gap != 0
    assert not bad.any(), "key %d sits in bucket %d, home %d, past a bucket that is not full" % (
        int(keys[bad][0]), int(b[bad][0]), int(h[bad][0]))
    return dist


def probe(table, keys):
    """probe_kernel's lookup restated: home bucket, the four slots front to back, stop on an empty last slot, next bucket
    with wrap.  Returns (found, start, count) arrays (scalar key -> scalars)."""
    scalar = np.ndim(keys) == 0
    t = np.asarray(table, np.uint64).reshape(-1, 4)
    nb = len(t)
    q = np.atleast_1d(np.asarray(keys, np.uint64))
    found = np.zeros(len(q), bool)
    ent = np.zeros(len(q), np.uint64)
    b = home(q, 4 * nb)
    live = np.ones(len(q), bool)
    for _ in range(nb + 1):
        if not live.any():
            break
        i = np.nonzero(live)[0]
        row = t[b[i]]
        hit = ((row >> U64(32)) == q[i, None]) & (row != 0)
        any_hit = hit.any(1)
        j = i[any_hit]
        found[j] = True
        ent[j] = row[any_hit, np.argmax(hit[any_hit], 1)]
        live[j] = False
        stop = ~any_hit & (row[:, 3] == 0)
        live[i[stop]] = False
        b = (b + 1) % nb
    assert not live.any(), "probe does not end: every bucket is full"
    start = ((ent >> U64(12)) & U64((1 << START_BITS) - 1)).astype(np.int64)
    count = (ent & U64(COUNT_MAX)).astype(np.int64)
    return (found[0], int(start[0]), int(count[0])) if scalar else (found, start, count)


def check_lookups(table, keys, starts, counts, absent):
    """probe() finds every key with (start, min(count, 4095)) and misses every absent key"""
    f, s, c = probe(table, keys)
    assert f.all(), "key %d not found" % int(np.asarray(keys)[~f][0])
    assert np.array_equal(s, starts), "wrong start"
    assert np.array_equal(c, np.minimum(counts, COUNT_MAX)), "wrong count"
    absent = np.setdiff1d(np.asarray(absent, np.uint32), keys)
    f, _, _ = probe(table, absent)
    assert not f.any(), "absent key %d found" % int(absent[f][0])


def build_table(keys, starts, counts, cap, order=None):
    """A table built sequentially by the contract (keys inserted in `order`, default key order)"""
    t = np.zeros(cap, np.uint64)
    nb = cap // 4
    h = home(keys, cap)
    e = entry(keys, starts, counts)
    for i in (range(len(keys)) if order is None else order):
        b = int(h[i])
        while True:
            free = np.nonzero(t[4 * b:4 * b + 4] == 0)[0]
            if len(free):
                t[4 * b + free[0]] = e[i]
                break
            b = (b + 1) % nb
    return t


# ---------------------------------------------------------------------------------------------------------------------
# seeding (for planting chosen k-mers): seed_ref's restatement of the 4-lane FracMinHash seeder
# ---------------------------------------------------------------------------------------------------------------------


def window_seeds(seqs, k, c):
    """seqs: (n, L) uint8 ASCII rows of A/C/G/T.  For every window end i in [20, L) (each window a 21-mer): the seed key
    min(forward k-mer ending at i, reverse complement of the k-mer starting at i - 20) and whether it is a seed at c.
    Returns (keys (n, L - 20) uint32, is_seed (n, L - 20) bool); column j is window end 20 + j."""
    _, _, fs, rs = seed_ref.windows(seqs, k)
    seed = np.where(fs < rs, fs, rs)
    return seed.astype(np.uint32), is_seed(seed, c)


def contig_records(seq, k, c):
    """(window end positions, keys) of the records one contig contributes under the 4-lane seeder"""
    pos, keys, _, _ = seed_ref.contig_seeds(seq, k, c)
    return pos.astype(np.int64), keys
