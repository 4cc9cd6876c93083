"""CPU: the k-mer table checker of ktable_ref rejects every kind of broken table, its probe restatement finds wrapped keys
and misses absent ones, and its seeding restatement gives the oracle's records (the GPU table tests plant k-mers with it)."""
import numpy as np
import pytest

import ktable_ref as T
import oracle_py as O
from chain_testlib import rand_seq

CAP = 64                                   # 16 buckets
NB = CAP // 4


def keys_homed(buckets, rng, cap=CAP):
    """one distinct random key per entry of `buckets`, homed on that bucket"""
    out, used = [], set()
    for b in buckets:
        while True:
            k = int(rng.integers(0, 1 << 32))
            if k not in used and T.home(k, cap) == b:
                used.add(k); out.append(k)
                break
    return np.array(out, np.uint32)


def fixture_table(seed=1):
    """keys homed so that bucket 3 spills twice (9 keys), the last bucket wraps into 0 and 1 (7 keys + 2 + 1), sorted"""
    rng = np.random.default_rng(seed)
    keys = keys_homed([3] * 9 + [NB - 1] * 7 + [0] * 2 + [1] + [8, 9, 9], rng)
    o = np.argsort(keys)
    keys = keys[o]
    starts = np.arange(len(keys)) * 7 + 3
    counts = np.array([1, 2, 4095, 4096, 5000] + [3] * (len(keys) - 5))
    return keys, starts, counts, T.build_table(keys, starts, counts, CAP)


def slot_of(t, key):
    return int(np.nonzero((t >> np.uint64(32)) == key)[0][0])


def test_valid_table_passes_and_reports_spills():
    keys, starts, counts, t = fixture_table()
    d = T.check_table(t, keys, starts, counts)
    h = T.home(keys, CAP)
    assert d[h == 3].max() == 2 and sorted(d[h == 3].tolist()).count(0) == 4
    wrapped = (h + d) >= NB
    assert wrapped.sum() == 3                              # the last bucket's 7 keys: 4 stay, 3 wrap into bucket 0 / 1
    assert np.array_equal(T.entry(keys, starts, counts) >> np.uint64(32), keys.astype(np.uint64))
    for order in (np.arange(len(keys))[::-1], np.random.default_rng(2).permutation(len(keys))):   # any insertion order
        T.check_table(T.build_table(keys, starts, counts, CAP, order), keys, starts, counts)


def test_probe_finds_wrapped_keys_and_misses_absent_ones():
    keys, starts, counts, t = fixture_table()
    h = T.home(keys, CAP)
    d = T.check_table(t, keys, starts, counts)
    for i in np.nonzero(h + d >= NB)[0]:
        assert slot_of(t, keys[i]) // 4 < h[i]              # stored before its home: it wrapped
        assert T.probe(t, int(keys[i])) == (True, int(starts[i]), int(min(counts[i], 4095)))
    rng = np.random.default_rng(3)
    absent = np.concatenate([keys_homed([NB - 1, NB - 1, 0, 3, 5], rng), rng.integers(0, 1 << 32, 2000).astype(np.uint32)])
    T.check_lookups(t, keys, starts, counts, absent)
    assert not T.probe(t, 0)[0]                              # key 0 is not an empty slot's key
    k0 = np.array([0], np.uint32)
    t0 = T.build_table(k0, [5], [1], 16)
    assert T.probe(t0, 0) == (True, 5, 1)
    T.check_table(t0, k0, [5], [1])


def rejects(t, keys, starts, counts, match):
    with pytest.raises(AssertionError, match=match):
        T.check_table(t, keys, starts, counts)


def test_rejects_key_past_an_empty_last_slot():
    keys, starts, counts, t = fixture_table()
    h = T.home(keys, CAP)
    i = int(np.nonzero(h == 8)[0][0])                      # bucket 8 holds one key; move it into bucket 9's free slot
    s = slot_of(t, keys[i])
    t2 = t.copy()
    free9 = 4 * 9 + int(np.nonzero(t2[36:40] == 0)[0][0])
    t2[free9], t2[s] = t2[s], 0
    rejects(t2, keys, starts, counts, "past a bucket that is not full")


def test_rejects_key_before_its_home_without_wrap():
    keys, starts, counts, t = fixture_table()
    h = T.home(keys, CAP)
    i = int(np.nonzero(h == 9)[0][0])
    s = slot_of(t, keys[i])
    t2 = t.copy()
    dst = 4 * 8 + int(np.nonzero(t2[32:36] == 0)[0][0])   # one bucket before its home: cyclically 15 buckets past it
    t2[dst], t2[s] = t2[s], 0
    t2[4 * 9:4 * 9 + 4] = np.sort(t2[4 * 9:4 * 9 + 4])[::-1]   # keep bucket 9 front-filled
    rejects(t2, keys, starts, counts, "past a bucket that is not full")


def test_rejects_duplicated_key():
    keys, starts, counts, t = fixture_table()
    t2 = t.copy()
    s = slot_of(t, keys[0])
    free = int(np.nonzero(t2.reshape(-1, 4)[:, 0] == 0)[0][0]) * 4
    t2[free] = t2[s]
    rejects(t2, keys, starts, counts, "stored twice")


def test_rejects_hole_in_a_bucket():
    keys, starts, counts, t = fixture_table()
    t2 = t.copy()
    b = int(T.home(keys[T.home(keys, CAP) == 8][0], CAP))
    t2[4 * b + 1], t2[4 * b] = t2[4 * b], 0
    rejects(t2, keys, starts, counts, "empty slot before a filled one")


@pytest.mark.parametrize("field", ["start", "count", "saturation", "key_bits"])
def test_rejects_wrong_entry(field):
    keys, starts, counts, t = fixture_table()
    t2 = t.copy()
    i = 3                                                    # count 4096: stored saturated at 4095
    s = slot_of(t, keys[i])
    if field == "start":
        t2[s] += np.uint64(1 << 12)
    elif field == "count":
        t2[s] -= np.uint64(1)
    elif field == "saturation":                              # 4096 wrapped into the 12-bit field instead of saturating
        t2[s] = (t2[s] & ~np.uint64(0xFFF)) | np.uint64(4096 & 0xFFF)
    else:
        t2[s] ^= np.uint64(1 << 40)
    rejects(t2, keys, starts, counts, "entry|stray")


def test_rejects_missing_and_stray_entries():
    keys, starts, counts, t = fixture_table()
    t2 = t.copy()
    t2[slot_of(t, keys[5])] = 0
    t2 = t2.reshape(-1, 4)
    t2 = np.array([np.concatenate([r[r != 0], r[r == 0]]) for r in t2]).reshape(-1)    # front-filled again
    rejects(t2, keys, starts, counts, "entries for")
    rejects(t, keys[1:], starts[1:], counts[1:], "entries for")


def test_probe_restatement_stops_on_the_last_slot_only():
    """a bucket with an empty FIRST slot cannot exist in a valid table; a full bucket without the key continues the chain"""
    keys, starts, counts, t = fixture_table()
    h = T.home(keys, CAP)
    d = T.check_table(t, keys, starts, counts)
    far = np.nonzero((h == 3) & (d == 2))[0]
    assert len(far)
    assert all(T.probe(t, int(keys[i]))[0] for i in far)     # two full buckets crossed
    full = np.full(CAP, 0, np.uint64)
    full[:] = T.entry(np.arange(CAP) + 1, np.zeros(CAP), np.ones(CAP))
    with pytest.raises(AssertionError, match="does not end"):
        T.probe(full, 0)


@pytest.mark.parametrize("k", [13, 15, 16])
@pytest.mark.parametrize("c", [6, 125])
def test_seeding_restatement_equals_oracle(k, c):
    rng = np.random.default_rng(k * 1000 + c)
    contigs = [rand_seq(rng, n) for n in (600, 1_001, 5_002, 20_003)]
    contigs.append(np.tile(np.frombuffer(b"ACGTTGCAAC", np.uint8), 70))
    o = O.sketch_from_contigs("g", contigs, c=c, k=k, marker_c=max(c, 200)).export()
    pos, key, ctg = [], [], []
    for ci, s in enumerate(contigs):
        p, kk = T.contig_records(s, k, c)
        pos.append(p); key.append(kk); ctg.append(np.full(len(p), ci))
    pos, key, ctg = (np.concatenate(x) for x in (pos, key, ctg))
    mine = np.lexsort((pos, ctg))
    theirs = np.lexsort((o["pos"], o["cc"] >> 1))
    assert len(mine) == len(theirs) > 0
    assert np.array_equal(pos[mine], o["pos"][theirs]) and np.array_equal(ctg[mine], (o["cc"] >> 1)[theirs])
    assert np.array_equal(key[mine], o["kmer"][theirs])
    assert np.all(T.is_seed(key, c)) and T.expected(o)[3] == T.capacity(len(np.unique(key)), len(key))


def test_key_zero_is_no_seed_at_any_chaining_c():
    """the all-A k-mer hashes to 0x77cf...: a seed only for c <= 2, so the GPU tests plant the smallest reachable seed key"""
    h0 = int(O.lib().orc_mm_hash64(0))
    assert int(T.mm_hash64(0)) == h0
    assert not any(T.is_seed(0, c) for c in range(6, 1001))
