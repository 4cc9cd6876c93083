"""CPU: seed_ref (the numpy restatement of both seeders and of a genome's layout) against the CPU oracle, bit for bit, under
the AVX2 and the scalar semantics, on the seeding parity set and on every input seed_cases builds for the GPU edge tests.
The two restatements of the reference check each other here before either judges the GPU."""
import numpy as np
import pytest

import oracle_py as O
import seed_cases as SC
import seed_ref as R
from test_gpu_seeding import parity_set

SEM = [True, False]
SEM_IDS = ["avx2", "scalar"]


def oracle_contig(s, c, k, mc, avx2):
    """the oracle's seeder on one contig of any length (its sketch_from_contigs drops contigs under 500 bases)"""
    buf = np.ascontiguousarray(s, np.uint8)
    return O.Sketch(O.lib().orc_seed_one_contig(buf.ctypes.data, len(buf), c, k, mc, int(avx2))).export()


def check_genome(contigs, c, k, mc, avx2):
    """seed_ref equals the oracle on every contig alone, and on the genome of its contigs of >= 500 bases"""
    for s in contigs:
        e, r = oracle_contig(s, c, k, mc, avx2), R.sketch([s], k, c, mc, avx2)
        for key in ("kmer", "pos", "cc", "markers"):
            assert np.array_equal(r[key], e[key]), (len(s), key)
    long = [s for s in contigs if len(s) >= 500]
    if long:
        o = O.sketch_from_contigs("g", long, c=c, k=k, marker_c=mc, avx2sem=avx2)
        e, r = o.export(), R.sketch(long, k, c, mc, avx2)
        for key in ("kmer", "pos", "cc", "markers", "contig_lengths"):
            assert np.array_equal(r[key], e[key]), key
        assert len(r["ukmer"]) == o.n_kmers
    return R.sketch(contigs, k, c, mc, avx2)


def check_genomes(genomes, c, k, mc, avx2):
    return [check_genome(g, c, k, mc, avx2) for g in genomes]


def test_byte_to_seq_table():
    """src/types.rs:40-49: bytes 0..3 map to themselves, C/c 1, G/g 2, T/t/U/u 3, every other byte 0; only 'N' breaks a
    window under the AVX2 semantics, 'N' and 'n' under the scalar ones"""
    want = {b: 0 for b in range(256)}
    want.update({0: 0, 1: 1, 2: 2, 3: 3})
    for ch, v in zip(b"CGTUcgtu", (1, 2, 3, 3, 1, 2, 3, 3)):
        want[ch] = v
    assert R.BYTE_TO_SEQ.tolist() == [want[b] for b in range(256)]
    b = np.arange(256, dtype=np.uint8)
    assert np.nonzero(R.is_n(b, True))[0].tolist() == [78]
    assert np.nonzero(R.is_n(b, False))[0].tolist() == [78, 110]
    assert all(int(R.mm_hash64(x)) == int(O.lib().orc_mm_hash64(x)) for x in (0, 1, 12345, (1 << 32) - 1, (1 << 42) - 1))


@pytest.mark.parametrize("avx2", SEM, ids=SEM_IDS)
@pytest.mark.parametrize("c,k,mc", [(125, 15, 1000), (10, 13, 40), (1, 16, 1), (30, 16, 200)])
def test_parity_set(avx2, c, k, mc):
    contigs = parity_set(np.random.default_rng(1234 + c), 30)
    check_genomes([contigs[0:7], contigs[7:8], contigs[8:30]], c, k, mc, avx2)


@pytest.mark.parametrize("avx2", SEM, ids=SEM_IDS)
def test_pack_case(avx2):
    genomes, starts, lens = SC.pack_case()
    assert {(int(a) % 4, int(n) % 32) for a, n in zip(starts, lens)} >= {(a, r) for a in range(4) for r in range(32)}
    for r in check_genomes(genomes, 1, 15, 1, avx2):
        assert len(r["kmer"]) > 0


@pytest.mark.parametrize("avx2", SEM, ids=SEM_IDS)
def test_window_case(avx2):
    genomes, lens = SC.window_case()
    for g, r in zip(genomes, check_genomes(genomes, 1, 15, 1000, avx2)):
        assert np.array_equal(r["ctg_rec_off"][1:] - r["ctg_rec_off"][:-1], [R.n_windows(len(s), avx2) for s in g])


@pytest.mark.parametrize("avx2", SEM, ids=SEM_IDS)
@pytest.mark.parametrize("byte", [ord("N"), ord("n")], ids=["N", "n"])
def test_n_case(avx2, byte):
    genomes, where = SC.n_case(byte)
    check_genomes(genomes, 1, 15, 1000, avx2)
    check_genomes(genomes, 125, 13, 1000, avx2)


@pytest.mark.parametrize("total", SC.LOOKUP_TOTALS)
def test_lookup_case(total):
    genomes, _ = SC.lookup_case(total)
    check_genomes(genomes, 1, 15, 1, True)
    check_genomes(genomes, 1, 15, 1, False)


@pytest.mark.parametrize("k", [6, 8, 10])
def test_tie_case(k):
    genomes, ends = SC.tie_case(k)
    for avx2 in SEM:
        check_genomes(genomes, 1, k, 1, avx2)
    _, _, fs, rs = R.windows(genomes[0][0], k)
    assert np.all(fs[0, ends - 20] == rs[0, ends - 20])


def test_no_tie_at_k_11_and_above():
    """for k >= 11 the forward and the reverse-complemented k-mer of a window overlap so that one base would have to equal
    its own complement: no 21-base window has Fs == Rs (checked over every window of 2 Mbp with the ties of k = 10 planted)"""
    genomes, _ = SC.tie_case(10)
    s = np.concatenate([genomes[0][0]] + [SC.rand_acgt(np.random.default_rng(3), 2_000_000)])
    for k in range(11, 17):
        _, _, fs, rs = R.windows(s, k)
        assert not np.any(fs == rs), k


def test_mult_case():
    genomes = SC.mult_case()
    r, = check_genomes(genomes, 1, 15, 1000, True)
    assert r["pv_mult"].max() == R.MULT_MAX and np.count_nonzero(r["pv_mult"] == R.MULT_MAX) > R.MULT_MAX


@pytest.mark.parametrize("extra", [0, 4])
def test_kview_case(extra):
    genomes = SC.kview_case(extra)
    rs = check_genomes(genomes[:1] + genomes[1:41], 1, 16, 1000, True)
    assert len(rs[0]["kmer"]) == (1 << 21) + extra
    assert SC.kview_bits(len(rs[0]["kmer"]), 16, SC.KVIEW_G) == 64 + (extra > 0)


def test_marker_rows_equal_oracle():
    rows = SC.marker_rows(SC.MARKER_G)
    assert SC.marker_bits(SC.MARKER_G) == 64 and SC.marker_bits(SC.MARKER_G + 1) == 65
    idx = np.random.default_rng(5).choice(len(rows), 600, replace=False)
    mk, off = R.markers_rows(rows[idx], 15, 8, 8, chunk=128)
    for i, g in enumerate(idx):
        e = oracle_contig(rows[g], 8, 15, 8, True)
        assert np.array_equal(mk[int(off[i]):int(off[i + 1])], e["markers"]), g
    assert (off[1:] > off[:-1]).mean() > 0.9


def test_marker_gate_case():
    genomes = SC.marker_gate_case()
    a = check_genomes(genomes, 30, 15, 30, True)
    b = check_genomes(genomes, 30, 15, 2 ** 32 - 1, True)
    for s in (c for g in genomes for c in g):                            # marker_c == c: every record inserts its marker
        pos, _, _, mk = R.contig_seeds(s, 15, 30, 30)
        assert len(mk) == len(pos) > 0
    assert all(len(x["markers"]) == 0 for x in b)
    raw = sum(len(R.contig_seeds(s, 15, 30, 30)[3]) for s in genomes[0])
    assert raw > len(a[0]["markers"])                                    # the repeated contigs' markers are stored once
