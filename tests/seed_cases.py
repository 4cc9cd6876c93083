"""Constructed seeding inputs, one builder per edge of pack_kernel, hashpass_kernel, expand_kernel and build_views.  Each
builder returns genomes (lists of contigs, uint8 ASCII) and the facts its reach assertions need.  test_seed_ref.py checks
seed_ref against the oracle on them; test_gpu_seed_edges.py checks the GPU against seed_ref.  TEST INFRASTRUCTURE ONLY."""
import numpy as np

import seed_ref as R

ACGT = np.frombuffer(b"ACGT", np.uint8)
COMP = np.zeros(256, np.uint8)
COMP[ACGT] = np.frombuffer(b"TGCA", np.uint8)
FAST = np.frombuffer(b"ACGTUacgtu", np.uint8)          # the bytes of pack_word's letter fast path


def rand_acgt(rng, n):
    return rng.choice(ACGT, n).astype(np.uint8)


def flat(genomes):
    """(bases, contig_off, genome_of_contig) of genomes laid out back to back"""
    contigs = [c for g in genomes for c in g]
    off = np.concatenate([[0], np.cumsum([len(c) for c in contigs])]).astype(np.uint64)
    goc = np.concatenate([np.full(len(g), i, np.uint32) for i, g in enumerate(genomes)] + [np.zeros(0, np.uint32)])
    bases = np.concatenate(contigs) if contigs else np.zeros(0, np.uint8)
    return bases, off, goc


# ---- a. pack realignment -----------------------------------------------------------------------------------------------
def all_bytes_contig(rng):
    """every byte value 0..255 at a position of each residue mod 4 (one odd byte per 24 bases, inside A/C/G/T)"""
    s = rand_acgt(rng, 24 * 1024 + 64)
    for b in range(256):
        for j in range(4):
            s[24 * (4 * b + j) + 32 + j] = b
    return s


def pack_case(seed=11):
    """Contigs starting at every byte offset mod 4 crossed with every length mod 32, plus the all-bytes contig at every
    start offset mod 4.  Contigs carry 'N', 'n', lower case and IUPAC codes.  Returns (genomes, starts, lengths)."""
    rng = np.random.default_rng(seed)
    contigs, start = [], 0

    def add(s):
        nonlocal start
        contigs.append(s)
        start += len(s)

    def align(a):
        if start % 4 != a:
            add(rand_acgt(rng, 44 + (a - start) % 4))

    odd = np.frombuffer(b"NnacgtRYKM-*", np.uint8)
    for r in range(32):
        for a in range(4):
            align(a)
            s = rand_acgt(rng, 64 + r + 32 * ((r + a) % 3))
            s[rng.integers(0, len(s), 3)] = rng.choice(odd, 3)
            add(s)
    for a in range(4):
        align(a)
        add(all_bytes_contig(rng))
    lens = np.array([len(c) for c in contigs])
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    genomes = [contigs[i:i + 40] for i in range(0, len(contigs), 40)]
    return genomes, starts, lens


def pack_word_paths(s):
    """(words on pack_word's letter fast path, words on its per-byte path) of a contig: 4-byte words from its first base"""
    w = np.asarray(s[:len(s) // 4 * 4], np.uint8).reshape(-1, 4)
    fast = np.isin(w, FAST).all(1)
    return int(fast.sum()), int((~fast).sum())


# ---- b. window existence -----------------------------------------------------------------------------------------------
def window_case(seed=12):
    """Lengths 41..48, and lengths whose last visited window end + 1 (4q + 20) lies 4 before, on or 4 after a 32-base unit
    boundary, with every (n - 20) mod 4 tail.  Returns (genomes, lengths)."""
    rng = np.random.default_rng(seed)
    lens = list(range(41, 49))
    for m in (2, 3, 4, 7, 32):
        for d in (-4, 0, 4):
            lens += [32 * m + d + t for t in range(4)]
    contigs = [rand_acgt(rng, n) for n in lens]
    return [contigs[:20], contigs[20:]], np.array(lens)


# ---- c. N placement ----------------------------------------------------------------------------------------------------
def n_positions(n):
    """the N positions of case c for a contig of n bases, with their names"""
    q = (n - 20) // 4
    out = []
    for l in range(4):
        out += [("l%d_q+19" % l, l * q + 19), ("l%d_q+20" % l, l * q + 20), ("l%d_q+40" % l, l * q + 40), ("l%d_q+41" % l, l * q + 41)]
    out += [("4q+19", 4 * q + 19), ("4q+20", 4 * q + 20)]
    out += [("32m-1", 32 * m - 1) for m in (1, 2, n // 64)] + [("32m", 32 * m) for m in (1, 2, n // 64)]
    return [(name, p) for name, p in out if 0 <= p < n]


def n_case(byte, seed=13):
    """One contig per (length, N position) with a single `byte` there; then a contig ending in `byte` followed by a clean
    one, twice (the break must not leak into the next contig).  Returns (genomes, [(contig index, n, name, p)])."""
    rng = np.random.default_rng(seed)
    contigs, where = [], []
    for n in (203, 1046, 1000 + 32 * 7 + 3):
        clean = rand_acgt(rng, n)
        for name, p in n_positions(n):
            s = clean.copy()
            s[p] = byte
            where.append((len(contigs), n, name, p))
            contigs.append(s)
    for n in (96, 130):                     # the broken contig ends a unit exactly (96) and inside one (130)
        s = rand_acgt(rng, n)
        s[-1] = byte
        where.append((len(contigs), n, "last", n - 1))
        contigs += [s, rand_acgt(rng, 100)]
    return [contigs[:30], contigs[30:]], where


# ---- d. contig lookup --------------------------------------------------------------------------------------------------
LOOKUP_TOTALS = (4095, 4096, 4097)       # unit totals just below, at and above a multiple of 256


def lookup_case(total_units, seed=14):
    """Contigs of 0..64 bases (0..2 units each) with zero-length contigs among them, filling exactly `total_units` units;
    a zero-length contig and a real one start at some units 256 m.  Returns (genomes, unit offsets of the contigs)."""
    rng = np.random.default_rng(seed + total_units)
    contigs, units, cuoff = [], 0, []
    while units < total_units:
        if units % 256 == 0 and units and rng.random() < 0.7:
            cuoff.append(units)
            contigs.append(np.zeros(0, np.uint8))
        n = int(rng.integers(0, 65))
        u = (n + 31) // 32
        if units + u > total_units:
            n, u = 32, 1
        cuoff.append(units)
        contigs.append(rand_acgt(rng, n))
        units += u
    cut = np.linspace(0, len(contigs), 6).astype(int)
    return [contigs[a:b] for a, b in zip(cut[:-1], cut[1:])], np.array(cuoff)


# ---- e. canonical ties -------------------------------------------------------------------------------------------------
def plant_tie(s, e, k):
    """make window e's forward k-mer (bases e-k+1..e) the reverse complement of its first k bases (e-20..e-21+k): Fs == Rs.
    Possible only for k <= 10: for k >= 11 the two k-mers overlap and base e-k+1+i (i = k - 11) would have to be its own
    complement."""
    assert k <= 10
    for i in range(k):
        s[e - k + 1 + i] = COMP[s[e - 20 + k - 1 - i]]


def tie_case(k, seed=15):
    """a contig with ties planted at every 40th window end (and one at the first and last visited ends).  Returns
    (genomes, planted window ends)."""
    rng = np.random.default_rng(seed + k)
    n = 4020
    s = rand_acgt(rng, n)
    ends = [20] + list(range(61, 4000, 40)) + [4019]
    for e in ends:
        plant_tie(s, e, k)
    return [[s, rand_acgt(rng, 500)]], np.array(ends)


# ---- f. multiplicity ---------------------------------------------------------------------------------------------------
def mult_case(seed=16):
    """a 70 kbp poly-A contig (k-mer 0 in every window) and a random contig"""
    rng = np.random.default_rng(seed)
    return [[rand_acgt(rng, 3000), np.full(70_000, ord("A"), np.uint8), rand_acgt(rng, 5000)]]


# ---- g. sort-width switches --------------------------------------------------------------------------------------------
KVIEW_G = 1025
MARKER_G = 1 << 22


def kview_case(extra, seed=17):
    """KVIEW_G genomes; genome 0 is one contig of 2^21 + extra + 20 bases (2^21 + extra records at c = 1, extra % 4 == 0),
    the others 42..300 bases."""
    rng = np.random.default_rng(seed)
    small = [[rand_acgt(rng, int(n))] for n in rng.integers(42, 301, KVIEW_G - 1)]     # the same for every `extra`
    big = rand_acgt(rng, (1 << 21) + extra + 20)
    return [[big]] + small


def kview_bits(max_rec, k, G):
    """build_views' rule: the record index rides in the sort key (keys-only sort) iff index, k-mer and genome bits fit 64"""
    ibits = (max_rec - 1).bit_length() if max_rec > 1 else 1
    gbits = (G - 1).bit_length() if G > 1 else 0
    return ibits + 2 * k + gbits


def marker_bits(G):
    """build_views' rule: one global marker sort of (genome << 42 | marker) iff that fits 64 bits, else per-genome segments"""
    return 2 * R.MARKER_K + ((G - 1).bit_length() if G > 1 else 0)


def marker_rows(G, seed=18):
    """G one-contig genomes of 42 bases (20 visited windows each)"""
    return np.random.default_rng(seed).choice(ACGT, (G, 42)).astype(np.uint8)


# ---- h. marker gating --------------------------------------------------------------------------------------------------
def marker_gate_case(seed=19):
    """genome 0: one contig three times over (the same markers from several contigs); genome 1: random contigs"""
    rng = np.random.default_rng(seed)
    s = rand_acgt(rng, 3000)
    return [[s, rand_acgt(rng, 800), s.copy(), s.copy()], [rand_acgt(rng, n) for n in (900, 2000, 4100)]]
