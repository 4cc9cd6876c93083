"""Plain numpy reference of FracMinHash seeding and of a genome's sketch layout, restated from the reference's Rust source
(avx2_fmh_seeds, src/avx2_seeding.rs:33-272; fmh_seeds, src/seeding.rs:225-323; BYTE_TO_SEQ and Sketch::add_seed_position,
src/types.rs:40-49,281-304).  TEST INFRASTRUCTURE ONLY.

Both seeders slide a 21-base window (the marker k) over a contig and look at the window ending at base e:
  F21 = the window's 2-bit codes, base e in the low bits; R21 = its reverse complement, complement of base e - 20 in the
  low bits.  Fs / Rs = their low 2k bits (the last k bases forward, the first k bases reverse-complemented).
  canonical = Fs < Rs, and the seed is Fs if canonical else Rs (a tie takes Rs with canonical 0).
  A record (seed, pos = e, contig << 1 | canonical) is kept when mm_hash64(seed) < u64::MAX / c and the window is not
  broken by an N; its marker min(F21, R21) is kept when mm_hash64(seed) < u64::MAX / marker_c.
  Contigs shorter than 42 bases give nothing.
4-lane AVX2 seeder: q = (n - 20) / 4; lane l reads bases [l q, l q + q + 20) and visits the window ends l q + 20 ..
  l q + q + 19, so the last (n - 20) mod 4 windows are never visited.  Only byte 78 ('N') is an N.  The 20-base prefill of a
  lane never tests for N; an N at a visited window end p sets resume = p + 21, so a window e of lane l is dropped iff an N
  lies in [max(e - 20, l q + 20), e].  An N in lane l's prefill is seen only by lane l - 1's last windows.
Scalar seeder: every window end 20 .. n - 1; 'N' and 'n' at p >= 20 set resume = p + k, so window e is dropped iff one lies
  in [max(e - k + 1, 20), e].

A genome's layout: the position view (records in contig, pos order), the k-mer view (records stably sorted by k-mer: kmer,
contig, pos order), the distinct k-mers with each group's start (one sentinel = the record count per genome),
pv_mult = min(group size, 65535) per record in position-view order, ctg_rec_off (each contig's first record, plus the
sentinel) and the sorted distinct markers (the reference's HashSet)."""
import numpy as np

MARKER_K = 21
U64 = np.uint64
U64_MAX = 2 ** 64 - 1
ASCII_N, ASCII_N_SMALL = 78, 110
MULT_MAX = 65535                  # pv_mult is a u16

# src/types.rs:40-49, row by row: rows 0, 2 and 3 of the 32-byte rows hold non-zero codes
BYTE_TO_SEQ = np.zeros(256, np.uint64)
BYTE_TO_SEQ[0:4] = [0, 1, 2, 3]
for _row in (64, 96):             # ..C...G............TU.. in upper and lower case
    BYTE_TO_SEQ[_row + 3], BYTE_TO_SEQ[_row + 7], BYTE_TO_SEQ[_row + 20], BYTE_TO_SEQ[_row + 21] = 1, 2, 3, 3


def mm_hash64(x):
    """src/types.rs:86-96, wrapping u64 arithmetic"""
    with np.errstate(over="ignore"):
        x = np.asarray(x, np.uint64)
        x = ~(x + (x << U64(21)))
        x = x ^ (x >> U64(24))
        x = (x + (x << U64(3))) + (x << U64(8))
        x = x ^ (x >> U64(14))
        x = (x + (x << U64(2))) + (x << U64(4))
        x = x ^ (x >> U64(28))
        return x + (x << U64(31))


def threshold(c):
    return U64(U64_MAX // c)


def is_seed(keys, c):
    return mm_hash64(keys) < threshold(c)


def is_n(seqs, avx2=True):
    """the bytes that break windows: 'N' under the AVX2 semantics, 'N' and 'n' under the scalar ones"""
    s = np.asarray(seqs, np.uint8)
    return (s == ASCII_N) if avx2 else (s == ASCII_N) | (s == ASCII_N_SMALL)


def windows(seqs, k):
    """rows (R, n) of bytes -> (F21, R21, Fs, Rs), each (R, max(n - 20, 0)) uint64; column j is window end 20 + j"""
    s = np.atleast_2d(np.asarray(seqs, np.uint8))
    code = BYTE_TO_SEQ[s]
    n = s.shape[1]
    W = max(n - (MARKER_K - 1), 0)
    f21 = np.zeros((len(s), W), np.uint64)
    r21 = np.zeros((len(s), W), np.uint64)
    for j in range(MARKER_K):
        f21 |= code[:, MARKER_K - 1 - j:MARKER_K - 1 - j + W] << U64(2 * j)      # base e - j at bits 2j
        r21 |= (U64(3) - code[:, j:j + W]) << U64(2 * j)                           # complement of base e - 20 + j at bits 2j
    mask = U64((1 << (2 * k)) - 1)
    return f21, r21, f21 & mask, r21 & mask


def n_windows(n, avx2=True):
    """number of windows the seeder visits in a contig of n bases (the record count at c = 1 without N)"""
    if n < 2 * MARKER_K:
        return 0
    return 4 * ((n - 20) // 4) if avx2 else n - 20


def seed_rows(seqs, k, c, marker_c, avx2=True):
    """The seeder over R contigs of one length n (the rows of `seqs`).  Returns a dict of (R, max(n - 20, 0)) arrays over
    the window ends e = 20 + column: keep (a record), kmer (uint32 seed), canon, marker (uint64 min(F21, R21)) and mkeep
    (the marker is inserted)."""
    s = np.atleast_2d(np.asarray(seqs, np.uint8))
    R, n = s.shape
    f21, r21, fs, rs = windows(s, k)
    W = f21.shape[1]
    canon = fs < rs
    seed = np.where(canon, fs, rs)
    h = mm_hash64(seed)
    e = np.arange(MARKER_K - 1, MARKER_K - 1 + W)
    ncum = np.zeros((R, n + 1), np.int64)
    np.cumsum(is_n(s, avx2), axis=1, out=ncum[:, 1:])
    if n < 2 * MARKER_K:
        visited = np.zeros(W, bool)
        lo = e
    elif avx2:
        q = (n - 20) // 4
        visited = e < 4 * q + 20
        lane = np.minimum((e - 20) // q, 3)
        lo = np.maximum(e - 20, lane * q + 20)           # resume = p + 21, and lane l tests for N from its base l q + 20 on
    else:
        visited = np.ones(W, bool)
        lo = np.maximum(e - k + 1, 20)                    # resume = p + k, tested from base 20 on
    broken = ncum[:, e + 1] - ncum[:, lo] > 0
    keep = (h < threshold(c)) & visited & ~broken
    return dict(keep=keep, kmer=seed.astype(np.uint32), canon=canon, marker=np.minimum(f21, r21),
                mkeep=keep & (h < threshold(marker_c)))


def contig_seeds(seq, k, c, marker_c=None, avx2=True):
    """(pos, kmer, canonical, markers) of one contig's records, in position order; markers as inserted (with repeats)"""
    r = seed_rows(np.asarray(seq, np.uint8)[None], k, c, marker_c or c, avx2)
    j = np.nonzero(r["keep"][0])[0]
    return (j + MARKER_K - 1).astype(np.uint32), r["kmer"][0, j], r["canon"][0, j], r["marker"][0][r["mkeep"][0]]


def layout(kmer, pos, cc, markers, contig_lengths):
    """a genome's arrays from its records in position-view order (contig, pos)"""
    kmer, pos, cc = (np.asarray(x, np.uint32) for x in (kmer, pos, cc))
    order = np.argsort(kmer, kind="stable")                  # k-mer view: (kmer, contig, pos)
    uk, first, cnt = np.unique(kmer[order], return_index=True, return_counts=True)
    mult = np.minimum(cnt[np.searchsorted(uk, kmer)], MULT_MAX).astype(np.uint16)
    nc = len(contig_lengths)
    ctg_rec_off = np.searchsorted(cc >> np.uint32(1), np.arange(nc + 1)).astype(np.uint32)
    return dict(kmer=kmer[order], pos=pos[order], cc=cc[order], markers=np.unique(np.asarray(markers, np.uint64)),
                contig_lengths=np.asarray(contig_lengths, np.uint32), pv_kmer=kmer, pv_pos=pos, pv_cc=cc, pv_mult=mult,
                ukmer=uk.astype(np.uint32), ustart=np.append(first, len(kmer)).astype(np.uint32), ctg_rec_off=ctg_rec_off)


def sketch(contigs, k, c, marker_c, avx2=True):
    """One genome (a list of contigs, in order) as the sketch set stores it: export()'s kmer / pos / cc (k-mer view),
    markers and contig_lengths, plus the position view pv_*, pv_mult, ukmer, ustart and ctg_rec_off.  Contigs of one length
    are seeded together."""
    seqs = [np.asarray(s, np.uint8) for s in contigs]
    lens = np.array([len(s) for s in seqs], np.int64)
    per = [None] * len(seqs)
    for n in np.unique(lens):
        idx = np.nonzero(lens == n)[0]
        r = seed_rows(np.stack([seqs[i] for i in idx]) if n else np.zeros((len(idx), 0), np.uint8), k, c, marker_c, avx2)
        for row, ci in enumerate(idx):
            j = np.nonzero(r["keep"][row])[0]
            cc = (np.uint32(ci) << np.uint32(1)) | r["canon"][row, j].astype(np.uint32)
            per[ci] = ((j + MARKER_K - 1).astype(np.uint32), r["kmer"][row, j], cc, r["marker"][row][r["mkeep"][row]])
    cat = lambda i, dt: np.concatenate([p[i] for p in per]).astype(dt) if per else np.zeros(0, dt)      # noqa: E731
    return layout(cat(1, np.uint32), cat(0, np.uint32), cat(2, np.uint32), cat(3, np.uint64), lens)


def markers_rows(seqs, k, c, marker_c, avx2=True, chunk=1 << 18):
    """Sorted distinct markers of many one-contig genomes of one length (the rows of `seqs`): (markers, offsets)."""
    s = np.atleast_2d(np.asarray(seqs, np.uint8))
    out, counts = [], []
    for a in range(0, len(s), chunk):
        r = seed_rows(s[a:a + chunk], k, c, marker_c, avx2)
        m = np.where(r["mkeep"], r["marker"], U64(U64_MAX))
        m.sort(axis=1)
        first = np.ones(m.shape, bool)
        first[:, 1:] = m[:, 1:] != m[:, :-1]
        first &= m != U64(U64_MAX)                           # markers are < 2^42
        out.append(m[first])
        counts.append(first.sum(1))
    counts = np.concatenate(counts) if counts else np.zeros(0, np.int64)
    return (np.concatenate(out) if out else np.zeros(0, np.uint64)), np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
