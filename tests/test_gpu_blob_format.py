"""GPU: the sketch-set blob format, pinned byte for byte.

A blob (sk_sketch_set_pack_subset) holds twelve arrays, each 256-byte aligned, in the order pv_kmer pv_pos pv_cc pv_mult
kv_pos kv_cc ukmer ustart markers ctg_rec_off d_ctg_len htab; its metadata vector is the header G S U M C c k marker_c HT
flags, then seed_off uk_off mk_off ctg_off [G+1 each], total_len [G], the contig lengths and, with tables, ht_off [G+1].
Every word of every metadata vector and every byte of every blob (padding included) is derived here from info() / export()
alone, for flags 0, SK_PACK_MARKERS_ONLY and SK_PACK_TABLES and genome lists of every shape, over a set holding a genome
without contigs, one with fewer than 20 markers, one of >= 2^20 records (no k-mer table) and one with many contigs.  The
legacy whole-set pack, an unpack of two halves and a host store round trip must reproduce the same bytes."""
import ctypes as C

import numpy as np
import pytest

from bench_support import synth
from chain_testlib import rand_seq

pytestmark = pytest.mark.gpu

MO, TABLES = 1, 2
KW = dict(c=10, k=15, marker_c=200)
BIG, SMALL, EMPTY, MANY = 6, 7, 8, 9
LISTS = {
    "all": None,
    "two_runs": [2, 3, 4, 6, 7, 8, 9],
    "ten_runs": [15, 0, 2, 4, 6, 7, 9, 11, 13, 8, 1],
    "empty": [],
    "duplicates": [9, 9, 6, 1, 1, 2, 8, 8, 8],
}
DT = [np.uint32] * 3 + [np.uint16] + [np.uint32] * 3 + [np.uint32, np.uint64, np.uint32, np.uint32, np.uint64]


def layout(G, S, U, M, C, HT):
    """(offsets, byte sizes, total) of a blob: the format's arithmetic, written out"""
    n = [S * 4, S * 4, S * 4, S * 2, S * 4, S * 4, U * 4, (U + G) * 4, M * 8, (C + G) * 4, C * 4, HT * 8]
    off, o = [], 0
    for b in n:
        off.append(o)
        o += (b + 255) & ~255
    return off, n, (o if o else 256)


def table_cap(nuk, nrec):
    if nuk == 0 or nrec >= 1 << 20:
        return 0
    cap = 16
    while cap < 2 * nuk:
        cap <<= 1
    return cap


def expected_genome(s, g):
    """every array slice of genome g, from export()"""
    info, e = s.info(g), s.export(g)
    kmer, pos, cc = e["kmer"], e["pos"], e["cc"]
    uk, first, cnt = np.unique(kmer, return_index=True, return_counts=True)
    order = np.lexsort((pos, cc >> 1))                         # position view: (contig, pos)
    mult = np.minimum(cnt[np.searchsorted(uk, kmer)], 0xFFFF).astype(np.uint16)
    nc = info["n_contigs"]
    cap = table_cap(len(uk), len(kmer))
    ent = (uk.astype(np.uint64) << np.uint64(32)) | (first.astype(np.uint64) << np.uint64(12)) | np.minimum(cnt, 4095).astype(np.uint64)
    return dict(info=info, pv=[kmer[order], pos[order], cc[order], mult[order]], kv=[pos, cc], ukmer=uk.astype(np.uint32),
                ustart=np.append(first, len(kmer)).astype(np.uint32), markers=e["markers"], ctg_len=e["contig_lengths"],
                ctg_rec_off=np.searchsorted(cc[order] >> 1, np.arange(nc + 1)).astype(np.uint32), cap=cap,
                htab=np.sort(ent) if cap else np.zeros(0, np.uint64))      # >= 2^20 records: no table


@pytest.fixture(scope="module")
def env():
    import skani_b200 as sk
    ctx = sk.Context(0)
    sp = sk.sketch_params(**KW)
    bases, off, goc = synth.generate(0, 12, 200_000, G=4)        # members 2, 6, 10 have 50 contigs
    gen = [[bases[int(off[i]):int(off[i + 1])] for i in np.nonzero(goc == g)[0]] for g in range(12)]
    rng = np.random.default_rng(7)
    many = rand_seq(rng, 400_000)
    genomes = gen[:6] + [[rand_seq(rng, 12_000_000)], [gen[0][0][:2_000]], [], [many[i:i + 1000] for i in range(0, len(many), 1000)]] + gen[6:]
    contigs = [c for g in genomes for c in g]
    o = np.concatenate([[0], np.cumsum([len(c) for c in contigs])]).astype(np.uint64)
    gc = np.concatenate([np.full(len(g), i, np.uint32) for i, g in enumerate(genomes)])
    full = sk.sketch_contigs(ctx, np.concatenate(contigs), o, gc, len(genomes), sp)
    assert full.info(BIG)["n_records"] >= 1 << 20 and full.info(SMALL)["n_markers"] < 20
    assert full.info(EMPTY)["n_contigs"] == 0 and full.info(MANY)["n_contigs"] == 400
    want = [expected_genome(full, g) for g in range(len(full))]
    assert want[BIG]["cap"] == 0 and all(want[g]["cap"] > 0 for g in range(len(full)) if g not in (BIG, EMPTY))
    yield sk, ctx, sp, full, want
    full.free()
    ctx.close()


def pack(s, genomes, flags):
    """(zero-filled device blob, metadata) of pack_subset"""
    import torch
    nb, nw = s.subset_blob_size(genomes, flags)
    t = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    meta = s.pack_subset(genomes, flags, t.data_ptr(), nw)
    assert len(meta) == nw
    return t, meta


def unpack(ctx, parts):
    import skani_b200 as sk
    n = len(parts)
    bp = (C.c_void_p * n)(*[t.data_ptr() for t, _ in parts])
    mp_ = (C.c_void_p * n)(*[m.ctypes.data for _, m in parts])
    h = C.c_void_p()
    ctx.check(ctx.L.sk_sketch_set_unpack(ctx.h, n, bp, mp_, C.byref(h)))
    return sk.SketchSet(ctx, h)


def check_blob(sp, want, sel, flags, blob, meta):
    mo, tables = flags == MO, flags == TABLES
    G = len(sel)
    w = [want[g] for g in sel]
    cnt = lambda key, on: np.array([x["info"][key] if on else 0 for x in w], np.uint64)
    per = [cnt("n_records", not mo), cnt("n_kmers", not mo), cnt("n_markers", True), cnt("n_contigs", not mo),
           np.array([x["cap"] if tables else 0 for x in w], np.uint64)]
    offs = [np.concatenate([[0], np.cumsum(p)]).astype(np.uint64) for p in per]
    S, U, M, Cn, HT = (int(o[-1]) for o in offs)
    words = [G, S, U, M, Cn, sp.c, sp.k, sp.marker_c, HT, int(tables)] + [v for o in offs[:4] for v in o.tolist()]
    words += [x["info"]["total_len"] for x in w]
    if not mo:
        words += [int(v) for x in w for v in x["ctg_len"]]
    if tables:
        words += offs[4].tolist()
    assert meta.tolist() == words
    off, nbytes, total = layout(G, S, U, M, Cn, HT)
    raw = blob.cpu().numpy()
    assert len(raw) == total
    arr = [raw[off[a]:off[a] + nbytes[a]].view(DT[a]) for a in range(12)]
    for a in range(12):                                       # nothing written outside the arrays
        end = off[a + 1] if a < 11 else total
        assert not raw[off[a] + nbytes[a]:end].any(), a
    so, uo, mko, co, ho = offs
    for i, x in enumerate(w):
        if not mo:
            r = slice(int(so[i]), int(so[i + 1]))
            for a in range(4):
                assert np.array_equal(arr[a][r], x["pv"][a]), (sel[i], a)
            assert np.array_equal(arr[4][r], x["kv"][0]) and np.array_equal(arr[5][r], x["kv"][1]), sel[i]
            assert np.array_equal(arr[6][int(uo[i]):int(uo[i + 1])], x["ukmer"]), sel[i]
            assert np.array_equal(arr[7][int(uo[i]) + i:int(uo[i + 1]) + i + 1], x["ustart"]), sel[i]
            assert np.array_equal(arr[9][int(co[i]) + i:int(co[i + 1]) + i + 1], x["ctg_rec_off"]), sel[i]
            assert np.array_equal(arr[10][int(co[i]):int(co[i + 1])], x["ctg_len"]), sel[i]
        assert np.array_equal(arr[8][int(mko[i]):int(mko[i + 1])], x["markers"]), sel[i]
        if tables:
            t = arr[11][int(ho[i]):int(ho[i + 1])]
            assert np.array_equal(np.sort(t[t != 0]), x["htab"]) and (t == 0).sum() == x["cap"] - len(x["htab"]), sel[i]
            if x["cap"]:
                assert np.array_equal(np.unique(t[t != 0] >> np.uint64(32)).astype(np.uint32), x["ukmer"]), sel[i]
    if mo:                                                    # one zero sentinel per genome
        assert len(arr[7]) == len(arr[9]) == G and not arr[7].any() and not arr[9].any()


@pytest.mark.parametrize("flags", [0, MO, TABLES], ids=["plain", "markers_only", "tables"])
@pytest.mark.parametrize("which", sorted(LISTS))
def test_pack_subset_format(env, which, flags):
    sk, ctx, sp, full, want = env
    genomes = LISTS[which]
    sel = list(range(len(full))) if genomes is None else genomes
    blob, meta = pack(full, genomes, flags)
    check_blob(sp, want, sel, flags, blob, meta)


def test_whole_set_pack_equals_subset_pack(env):
    import torch
    sk, ctx, sp, full, want = env
    L = ctx.L
    nb, nw = C.c_uint64(), C.c_uint64()
    ctx.check(L.sk_sketch_set_blob_size(full.h, C.byref(nb), C.byref(nw)))
    assert (nb.value, nw.value) == full.subset_blob_size(None, 0)
    t = torch.zeros(nb.value, dtype=torch.uint8, device="cuda")
    meta = np.zeros(nw.value, np.uint64)
    ctx.check(L.sk_sketch_set_pack(full.h, C.c_void_p(t.data_ptr()), meta.ctypes.data))
    sb, sm = pack(full, None, 0)
    assert np.array_equal(meta, sm) and torch.equal(t, sb)
    check_blob(sp, want, list(range(len(full))), 0, t, meta)


def test_two_halves_repack_equals_whole(env):
    import torch
    sk, ctx, sp, full, want = env
    n = len(full)
    halves = unpack(ctx, [pack(full, list(range(0, 7)), 0), pack(full, list(range(7, n)), 0)])
    for flags in (0, MO):
        a, am = pack(halves, None, flags)
        b, bm = pack(full, None, flags)
        assert np.array_equal(am, bm) and torch.equal(a, b), flags
    halves.free()


def test_store_round_trip_bytes(env):
    import torch
    sk, ctx, sp, full, want = env
    n = len(full)
    nobig = unpack(ctx, [pack(full, [g for g in range(n) if g != BIG], TABLES)])     # every genome with a table
    for src, exact in ((nobig, True), (full, False)):
        st = sk.SketchStore(sp)
        st.add(src)
        for g in range(len(src)):
            i = src.info(g)
            cap = table_cap(i["n_kmers"], i["n_records"])
            assert st.genome_bytes(g) == 22 * i["n_records"] + 8 * (i["n_kmers"] + i["n_markers"] + i["n_contigs"] + cap) + 8
        got = st.gather(ctx)
        a, am = pack(got, None, TABLES)
        b, bm = pack(src, None, TABLES)
        assert np.array_equal(am, bm)
        if exact:
            assert torch.equal(a, b)
        else:       # the unpack rebuilds every table (atomicCAS slot order inside a bucket is not fixed): all but htab
            off = layout(*[int(v) for v in bm[:5]], int(bm[8]))[0]
            assert torch.equal(a[:off[11]], b[:off[11]])
        got.free()
        st.free()
    nobig.free()
