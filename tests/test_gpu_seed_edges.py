"""GPU: seeding (pack_kernel or the host packer, hashpass_kernel, expand_kernel, build_views) against seed_ref, bit for bit,
at the edges where the kernels can go wrong.  Records (kmer, pos, cc), markers and contig lengths come from export(); the
position view, pv_mult, the k-mer view, ukmer / ustart and ctg_rec_off come from a pack_subset blob (layout pinned by
test_gpu_blob_format.py).  At c = 1 every visited window is a record, so record counts are exact.  Every case asserts from its
own data that it reached its edge:
  a  pack realignment: every contig start mod 4 x every length mod 32, all 256 byte values at every position of a word,
     through the device packer, the host packer and a device buffer at byte offsets 0..3
  b  window existence: lengths 41..48, the last visited window just before, on and after a unit boundary
  c  'N' / 'n' placement under both semantics: lane prefills, lane starts, the dropped tail, unit edges, a broken contig end
  d  contig lookup: thousands of 0..64-base contigs, zero-length ones, contigs starting at unit 256 m, 4095 / 4096 / 4097 units
  e  canonical ties (Fs == Rs: the seed is Rs with canonical bit 0), planted at k = 6, 8, 10
  f  a k-mer seen more than 65 535 times: pv_mult saturates, the table count at 4 095
  g  sort-width switches: the k-mer view's keys-only / pairs sort, the markers' global / segmented sort
  h  marker gating: marker_c == c, a marker_c that admits no marker, one marker from several contigs"""
import numpy as np
import pytest

import ktable_ref as T
import seed_cases as SC
import seed_ref as R

pytestmark = pytest.mark.gpu

MO, TABLES = 1, 2
ARRAYS = ("pv_kmer", "pv_pos", "pv_cc", "pv_mult", "kv_pos", "kv_cc", "ukmer", "ustart", "markers", "ctg_rec_off", "ctg_len", "htab")
DT = [np.uint32] * 3 + [np.uint16] + [np.uint32] * 4 + [np.uint64, np.uint32, np.uint32, np.uint64]
SEM = [True, False]
SEM_IDS = ["avx2", "scalar"]
PATHS = ["host_pack0", "host_pack1", "dev0", "dev1", "dev2", "dev3"]


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def blob(s, flags=0):
    """(meta dict, arrays dict) of a pack_subset blob of the whole set"""
    import torch
    nb, nw = s.subset_blob_size(None, flags)
    t = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    meta = s.pack_subset(None, flags, t.data_ptr(), nw).astype(np.int64)
    G, S, U, M, Cn, HT = (int(meta[i]) for i in (0, 1, 2, 3, 4, 8))
    o = 10
    m = {"G": G}
    for name in ("seed_off", "uk_off", "mk_off", "ctg_off"):
        m[name] = meta[o:o + G + 1]
        o += G + 1
    if flags == TABLES:
        m["ht_off"] = meta[len(meta) - G - 1:]
    sizes = [S * 4, S * 4, S * 4, S * 2, S * 4, S * 4, U * 4, (U + G) * 4, M * 8, (Cn + G) * 4, Cn * 4, HT * 8]
    raw = t.cpu().numpy()
    a, off = {}, 0
    for name, dt, b in zip(ARRAYS, DT, sizes):
        a[name] = raw[off:off + b].view(dt)
        off += (b + 255) & ~255
    del t
    return m, a


def sketch(ctx, genomes, c, k, mc, avx2=True, path="host_pack0", monkeypatch=None):
    """sketch the genomes (seeding semantics `avx2`) through one input path"""
    import skani_b200 as sk
    import torch
    bases, off, goc = SC.flat(genomes)
    sp = sk.sketch_params(c, k, mc)
    ctx.set_seeding_semantics(scalar=not avx2)
    try:
        if path.startswith("dev"):
            o = int(path[3:])
            t = torch.zeros(len(bases) + 8, dtype=torch.uint8, device="cuda")
            t[o:o + len(bases)] = torch.from_numpy(bases).cuda()
            assert (t.data_ptr() + o) % 4 == o
            return sk.sketch_contigs(ctx, None, off, goc, len(genomes), sp, device_ptr=t.data_ptr() + o)
        monkeypatch.setenv("SK_HOST_PACK", path[len("host_pack"):])
        try:
            return sk.sketch_contigs(ctx, bases, off, goc, len(genomes), sp)
        finally:
            monkeypatch.delenv("SK_HOST_PACK")
    finally:
        ctx.set_seeding_semantics(scalar=False)


def check_set(s, genomes, c, k, mc, avx2=True, refs=None, export=True, flags=0):
    """every genome of the set equals seed_ref: blob arrays always, export() unless export=False.  Returns (refs, meta, arrays)."""
    refs = refs if refs is not None else [R.sketch(g, k, c, mc, avx2) for g in genomes]
    m, a = blob(s, flags)
    assert m["G"] == len(genomes) == len(refs)
    so, uo, mo, co = (m[x] for x in ("seed_off", "uk_off", "mk_off", "ctg_off"))
    for g, r in enumerate(refs):
        rs, us = slice(so[g], so[g + 1]), slice(uo[g], uo[g + 1])
        got = dict(pv_kmer=a["pv_kmer"][rs], pv_pos=a["pv_pos"][rs], pv_cc=a["pv_cc"][rs], pv_mult=a["pv_mult"][rs],
                   pos=a["kv_pos"][rs], cc=a["kv_cc"][rs], ukmer=a["ukmer"][us], ustart=a["ustart"][uo[g] + g:uo[g + 1] + g + 1],
                   markers=a["markers"][mo[g]:mo[g + 1]], ctg_rec_off=a["ctg_rec_off"][co[g] + g:co[g + 1] + g + 1],
                   contig_lengths=a["ctg_len"][co[g]:co[g + 1]])
        for key, v in got.items():
            assert np.array_equal(v, r[key]), (g, key)
        if export:
            e = s.export(g)
            for key in ("kmer", "pos", "cc", "markers", "contig_lengths"):
                assert np.array_equal(e[key], r[key]), (g, key)
    return refs, m, a


# ---- a -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("avx2", SEM, ids=SEM_IDS)
def test_a_pack_realignment(ctx, monkeypatch, avx2, path):
    genomes, starts, lens = SC.pack_case()
    assert {(int(a) % 4, int(n) % 32) for a, n in zip(starts, lens)} >= {(a, r) for a in range(4) for r in range(32)}
    contigs = [x for g in genomes for x in g]
    allb = [i for i, x in enumerate(contigs) if len(x) == len(SC.all_bytes_contig(np.random.default_rng(0)))]
    assert sorted(int(starts[i]) % 4 for i in allb) == [0, 1, 2, 3]
    for i in allb:
        x = contigs[i]
        for j in range(4):
            assert len(np.unique(x[j::4])) == 256, j           # every byte value at word position j
        fast, slow = SC.pack_word_paths(x)
        assert fast > 0 and slow >= 4 * (256 - len(SC.FAST))      # every odd byte outside the letters takes the per-byte path
    s = sketch(ctx, genomes, 1, 15, 1, avx2, path, monkeypatch)
    refs, _, _ = check_set(s, genomes, 1, 15, 1, avx2)
    assert all(len(r["pv_kmer"]) > 0 for r in refs)
    s.free()


# ---- b -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("avx2", SEM, ids=SEM_IDS)
def test_b_window_existence(ctx, monkeypatch, avx2):
    genomes, lens = SC.window_case()
    ehi = np.array([20 + 4 * ((n - 20) // 4) for n in lens])
    big = lens >= 42
    for d in (28, 0, 4):                                      # 4q + 20 four bases before, on and after a unit boundary
        assert np.any(big & (ehi % 32 == d) & (lens > ehi)), d
    assert set(lens[lens < 49].tolist()) == set(range(41, 49))
    # the dropped tail (ends 4q + 20 .. n - 1, at most 3) never crosses a unit: 4q + 20 is a multiple of 4
    assert np.all((ehi % 32) + (lens - ehi) <= 32)
    for path in ("host_pack0", "host_pack1", "dev1"):
        s = sketch(ctx, genomes, 1, 15, 1000, avx2, path, monkeypatch)
        refs, _, _ = check_set(s, genomes, 1, 15, 1000, avx2)
        for g, r in zip(genomes, refs):
            assert np.array_equal(np.diff(r["ctg_rec_off"]), [R.n_windows(len(x), avx2) for x in g])
        s.free()


# ---- c -----------------------------------------------------------------------------------------------------------------
def missing_windows(r, ci, n, avx2):
    cc = r["pv_cc"] >> np.uint32(1)
    got = set(r["pv_pos"][cc == ci].tolist())
    visited = set(range(20, 20 + R.n_windows(n, avx2)))
    assert got <= visited
    return visited - got


@pytest.mark.parametrize("avx2", SEM, ids=SEM_IDS)
@pytest.mark.parametrize("byte", [ord("N"), ord("n")], ids=["N", "n"])
def test_c_n_placement(ctx, monkeypatch, avx2, byte):
    genomes, where = SC.n_case(byte)
    k = 15
    breaks = byte == ord("N") or not avx2
    for path in ("host_pack0", "host_pack1", "dev2"):
        s = sketch(ctx, genomes, 1, k, 1000, avx2, path, monkeypatch)
        refs, _, _ = check_set(s, genomes, 1, k, 1000, avx2)
        s.free()
    first = [0] + list(np.cumsum([len(g) for g in genomes]))
    gi = lambda ci: int(np.searchsorted(first, ci, side="right") - 1)          # noqa: E731
    seen = set()
    for ci, n, name, p in where:
        g = gi(ci)
        miss = missing_windows(refs[g], ci - first[g], n, avx2)
        q = (n - 20) // 4
        if not breaks:
            want = set()
        elif avx2:
            lane = [l for l in range(4) if l * q + 20 <= p < l * q + q + 20]   # the lane that visits end p
            want = set(range(p, min(p + 21, lane[0] * q + q + 20))) if lane else set()
        else:
            want = set(range(p, min(p + k, n))) if p >= 20 else set()     # the scalar loop tests from base 20 on
        assert miss == want, (n, name, p, sorted(miss), sorted(want))
        if avx2 and breaks and name.endswith("_q+19") and name != "l0_q+19":
            assert miss == {p}                              # only the previous lane's last window
            seen.add("prefill")
        if name == "last":
            nxt = ci + 1 - first[gi(ci + 1)]
            assert not missing_windows(refs[gi(ci + 1)], nxt, len(genomes[gi(ci + 1)][nxt]), avx2)
            seen.add("next_clean")
        if avx2 and name in ("4q+19", "4q+20") and p >= 4 * q + 20:
            assert not miss                                   # an N past the last visited window breaks nothing
            seen.add("tail")
    assert seen >= ({"next_clean"} | ({"tail"} if avx2 else set()) | ({"prefill"} if avx2 and breaks else set()))


# ---- d -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("total", SC.LOOKUP_TOTALS)
def test_d_contig_lookup(ctx, monkeypatch, total):
    genomes, cuoff = SC.lookup_case(total)
    contigs = [x for g in genomes for x in g]
    lens = np.array([len(x) for x in contigs])
    assert len(contigs) >= 2000 and lens.max() <= 64 and int(((lens + 31) // 32).sum()) == total
    assert np.count_nonzero(lens == 0) >= 5
    at = (cuoff % 256 == 0) & (cuoff > 0)
    assert np.count_nonzero(at & (lens > 0)) >= 3 and np.count_nonzero(at & (lens == 0)) >= 2
    for path in ("host_pack0", "host_pack1", "dev3"):
        for avx2 in SEM:
            s = sketch(ctx, genomes, 1, 15, 1, avx2, path, monkeypatch)
            refs, _, _ = check_set(s, genomes, 1, 15, 1, avx2, export=False)
            for g, r in zip(genomes, refs):
                assert np.array_equal(np.diff(r["ctg_rec_off"]), [R.n_windows(len(x), avx2) for x in g])
            s.free()


# ---- e -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [6, 8, 10])
def test_e_canonical_ties(ctx, monkeypatch, k):
    genomes, ends = SC.tie_case(k)
    _, _, fs, rs = R.windows(genomes[0][0], k)
    assert np.all(fs[0, ends - 20] == rs[0, ends - 20])
    for avx2 in SEM:
        s = sketch(ctx, genomes, 1, k, 1, avx2, "host_pack0", monkeypatch)
        refs, _, _ = check_set(s, genomes, 1, k, 1, avx2)
        e = s.export(0)
        at = np.isin(e["pos"], ends) & (e["cc"] >> np.uint32(1) == 0)
        assert np.count_nonzero(at) == len(ends)                # every planted tie is a record ...
        assert not np.any(e["cc"][at] & np.uint32(1))           # ... with canonical bit 0 ...
        assert np.array_equal(np.sort(e["kmer"][at]), np.sort(rs[0, e["pos"][at] - 20].astype(np.uint32)))   # ... and seed Rs
        s.free()


# ---- f -----------------------------------------------------------------------------------------------------------------
def test_f_multiplicity(ctx, monkeypatch):
    genomes = SC.mult_case()
    s = sketch(ctx, genomes, 1, 15, 1000, True, "host_pack0", monkeypatch)
    (r,), m, a = check_set(s, genomes, 1, 15, 1000, flags=TABLES)
    n0 = np.count_nonzero(r["pv_kmer"] == 0)
    assert n0 > R.MULT_MAX and len(r["pv_kmer"]) < 1 << 20
    assert np.all(r["pv_mult"][r["pv_kmer"] == 0] == R.MULT_MAX)
    assert np.all(r["pv_mult"][r["pv_kmer"] != 0] < 100)
    ht = a["htab"][m["ht_off"][0]:m["ht_off"][1]]
    cnt = np.diff(r["ustart"])
    T.check_table(ht, r["ukmer"], r["ustart"][:-1], cnt)
    found, _, count = T.probe(ht, 0)
    assert found and count == T.COUNT_MAX and r["ukmer"][0] == 0 and cnt[0] == n0
    s.free()


# ---- g -----------------------------------------------------------------------------------------------------------------
def test_g_kview_sort_switch(ctx, monkeypatch):
    out = {}
    for extra in (0, 4):
        genomes = SC.kview_case(extra)
        s = sketch(ctx, genomes, 1, 16, 1000, True, "host_pack0", monkeypatch)
        max_rec = max(s.info(g)["n_records"] for g in range(len(s)))
        assert max_rec == (1 << 21) + extra and s.info(0)["n_records"] == max_rec
        assert SC.kview_bits(max_rec, 16, SC.KVIEW_G) == (64 if extra == 0 else 65)   # keys-only vs pairs sort
        refs, m, a = check_set(s, genomes, 1, 16, 1000, export=False)
        for g in (0, 1, SC.KVIEW_G - 1):
            e = s.export(g)
            for key in ("kmer", "pos", "cc", "markers"):
                assert np.array_equal(e[key], refs[g][key]), (g, key)
        out[extra] = (m, a)
        s.free()
    # the 1024 small genomes are the same on both sides of the switch
    (m0, a0), (m4, a4) = out[0], out[4]
    for name, om in (("pv_kmer", "seed_off"), ("kv_pos", "seed_off"), ("kv_cc", "seed_off"), ("pv_mult", "seed_off"),
                     ("ukmer", "uk_off"), ("markers", "mk_off")):
        assert np.array_equal(a0[name][m0[om][1]:], a4[name][m4[om][1]:]), name


def test_g_marker_sort_switch(ctx, monkeypatch):
    import skani_b200 as sk
    rows = SC.marker_rows(SC.MARKER_G + 1)
    want, want_off = R.markers_rows(rows, 15, 8, 8)
    assert np.mean(np.diff(want_off) >= 2) > 0.5
    for G in (SC.MARKER_G, SC.MARKER_G + 1):
        assert SC.marker_bits(G) == (64 if G == SC.MARKER_G else 65)       # global sort vs per-genome segments
        off = np.arange(G + 1, dtype=np.uint64) * np.uint64(42)
        s = sk.sketch_contigs(ctx, rows[:G].reshape(-1), off, np.arange(G, dtype=np.uint32), G, sk.sketch_params(8, 15, 8))
        m, a = blob(s, MO)
        s.free()
        assert m["G"] == G
        assert np.array_equal(m["mk_off"], want_off[:G + 1].astype(np.int64))
        assert np.array_equal(a["markers"], want[:int(want_off[G])])


# ---- h -----------------------------------------------------------------------------------------------------------------
def test_h_marker_gating(ctx, monkeypatch):
    genomes = SC.marker_gate_case()
    for mc, some in ((30, True), (2 ** 32 - 1, False)):
        s = sketch(ctx, genomes, 30, 15, mc, True, "host_pack0", monkeypatch)
        refs, _, _ = check_set(s, genomes, 30, 15, mc)
        s.free()
        if some:                                              # marker_c == c: every record inserts its marker
            raw = [np.concatenate([R.contig_seeds(x, 15, 30, mc)[3] for x in g]) for g in genomes]
            assert all(len(w) == len(r["pv_kmer"]) for w, r in zip(raw, refs))
            assert len(raw[0]) > len(refs[0]["markers"]) == len(np.unique(raw[0]))     # repeated contigs: stored once
            assert all(len(r["markers"]) > 0 for r in refs)
        else:
            assert all(len(r["markers"]) == 0 and len(r["pv_kmer"]) > 0 for r in refs)
