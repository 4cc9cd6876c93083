"""Thin Python host layer over the C ABI (ctypes).  Names follow the reference: Sketch sets, screen, chain."""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import AniResult, ChainDebug, ClusterParams, ClusterStats, DerepParams, DerepStats, LinkageParams, MapParams, NjStats, SketchParams, StoreStats, TriangleStats

# numpy view of sk_ani_result (include/skani_b200.h): lets callers take 10^5..10^6 results without per-row Python objects
RESULT_DTYPE = np.dtype([(n, np.float32) for n in ("ani", "af_query", "af_ref", "ci_lower", "ci_upper", "std", "q90_q", "q90_r", "q50_q",
                                                   "q50_r", "q10_q", "q10_r")] +
                        [(n, np.uint32) for n in ("num_contigs_q", "num_contigs_r", "avg_chain_int_len", "total_bases_covered",
                                                  "ref_id", "query_id")])
assert RESULT_DTYPE.itemsize == C.sizeof(AniResult)
# sk_mapping: one kept chain interval of a pair in the caller's orientation, with its chunk's identity estimate
MAPPING_DTYPE = np.dtype([(n, np.uint32) for n in ("query_contig", "ref_contig", "q0", "q1", "r0", "r1", "num_anchors", "chunk")] +
                         [("chunk_est", np.float64), ("chunk_weight", np.uint32)] +
                         [(n, np.uint8) for n in ("reverse", "switched", "chunk_valid", "pad")])
assert MAPPING_DTYPE.itemsize == 48

MIN_LENGTH_CONTIG = 500  # reference src/params.rs:42, applied by file_io::fastx_to_sketches (src/file_io.rs:176)


class SkaniError(RuntimeError):
    pass


def sketch_params(c=125, k=15, marker_c=1000):
    return SketchParams(c, k, marker_c)


def map_params(screen_val=0.0, min_af=0.15, both_min_af=-0.01, robust=False, median=False, learned_ani=True,
               rescue_small=True):
    return MapParams(screen_val, min_af, both_min_af, int(robust), int(median), int(learned_ani), int(rescue_small))


class Context:
    def __init__(self, device=0):
        self.L = _lib.load()
        h = C.c_void_p()
        rc = self.L.sk_ctx_create(device, C.byref(h))
        if rc != 0:
            raise SkaniError("sk_ctx_create failed (rc=%d): a CUDA device is required, there is no CPU fallback" % rc)
        self.h = h

    def check(self, rc):
        if rc != 0:
            raise SkaniError("rc=%d: %s" % (rc, self.L.sk_last_error(self.h).decode()))

    @property
    def launches(self):
        return self.L.sk_ctx_launch_count(self.h)

    @property
    def last_pack_share(self):
        return self.L.sk_ctx_last_pack_share(self.h)

    @property
    def stream(self):
        return self.L.sk_ctx_stream(self.h)

    def set_seeding_semantics(self, scalar=False):
        """False = avx2_fmh_seeds (default, src/avx2_seeding.rs:33); True = scalar fmh_seeds (src/seeding.rs:225)."""
        self.check(self.L.sk_ctx_set_seeding_semantics(self.h, 1 if scalar else 0))

    def set_timing(self, on=True):
        self.check(self.L.sk_ctx_set_timing(self.h, int(on)))

    def get_timing(self, reset=True):
        """{kernel_name: (total_ms, launches)} measured with CUDA events on the launch stream."""
        buf = C.create_string_buffer(1 << 16)
        self.check(self.L.sk_ctx_get_timing(self.h, buf, len(buf), int(reset)))
        out = {}
        for ln in buf.value.decode().splitlines():
            name, ms, n = ln.split()
            out[name] = (float(ms), int(n))
        return out

    def close(self):
        if self.h:
            self.L.sk_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SketchSet:
    """Device-resident Vec<Sketch> (reference src/types.rs:253-277)."""

    def __init__(self, ctx, handle, names=None):
        self.ctx, self.h, self.names = ctx, handle, names

    def __len__(self):
        return self.ctx.L.sk_sketch_set_n_genomes(self.h)

    def info(self, g):
        v = [C.c_uint64() for _ in range(5)]
        self.ctx.check(self.ctx.L.sk_sketch_set_genome_info(self.h, g, *[C.byref(x) for x in v]))
        return dict(zip(("n_records", "n_kmers", "n_markers", "n_contigs", "total_len"), [x.value for x in v]))

    def export(self, g):
        i = self.info(g)
        kmer = np.zeros(i["n_records"], np.uint32); pos = np.zeros_like(kmer); cc = np.zeros_like(kmer)
        mk = np.zeros(i["n_markers"], np.uint64); cl = np.zeros(i["n_contigs"], np.uint32)
        self.ctx.check(self.ctx.L.sk_sketch_set_export(self.h, g, kmer.ctypes.data, pos.ctypes.data, cc.ctypes.data,
                                                       mk.ctypes.data, cl.ctypes.data))
        return dict(kmer=kmer, pos=pos, cc=cc, markers=mk, contig_lengths=cl)

    def _entry_meta(self, g0, n, names, contigs, contig_order):
        """sk_entry_meta of genomes [g0, g0 + n): names[i] (str or bytes), contigs[i] (list of names), contig_order[i]"""
        enc = lambda s: s.encode() if isinstance(s, str) else bytes(s)          # noqa: E731
        nm = [enc(x) for x in names]
        cn = [[enc(x) for x in c] for c in contigs]
        if not (len(nm) == len(cn) == len(contig_order) == n):
            raise ValueError("names, contigs and contig_order need one entry per genome")
        keep = dict(
            names=np.frombuffer(b"".join(nm) + b"\0", np.uint8),
            name_off=np.cumsum([0] + [len(x) for x in nm], dtype=np.uint64),
            contig_names=np.frombuffer(b"".join(b"".join(c) for c in cn) + b"\0", np.uint8),
            contig_name_off=np.cumsum([0] + [len(x) for c in cn for x in c], dtype=np.uint64),
            contig_first=np.cumsum([0] + [len(c) for c in cn], dtype=np.uint64),
            contig_order=np.ascontiguousarray(list(contig_order) + [0], np.uint64))
        meta = _lib.EntryMeta(*[keep[f].ctypes.data for f, _ in _lib.EntryMeta._fields_])
        return meta, keep

    def encode_sizes(self, names, contigs, contig_order, g0=0, n=None, markers_only=False):
        """Lengths of the skani v0.3 entries encode writes for genomes [g0, g0 + n)."""
        n = len(self) - g0 if n is None else n
        meta, _keep = self._entry_meta(g0, n, names, contigs, contig_order)
        ln = np.zeros(max(n, 1), np.uint64)
        self.ctx.check(self.ctx.L.sk_sketch_set_encode_sizes(self.h, g0, n, int(markers_only), C.byref(meta), ln.ctypes.data))
        return ln[:n]

    def encode(self, names, contigs, contig_order, g0=0, n=None, markers_only=False, out=None):
        """Genomes [g0, g0 + n) as skani v0.3 entries, encoded on the device (sk_sketch_set_encode): (SketchParams, Sketch)
        each (a sketches.db entry or .sketch file), or Sketch::get_markers_only (an element of markers.bin) with
        markers_only.  names[i], contigs[i] and contig_order[i] are genome g0 + i's file name, contig names and
        contig_order.  out: optional uint8 array (pinned or pageable) to write into.  Returns (bytes, entry lengths)."""
        n = len(self) - g0 if n is None else n
        meta, _keep = self._entry_meta(g0, n, names, contigs, contig_order)
        if out is None:
            out = np.empty(int(self.encode_sizes(names, contigs, contig_order, g0, n, markers_only).sum()), np.uint8)
        ln = np.zeros(max(n, 1), np.uint64)
        buf = out if len(out) else np.zeros(1, np.uint8)
        self.ctx.check(self.ctx.L.sk_sketch_set_encode(self.h, g0, n, int(markers_only), C.byref(meta), buf.ctypes.data, len(out),
                                                       ln.ctypes.data))
        return out[:int(ln[:n].sum())], ln[:n]

    def set_name_ranks(self, ranks):
        """Order of the sketches' FILE names (equal names -> equal ranks): the tie-break of switch_qr
        (reference src/chain.rs:19-21) compares file names, and with -i / --qi / --ri all records of one file share a name."""
        r = np.ascontiguousarray(ranks, np.uint64)
        assert len(r) == len(self)
        self.ctx.check(self.ctx.L.sk_sketch_set_set_name_ranks(self.h, r.ctypes.data))

    def _genome_arg(self, genomes):
        if genomes is None:
            return None, 0, None
        g = np.ascontiguousarray(genomes, np.uint32)
        keep = g if len(g) else np.zeros(1, np.uint32)      # never hand the library a NULL pointer for "no genomes"
        return keep.ctypes.data, len(g), keep

    def subset_blob_size(self, genomes=None, flags=0):
        """(device bytes, metadata words) of the blob sk_sketch_set_pack_subset would write; genomes=None -> all."""
        ptr, n, _keep = self._genome_arg(genomes)
        nb, nw = C.c_uint64(), C.c_uint64()
        self.ctx.check(self.ctx.L.sk_sketch_set_subset_blob_size(self.h, ptr, n, flags, C.byref(nb), C.byref(nw)))
        return nb.value, nw.value

    def pack_subset(self, genomes, flags, device_ptr, n_words):
        """Pack the chosen genomes into caller-owned device memory; returns the host metadata vector (uint64)."""
        ptr, n, _keep = self._genome_arg(genomes)
        meta = np.zeros(n_words, np.uint64)
        self.ctx.check(self.ctx.L.sk_sketch_set_pack_subset(self.h, ptr, n, flags, device_ptr, meta.ctypes.data))
        return meta

    def append(self, other):
        self.ctx.check(self.ctx.L.sk_sketch_set_append(self.h, other.h))

    def copy_to(self, ctx):
        """sk_sketch_set_copy: the same set (k-mer tables and name ranks included) on another context, which may share the device."""
        h = C.c_void_p()
        ctx.check(ctx.L.sk_sketch_set_copy(ctx.h, self.h, C.byref(h)))
        return SketchSet(ctx, h, self.names)

    def free(self):
        if self.h and self.ctx.h:      # the set's storage lives in its context's arena
            self.ctx.L.sk_sketch_set_free(self.h)
        self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _as_u8(x):
    if isinstance(x, (bytes, bytearray)):
        return np.frombuffer(x, np.uint8)
    return np.ascontiguousarray(x, dtype=np.uint8)


def sketch_contigs(ctx, bases, contig_off, genome_of_contig, n_genomes, sp=None, device_ptr=None):
    """sk_sketch_batch on already-laid-out buffers (bases: uint8 array or None when device_ptr is given)."""
    sp = sp or sketch_params()
    contig_off = np.ascontiguousarray(contig_off, np.uint64)
    goc = np.ascontiguousarray(genome_of_contig, np.uint32)
    out = C.c_void_p()
    if device_ptr is not None:
        rc = ctx.L.sk_sketch_batch_dev(ctx.h, device_ptr, contig_off.ctypes.data, len(goc), goc.ctypes.data, n_genomes,
                                       C.byref(sp), C.byref(out))
    else:
        arr = None if isinstance(bases, int) else _as_u8(bases)   # keep the (possibly copied) array alive across the call
        ptr = bases if arr is None else arr.ctypes.data
        rc = ctx.L.sk_sketch_batch(ctx.h, ptr, contig_off.ctypes.data, len(goc), goc.ctypes.data, n_genomes,
                                   C.byref(sp), C.byref(out))
    ctx.check(rc)
    return SketchSet(ctx, out)


def pack_contigs(L, bases, contig_off):
    """ASCII contigs -> (units uint64, nmask uint32, contig_len uint32) in sk_sketch_batch_2bit's layout (host side, sk_pack_contig)."""
    bases = _as_u8(bases)
    off = np.ascontiguousarray(contig_off, np.uint64)
    lens = np.diff(off).astype(np.uint32)
    uoff = np.concatenate([[0], np.cumsum((lens.astype(np.uint64) + 31) // 32)]).astype(np.uint64)
    units = np.zeros(max(int(uoff[-1]), 1), np.uint64); nmask = np.zeros(max(int(uoff[-1]), 1), np.uint32)
    for i in range(len(lens)):
        rc = L.sk_pack_contig(bases.ctypes.data + int(off[i]), int(lens[i]), units.ctypes.data + 8 * int(uoff[i]), nmask.ctypes.data + 4 * int(uoff[i]))
        assert rc == 0
    return units, nmask, lens


def sketch_contigs_2bit(ctx, units, nmask, contig_len, genome_of_contig, n_genomes, sp=None):
    """sk_sketch_batch_2bit: sequences already packed as 2-bit units (+ optional N mask, None = no 'N')."""
    sp = sp or sketch_params()
    units = np.ascontiguousarray(units, np.uint64)
    nm = None if nmask is None else np.ascontiguousarray(nmask, np.uint32)
    cl = np.ascontiguousarray(contig_len, np.uint32)
    goc = np.ascontiguousarray(genome_of_contig, np.uint32)
    out = C.c_void_p()
    ctx.check(ctx.L.sk_sketch_batch_2bit(ctx.h, units.ctypes.data, None if nm is None else nm.ctypes.data, cl.ctypes.data, len(cl),
                                         goc.ctypes.data, n_genomes, C.byref(sp), C.byref(out)))
    return SketchSet(ctx, out)


def sketch_sequences(ctx, genomes, sp=None, individual_contig=False):
    """genomes: list of genomes, each a list of contig byte strings (one file's records, in file order).
    Applies the reference's record rules (file_io.rs:141-362): records < 500 bp are dropped, files without a
    kept record yield no sketch; with individual_contig every kept record becomes its own sketch."""
    arrs, goc, g = [], [], 0
    kept_genomes = []
    for gi, contigs in enumerate(genomes):
        kept = [_as_u8(c) for c in contigs if len(c) >= MIN_LENGTH_CONTIG]
        if not kept:
            continue
        if individual_contig:
            for j, a in enumerate(kept):
                arrs.append(a); goc.append(g); g += 1
                kept_genomes.append((gi, j))
        else:
            for a in kept:
                arrs.append(a); goc.append(g)
            g += 1
            kept_genomes.append((gi, 0))
    off = np.zeros(len(arrs) + 1, np.uint64)
    if arrs:
        off[1:] = np.cumsum([len(a) for a in arrs])
    bases = np.concatenate(arrs) if arrs else np.zeros(1, np.uint8)
    s = sketch_contigs(ctx, bases, off, goc, g, sp)
    s.names = kept_genomes
    if individual_contig and g:
        s.set_name_ranks([gi for gi, _ in kept_genomes])   # records of one file share its name
    return s


def import_sketches(ctx, sketches, sp=None, seeds=True):
    """Device sketch set from host-side sketches (e.g. decoded from a skani database; reference
    file_io::sketches_from_sketch src/file_io.rs:680, sketch_db::get_sketch src/sketch_db.rs:104).  sketches: list of dicts
    with kmer / pos / cc (seed records, any order), markers (distinct), contig_lengths and optionally total_len, i.e. what
    SketchSet.export returns.  seeds=False imports the markers only (the markers.bin form, Sketch::get_markers_only)."""
    sp = sp or sketch_params()
    n = len(sketches)
    z32, z64 = np.zeros(0, np.uint32), np.zeros(0, np.uint64)
    cat = lambda key, z: np.ascontiguousarray(np.concatenate([np.asarray(s[key], z.dtype) for s in sketches] + [z]))
    off = lambda key: np.ascontiguousarray(np.concatenate([[0], np.cumsum([len(s[key]) for s in sketches])]).astype(np.uint64))
    if seeds:
        kmer, pos, cc, cl = cat("kmer", z32), cat("pos", z32), cat("cc", z32), cat("contig_lengths", z32)
        rec_off, ctg_off = off("kmer"), off("contig_lengths")
    else:
        kmer = pos = cc = cl = np.zeros(1, np.uint32)
        rec_off = ctg_off = np.zeros(n + 1, np.uint64)
    mk, mk_off = cat("markers", z64), off("markers")
    tl = np.ascontiguousarray([int(s["total_len"]) if "total_len" in s else int(np.sum(s["contig_lengths"], dtype=np.uint64)) for s in sketches],
                              np.uint64)
    h = C.c_void_p()
    ctx.check(ctx.L.sk_sketch_set_import_batch(ctx.h, C.byref(sp), n, rec_off.ctypes.data, kmer.ctypes.data, pos.ctypes.data, cc.ctypes.data,
                                               mk_off.ctypes.data, mk.ctypes.data, ctg_off.ctypes.data, cl.ctypes.data, tl.ctypes.data,
                                               C.byref(h)))
    return SketchSet(ctx, h)


class BlobError(SkaniError):
    """sk_sketch_set_import_blobs refused a blob: .blob is its index (None when the error is not a blob's)."""
    def __init__(self, msg, blob):
        super().__init__(msg)
        self.blob = blob


def import_blobs(ctx, data, offsets, lengths, sp=None):
    """Device sketch set from skani v0.3 sketch blobs as stored (.sketch file bytes or sketches.db slices located by
    index.db): blob g = data[offsets[g]:offsets[g] + lengths[g]], expanded on the device.  data: bytes or a uint8 array
    (pinned or pageable host memory).  Raises BlobError naming the first blob that does not decode."""
    sp = sp or sketch_params()
    buf = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else np.ascontiguousarray(data, np.uint8)
    off = np.ascontiguousarray(offsets, np.uint64)
    ln = np.ascontiguousarray(lengths, np.uint64)
    if len(off) != len(ln) or (len(off) and int((off + ln).max()) > len(buf)):
        raise ValueError("blob offsets / lengths outside the data")
    h, bad = C.c_void_p(), C.c_uint32()
    rc = ctx.L.sk_sketch_set_import_blobs(ctx.h, C.byref(sp), buf.ctypes.data if len(buf) else None, off.ctypes.data, ln.ctypes.data,
                                          len(off), C.byref(h), C.byref(bad))
    if rc != 0:
        raise BlobError("rc=%d: %s" % (rc, ctx.L.sk_last_error(ctx.h).decode()), None if bad.value == 0xFFFFFFFF else bad.value)
    return SketchSet(ctx, h)


def _pairs_out(ctx, fn, *args):
    pp = C.POINTER(C.c_uint64)(); n = C.c_uint64()
    ctx.check(fn(*args, C.byref(pp), C.byref(n)))
    arr = np.ctypeslib.as_array(pp, shape=(n.value,)).copy() if n.value else np.zeros(0, np.uint64)
    ctx.L.sk_free(pp)
    return arr


def screen_triangle(ctx, sset, mp=None):
    mp = mp or map_params()
    return _pairs_out(ctx, ctx.L.sk_screen_triangle, ctx.h, sset.h, C.byref(mp))


def screen_triangle_rows(ctx, sset, row_mod, row_rem, mp=None):
    """Pairs (i, j), i < j, of the triangle screen whose row i satisfies i % row_mod == row_rem."""
    mp = mp or map_params()
    return _pairs_out(ctx, ctx.L.sk_screen_triangle_rows, ctx.h, sset.h, C.byref(mp), int(row_mod), int(row_rem))


def screen_triangle_block(ctx, sset, g_begin, g_end, mp=None):
    """Pairs (i, j), i < j, g_begin <= j < g_end of the triangle screen (sharded screen: one block of rows)."""
    mp = mp or map_params()
    pp = C.POINTER(C.c_uint64)(); n = C.c_uint64()
    ctx.check(ctx.L.sk_screen_triangle_block(ctx.h, sset.h, int(g_begin), int(g_end), C.byref(mp), C.byref(pp), C.byref(n)))
    arr = np.ctypeslib.as_array(pp, shape=(n.value,)).copy() if n.value else np.zeros(0, np.uint64)
    ctx.L.sk_free(pp)
    return arr


def screen_query_ref(ctx, refs, queries, mp=None, mode=0):
    mp = mp or map_params()
    pp = C.POINTER(C.c_uint64)(); n = C.c_uint64()
    ctx.check(ctx.L.sk_screen_query_ref(ctx.h, refs.h, queries.h, C.byref(mp), mode, C.byref(pp), C.byref(n)))
    arr = np.ctypeslib.as_array(pp, shape=(n.value,)).copy() if n.value else np.zeros(0, np.uint64)
    ctx.L.sk_free(pp)
    return arr


class RefIndex:
    """sk_ref_index: the markers of a reference set sorted once on ctx, in contiguous parts of < 2^31 markers
    (SK_REF_INDEX_PART_MARKERS at creation lowers the bound).  screen() of any query set on ctx returns
    screen_query_ref(ctx, refs, queries, mp, mode); refs may be freed once the index exists."""

    def __init__(self, ctx, refs):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.check(ctx.L.sk_ref_index_create(ctx.h, refs.h, C.byref(h)))
        self.h = h

    def screen(self, queries, mp=None, mode=0):
        mp = mp or map_params()
        return _pairs_out(self.ctx, self.ctx.L.sk_ref_index_screen, self.ctx.h, self.h, queries.h, C.byref(mp), int(mode))

    def info(self):
        """(references, parts, device bytes held)"""
        g, p, b = C.c_uint32(), C.c_uint32(), C.c_uint64()
        self.ctx.check(self.ctx.L.sk_ref_index_info(self.h, C.byref(g), C.byref(p), C.byref(b)))
        return g.value, p.value, b.value

    def free(self):
        if self.h:
            self.ctx.L.sk_ref_index_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def chain_pairs(ctx, refs, queries, pairs, mp=None, as_array=False):
    """sk_chain_pairs.  as_array=True returns a numpy structured array (RESULT_DTYPE) instead of a list of AniResult."""
    mp = mp or map_params()
    pairs = np.ascontiguousarray(pairs, np.uint64)
    out = np.zeros(max(len(pairs), 1), RESULT_DTYPE)
    ctx.check(ctx.L.sk_chain_pairs(ctx.h, refs.h, queries.h, pairs.ctypes.data, len(pairs), C.byref(mp), out.ctypes.data))
    out = out[:len(pairs)]
    if as_array:
        return out
    return [AniResult.from_buffer_copy(out[i].tobytes()) for i in range(len(pairs))]


def _mappings_out(ctx, n, off, pp):
    m = np.frombuffer((C.c_uint8 * (int(off[n]) * 48)).from_address(pp.value), MAPPING_DTYPE).copy() \
        if off[n] else np.zeros(0, MAPPING_DTYPE)
    ctx.L.sk_free(pp)
    return m


def chain_pairs_mappings(ctx, refs, queries, pairs, mp=None):
    """sk_chain_pairs_mappings: (results, offsets, mappings).  results is chain_pairs(..., as_array=True); pair i's records
    are mappings[offsets[i]:offsets[i + 1]] (MAPPING_DTYPE), its kept chain intervals in the caller's orientation."""
    mp = mp or map_params()
    pairs = np.ascontiguousarray(pairs, np.uint64)
    out = np.zeros(max(len(pairs), 1), RESULT_DTYPE)
    off = np.zeros(len(pairs) + 1, np.uint64)
    pp = C.c_void_p()
    ctx.check(ctx.L.sk_chain_pairs_mappings(ctx.h, refs.h, queries.h, pairs.ctypes.data, len(pairs), C.byref(mp), out.ctypes.data,
                                            off.ctypes.data, C.byref(pp)))
    return out[:len(pairs)], off, _mappings_out(ctx, len(pairs), off, pp)


def _multi_args(ctxs, refs, ref_first, queries):
    hs = (C.c_void_p * len(ctxs))(*[c.h for c in ctxs])
    rh = (C.c_void_p * len(ctxs))(*[None if r is None else r.h for r in refs])
    qh = (C.c_void_p * len(ctxs))(*[q.h for q in queries])
    rf = np.ascontiguousarray(ref_first, np.uint32)
    assert len(refs) == len(queries) == len(rf) == len(ctxs)
    return hs, rh, rf, qh


def screen_query_ref_multi(ctxs, refs, ref_first, queries, mp=None, mode=0):
    """sk_screen_query_ref_multi: refs[d] (None or a set on ctxs[d]) holds the global refs [ref_first[d], ref_first[d] + len);
    queries[d] is the query set on ctxs[d].  Same pair list as screen_query_ref on one set of all refs."""
    mp = mp or map_params()
    hs, rh, rf, qh = _multi_args(ctxs, refs, ref_first, queries)
    c0 = ctxs[0]
    return _pairs_out(c0, c0.L.sk_screen_query_ref_multi, hs, len(ctxs), rh, rf.ctypes.data, qh, C.byref(mp), mode)


def chain_pairs_multi(ctxs, refs, ref_first, queries, pairs, mp=None, as_array=False):
    """sk_chain_pairs_multi: global (ref << 32 | query) pairs in any order, each chained on the context holding its ref.
    Same results as chain_pairs on one set of all refs, ref_id global."""
    mp = mp or map_params()
    hs, rh, rf, qh = _multi_args(ctxs, refs, ref_first, queries)
    pairs = np.ascontiguousarray(pairs, np.uint64)
    out = np.zeros(max(len(pairs), 1), RESULT_DTYPE)
    c0 = ctxs[0]
    c0.check(c0.L.sk_chain_pairs_multi(hs, len(ctxs), rh, rf.ctypes.data, qh, pairs.ctypes.data, len(pairs), C.byref(mp), out.ctypes.data))
    out = out[:len(pairs)]
    if as_array:
        return out
    return [AniResult.from_buffer_copy(out[i].tobytes()) for i in range(len(pairs))]


def chain_pairs_multi_mappings(ctxs, refs, ref_first, queries, pairs, mp=None):
    """sk_chain_pairs_multi_mappings: chain_pairs_multi plus mappings, returned as chain_pairs_mappings returns them."""
    mp = mp or map_params()
    hs, rh, rf, qh = _multi_args(ctxs, refs, ref_first, queries)
    pairs = np.ascontiguousarray(pairs, np.uint64)
    out = np.zeros(max(len(pairs), 1), RESULT_DTYPE)
    off = np.zeros(len(pairs) + 1, np.uint64)
    pp = C.c_void_p()
    c0 = ctxs[0]
    c0.check(c0.L.sk_chain_pairs_multi_mappings(hs, len(ctxs), rh, rf.ctypes.data, qh, pairs.ctypes.data, len(pairs), C.byref(mp),
                                                out.ctypes.data, off.ctypes.data, C.byref(pp)))
    return out[:len(pairs)], off, _mappings_out(c0, len(pairs), off, pp)


def _debug_dict(d):
    def arr(p, shape, dt):
        n = int(np.prod(shape))
        return np.ctypeslib.as_array(p, shape=(n,)).astype(dt).reshape(shape).copy() if n else np.zeros(shape, dt)
    return dict(result=AniResult.from_buffer_copy(d.result), switched=bool(d.switched),
                anchors=arr(d.anchors, (d.n_anchors, 5), np.uint32), score=arr(d.score, (d.n_anchors,), np.int64),
                pointer=arr(d.pointer, (d.n_anchors,), np.uint32),
                chunk_first=arr(d.chunk_first, (d.n_chunks + 1,), np.uint32) if d.n_chunks else np.zeros(1, np.uint32),
                chunk_nseeds=arr(d.chunk_nseeds, (d.n_chunks,), np.uint32),
                intervals=arr(d.intervals, (d.n_intervals, 11), np.int64),
                est=arr(d.est, (d.n_ests,), np.float64), weight=arr(d.weight, (d.n_ests,), np.uint64),
                chunk_stats=arr(d.chunk_stats, (d.n_chunks, 9), np.uint32))


def chain_pairs_debug(ctx, refs, queries, pairs, mp=None, keep=None):
    """sk_chain_pairs_debug: the intermediate products of every pair of `pairs` (same batching and kernels as chain_pairs).
    Returns one dict per pair, or with keep (pair indices) a {index: dict} of those pairs only."""
    mp = mp or map_params()
    pairs = np.ascontiguousarray(pairs, np.uint64)
    n = len(pairs)
    ds = (ChainDebug * max(n, 1))()
    ctx.check(ctx.L.sk_chain_pairs_debug(ctx.h, refs.h, queries.h, pairs.ctypes.data, n, C.byref(mp), ds))
    try:
        if keep is None:
            return [_debug_dict(ds[i]) for i in range(n)]
        return {int(i): _debug_dict(ds[int(i)]) for i in keep}
    finally:
        for i in range(n):
            ctx.L.sk_chain_debug_free(C.byref(ds[i]))


def chain_pair_debug(ctx, refs, queries, ref_id, query_id, mp=None):
    return chain_pairs_debug(ctx, refs, queries, [(ref_id << 32) | query_id], mp)[0]


CHUNK_STAT_FIELDS = ("total_anchors", "rq0", "rq1", "tbcq", "n_int", "n_seeds", "num_in", "upper_lower", "filtered")


def debug_chunk_estimate(ctx, inputs, c, k):
    """sk_debug_chunk_estimate: the device's chunk_estimate over rows (total_anchors, rq0, rq1, tbcq, n_int, n_seeds, num_in,
    upper_lower).  Returns (est f64, weight u32, valid u32: 0 no estimate, 1 estimate, 3 estimate with the filter applied)."""
    x = np.ascontiguousarray(inputs, np.uint32).reshape(-1, 8)
    n = len(x)
    est = np.zeros(max(n, 1), np.float64); w = np.zeros(max(n, 1), np.uint32); v = np.zeros(max(n, 1), np.uint32)
    ctx.check(ctx.L.sk_debug_chunk_estimate(ctx.h, n, x.ctypes.data, c, k, est.ctypes.data, w.ctypes.data, v.ctypes.data))
    return est[:n], w[:n], v[:n]


def _debug_pairs(ctx, fn, n, args, switched):
    sw = np.ascontiguousarray(np.broadcast_to(np.asarray(switched, np.uint32), (n,)))
    ds = (ChainDebug * max(n, 1))()
    sums = np.zeros((max(n, 1), 2), np.uint32)
    ctx.check(fn(*args, sw.ctypes.data, ds, sums.ctypes.data))
    try:
        out = []
        for i in range(n):
            d = _debug_dict(ds[i])
            d["pair_sumlen"], d["pair_nchains"] = int(sums[i, 0]), int(sums[i, 1])
            out.append(d)
        return out
    finally:
        for i in range(n):
            ctx.L.sk_chain_debug_free(C.byref(ds[i]))


def debug_chain_anchors(ctx, c, k, pairs, switched=0):
    """sk_debug_chain_anchors: the production DP and interval selection on given anchors.  pairs: one list of chunks per pair,
    each chunk an (n, 5) array of (query_contig, query_pos, ref_contig, ref_pos, reverse).  Returns one chain_pairs_debug dict
    per pair (chunk_stats columns 0-4 = the selection's per-chunk sums) plus pair_sumlen and pair_nchains."""
    chunks = [np.asarray(ch, np.uint32).reshape(-1, 5) for p in pairs for ch in p]
    pco = np.zeros(len(pairs) + 1, np.uint64); pco[1:] = np.cumsum([len(p) for p in pairs])
    cao = np.zeros(len(chunks) + 1, np.uint64); cao[1:] = np.cumsum([len(ch) for ch in chunks])
    a = np.ascontiguousarray(np.concatenate(chunks) if chunks else np.zeros((1, 5), np.uint32))
    return _debug_pairs(ctx, ctx.L.sk_debug_chain_anchors, len(pairs),
                        (ctx.h, c, k, len(pairs), pco.ctypes.data, cao.ctypes.data, a.ctypes.data), switched)


def debug_select_intervals(ctx, c, k, pairs, n_chunks, switched=0):
    """sk_debug_select_intervals: the interval selection alone.  pairs: one (n, 10) array per pair of (score, num_anchors, q0,
    q1, r0, r1, ref_contig, query_contig, chunk, reverse); n_chunks: chunks per pair (scalar or per pair)."""
    ivs = [np.asarray(p, np.int64).reshape(-1, 10) for p in pairs]
    off = np.zeros(len(pairs) + 1, np.uint64); off[1:] = np.cumsum([len(x) for x in ivs])
    x = np.ascontiguousarray(np.concatenate(ivs) if ivs else np.zeros((1, 10), np.int64))
    nc = np.ascontiguousarray(np.broadcast_to(np.asarray(n_chunks, np.uint32), (len(pairs),)))
    return _debug_pairs(ctx, ctx.L.sk_debug_select_intervals, len(pairs),
                        (ctx.h, c, k, len(pairs), off.ctypes.data, x.ctypes.data, nc.ctypes.data), switched)


def debug_derep_screen(ctx, sset, slot_genome, rows, upper=False, batches=None, mp=None):
    """sk_debug_derep_screen: dereplicate's marker index over the slots slot_genome (genome ids), built in index additions of
    batches[b] slots (default: one), and its row screen of rows (upper: rows == slot_genome, row k against the slots above
    k).  Returns (pairs, keys, bucket): the sorted min << 32 | max pairs that pass, the index keys marker << 22 | slot and the
    2^16 + 1 prefix buckets."""
    mp = mp or map_params()
    sg = np.ascontiguousarray(slot_genome, np.uint32)
    rw = np.ascontiguousarray(rows, np.uint32)
    bs = np.ascontiguousarray([len(sg)] if batches is None else batches, np.uint32)
    pp, kp = C.POINTER(C.c_uint64)(), C.POINTER(C.c_uint64)()
    n, nk = C.c_uint64(), C.c_uint64()
    bucket = np.zeros((1 << 16) + 1, np.uint32)
    ctx.check(ctx.L.sk_debug_derep_screen(ctx.h, sset.h, C.byref(mp), sg.ctypes.data if len(sg) else None, len(sg),
                                          bs.ctypes.data if len(bs) else None, len(bs), rw.ctypes.data if len(rw) else None, len(rw),
                                          int(bool(upper)), C.byref(pp), C.byref(n), C.byref(kp), C.byref(nk), bucket.ctypes.data))
    take = lambda p, m: np.ctypeslib.as_array(p, shape=(m,)).copy() if m else np.zeros(0, np.uint64)
    pairs, keys = take(pp, n.value), take(kp, nk.value)
    ctx.L.sk_free(pp)
    ctx.L.sk_free(kp)
    return pairs, keys, bucket


def triangle(ctx, bases, contig_off, genome_of_contig, n_genomes, sp=None, mp=None, as_array=False):
    """Whole `skani triangle` hot path from host buffers (reference src/triangle.rs:13-105)."""
    sp = sp or sketch_params(); mp = mp or map_params()
    contig_off = np.ascontiguousarray(contig_off, np.uint64)
    goc = np.ascontiguousarray(genome_of_contig, np.uint32)
    arr = None if isinstance(bases, int) else _as_u8(bases)       # keep the (possibly copied) array alive across the call
    ptr = bases if arr is None else arr.ctypes.data
    out = C.POINTER(AniResult)(); n = C.c_uint64(); st = TriangleStats()
    ctx.check(ctx.L.sk_triangle(ctx.h, ptr, contig_off.ctypes.data, len(goc), goc.ctypes.data, n_genomes, C.byref(sp),
                                C.byref(mp), C.byref(out), C.byref(n), C.byref(st)))
    if as_array:
        res = np.frombuffer(C.string_at(out, n.value * C.sizeof(AniResult)), RESULT_DTYPE).copy() if n.value else np.zeros(0, RESULT_DTYPE)
    else:
        res = [AniResult.from_buffer_copy(out[i]) for i in range(n.value)]
    ctx.L.sk_free(out)
    return res, st


def _take_results(ctx, out, n, as_array):
    if as_array:
        res = np.frombuffer(C.string_at(out, n.value * C.sizeof(AniResult)), RESULT_DTYPE).copy() if n.value else np.zeros(0, RESULT_DTYPE)
    else:
        res = [AniResult.from_buffer_copy(out[i]) for i in range(n.value)]
    ctx.L.sk_free(out)
    return res


def triangle_local(ctx, bases, contig_off, genome_of_contig, n_genomes, sp=None, mp=None, name_ranks=None, as_array=True):
    """sk_triangle_local: the whole triangle of one genome block + the block's device-resident sketch set (with k-mer tables)."""
    sp = sp or sketch_params(); mp = mp or map_params()
    contig_off = np.ascontiguousarray(contig_off, np.uint64)
    goc = np.ascontiguousarray(genome_of_contig, np.uint32)
    arr = None if isinstance(bases, int) else _as_u8(bases)
    ptr = bases if arr is None else arr.ctypes.data
    nr = None if name_ranks is None else np.ascontiguousarray(name_ranks, np.uint64)
    out = C.POINTER(AniResult)(); n = C.c_uint64(); st = TriangleStats(); h = C.c_void_p()
    ctx.check(ctx.L.sk_triangle_local(ctx.h, ptr, contig_off.ctypes.data, len(goc), goc.ctypes.data, n_genomes, C.byref(sp), C.byref(mp),
                                      None if nr is None else nr.ctypes.data, C.byref(out), C.byref(n), C.byref(st), C.byref(h)))
    return _take_results(ctx, out, n, as_array), SketchSet(ctx, h), st


def triangle_2bit(ctx, units, nmask, contig_len, genome_of_contig, n_genomes, sp=None, mp=None, name_ranks=None, as_array=True, keep_set=False):
    """sk_triangle_2bit: the triangle of genomes that are already 2-bit packed on the host (units may be an address).  Returns
    (results, stats) or, with keep_set, (results, SketchSet, stats)."""
    sp = sp or sketch_params(); mp = mp or map_params()
    cl = np.ascontiguousarray(contig_len, np.uint32)
    goc = np.ascontiguousarray(genome_of_contig, np.uint32)
    ua = None if isinstance(units, int) else np.ascontiguousarray(units, np.uint64)
    uptr = units if ua is None else ua.ctypes.data
    na = None if (nmask is None or isinstance(nmask, int)) else np.ascontiguousarray(nmask, np.uint32)
    nptr = nmask if na is None else na.ctypes.data
    nr = None if name_ranks is None else np.ascontiguousarray(name_ranks, np.uint64)
    out = C.POINTER(AniResult)(); n = C.c_uint64(); st = TriangleStats(); h = C.c_void_p()
    ctx.check(ctx.L.sk_triangle_2bit(ctx.h, uptr, nptr, cl.ctypes.data, len(cl), goc.ctypes.data, n_genomes, C.byref(sp), C.byref(mp),
                                     None if nr is None else nr.ctypes.data, C.byref(out), C.byref(n), C.byref(st),
                                     C.byref(h) if keep_set else None))
    res = _take_results(ctx, out, n, as_array)
    return (res, SketchSet(ctx, h), st) if keep_set else (res, st)


def triangle_multi(ctxs, bases, contig_off, genome_of_contig, n_genomes, sp=None, mp=None, name_ranks=None, as_array=True):
    """sk_triangle_multi: one host process, one context per GPU (a device may repeat: the exchange then stays on it)."""
    sp = sp or sketch_params(); mp = mp or map_params()
    contig_off = np.ascontiguousarray(contig_off, np.uint64)
    goc = np.ascontiguousarray(genome_of_contig, np.uint32)
    arr = None if isinstance(bases, int) else _as_u8(bases)
    ptr = bases if arr is None else arr.ctypes.data
    nr = None if name_ranks is None else np.ascontiguousarray(name_ranks, np.uint64)
    hs = (C.c_void_p * len(ctxs))(*[c.h for c in ctxs])
    out = C.POINTER(AniResult)(); n = C.c_uint64(); st = TriangleStats()
    c0 = ctxs[0]
    c0.check(c0.L.sk_triangle_multi(hs, len(ctxs), ptr, contig_off.ctypes.data, len(goc), goc.ctypes.data, n_genomes, C.byref(sp), C.byref(mp),
                                    None if nr is None else nr.ctypes.data, C.byref(out), C.byref(n), C.byref(st)))
    return _take_results(c0, out, n, as_array), st


class SketchStore:
    """sk_sketch_store: sketches (with their k-mer tables) in pinned host memory, genome-indexed.  Sets added to it may be freed
    afterwards; gather() brings any ascending list of genomes back to a device set that chains, screens and exports exactly
    like the set that was added."""

    def __init__(self, sp=None):
        self.L = _lib.load()
        self.sp = sp or sketch_params()
        h = C.c_void_p()
        if self.L.sk_sketch_store_create(C.byref(self.sp), C.byref(h)) != 0:
            raise SkaniError("sk_sketch_store_create failed")
        self.h = h

    def add(self, sset):
        """Append the genomes of a device set (ids continue; name ranks continue after the store's largest)."""
        sset.ctx.check(self.L.sk_sketch_store_add(self.h, sset.h))

    def n_genomes(self):
        return self.L.sk_sketch_store_n_genomes(self.h)

    def __len__(self):
        return self.n_genomes()

    def genome_bytes(self, g):
        """Device bytes genome g takes in a working set."""
        return self.L.sk_sketch_store_genome_bytes(self.h, int(g))

    def set_name_ranks(self, ranks):
        r = np.ascontiguousarray(ranks, np.uint64)
        assert len(r) == self.n_genomes()
        if self.L.sk_sketch_store_set_name_ranks(self.h, r.ctypes.data if len(r) else None) != 0:
            raise SkaniError("sk_sketch_store_set_name_ranks failed")

    def gather(self, ctx, genomes=None, markers_only=False):
        """Device set on ctx holding `genomes` (ascending, no duplicates; None = all) in list order."""
        g = np.arange(self.n_genomes(), dtype=np.uint32) if genomes is None else np.ascontiguousarray(genomes, np.uint32)
        keep = g if len(g) else np.zeros(1, np.uint32)
        h = C.c_void_p()
        ctx.check(self.L.sk_sketch_store_gather(ctx.h, self.h, keep.ctypes.data, len(g), 1 if markers_only else 0, C.byref(h)))
        return SketchSet(ctx, h)

    def free(self):
        if self.h:
            self.L.sk_sketch_store_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def triangle_store(ctxs, store, mp=None, device_budget=0, as_array=True):
    """sk_triangle_store: the triangle of every genome of `store`, chained in working sets of at most device_budget bytes per
    context (0 = derived from free device memory).  ctxs: one Context or a list (two on one device overlap gather and chain).
    Returns (results sorted by (ref_id, query_id), StoreStats)."""
    ctxs = list(ctxs) if isinstance(ctxs, (list, tuple)) else [ctxs]
    mp = mp or map_params()
    hs = (C.c_void_p * len(ctxs))(*[c.h for c in ctxs])
    out = C.POINTER(AniResult)(); n = C.c_uint64(); st = StoreStats()
    c0 = ctxs[0]
    c0.check(c0.L.sk_triangle_store(hs, len(ctxs), store.h, C.byref(mp), int(device_budget), C.byref(out), C.byref(n), C.byref(st)))
    return _take_results(c0, out, n, as_array), st


def query_ref_store(ctxs, ref_store, query_store, mp=None, mode=0, device_budget=0, as_array=True):
    """sk_query_ref_store: screen_query_ref (mode 0-3) + chain_pairs of every reference of ref_store against every query of
    query_store (the same store may be both), chained in working sets of at most device_budget bytes per context (0 = derived
    from free device memory).  Both stores' name ranks are used as stored: rank both sides in one file-name order.
    Returns (results with ani > 0.1 sorted by (ref_id, query_id), StoreStats)."""
    ctxs = list(ctxs) if isinstance(ctxs, (list, tuple)) else [ctxs]
    mp = mp or map_params()
    hs = (C.c_void_p * len(ctxs))(*[None if c is None else c.h for c in ctxs])
    out = C.POINTER(AniResult)(); n = C.c_uint64(); st = StoreStats()
    c0 = ctxs[0]
    c0.check(c0.L.sk_query_ref_store(hs, len(ctxs), None if ref_store is None else ref_store.h, None if query_store is None else query_store.h,
                                     C.byref(mp), int(mode), int(device_budget), C.byref(out), C.byref(n), C.byref(st)))
    return _take_results(c0, out, n, as_array), st


NO_EDGE = np.uint64(0xFFFFFFFFFFFFFFFF)   # edge[g] of a representative (sk_cluster)


def cluster(ctx, n_genomes, results, rank, min_ani=0.95, single_linkage=False):
    """sk_cluster: ANI clustering of triangle results (a RESULT_DTYPE array, as as_array=True returns).  Edges are the rows with
    ani > 0.1 and ani >= min_ani; rank[g] is a permutation, rank 0 the first choice as a representative.  Greedy
    representatives by default, connected components with single_linkage.  Returns (rep, cluster, edge, stats): rep[g] and
    cluster[g] (representatives numbered in rank order), edge[g] = the index in results of the row joining g to rep[g] or
    NO_EDGE, and the ClusterStats."""
    res = np.ascontiguousarray(results)
    if res.dtype != RESULT_DTYPE:
        raise TypeError("results must be a RESULT_DTYPE array")
    rk = np.ascontiguousarray(rank, np.uint32)
    if len(rk) != n_genomes:
        raise ValueError("rank needs one entry per genome")
    n = max(int(n_genomes), 1)
    rep = np.zeros(n, np.uint32); cl = np.zeros(n, np.uint32); edge = np.zeros(n, np.uint64)
    cp = ClusterParams(float(min_ani), int(bool(single_linkage))); st = ClusterStats()
    ctx.check(ctx.L.sk_cluster(ctx.h, int(n_genomes), res.ctypes.data if len(res) else None, len(res), rk.ctypes.data if len(rk) else None,
                               C.byref(cp), rep.ctypes.data, cl.ctypes.data, edge.ctypes.data, C.byref(st)))
    return rep[:n_genomes], cl[:n_genomes], edge[:n_genomes], st


MERGE_DTYPE = np.dtype([("a", np.uint32), ("b", np.uint32), ("height", np.float64), ("size", np.uint64)])   # sk_merge
LINKAGE_METHODS = {"average": 0, "complete": 1}


def cluster_linkage(ctx, n_genomes, results, rank, method="average", min_ani=0.95, dendrogram=False):
    """sk_cluster_linkage: average (UPGMA) or complete linkage of triangle results (a RESULT_DTYPE array) over the rows with
    ani > 0.1, similarity 0 for pairs without a row; flat clusters at min_ani in (0.1, 1].  Returns (rep, cluster, edge, Z,
    stats) with rep / cluster / edge as cluster() defines them and Z, when dendrogram is set, the (n - 1, 4) float64 scipy
    linkage matrix (a, b, 1 - similarity, size) over genome indices; None otherwise."""
    if method not in LINKAGE_METHODS:
        raise ValueError("method must be 'average' or 'complete'")
    res = np.ascontiguousarray(results)
    if res.dtype != RESULT_DTYPE:
        raise TypeError("results must be a RESULT_DTYPE array")
    rk = np.ascontiguousarray(rank, np.uint32)
    if len(rk) != n_genomes:
        raise ValueError("rank needs one entry per genome")
    n = max(int(n_genomes), 1)
    rep = np.zeros(n, np.uint32); cl = np.zeros(n, np.uint32); edge = np.zeros(n, np.uint64)
    merges = np.zeros(max(n - 1, 1), MERGE_DTYPE) if dendrogram else None
    lp = LinkageParams(float(min_ani), LINKAGE_METHODS[method], int(bool(dendrogram))); st = ClusterStats()
    ctx.check(ctx.L.sk_cluster_linkage(ctx.h, int(n_genomes), res.ctypes.data if len(res) else None, len(res),
                                       rk.ctypes.data if len(rk) else None, C.byref(lp), rep.ctypes.data, cl.ctypes.data,
                                       edge.ctypes.data, None if merges is None else merges.ctypes.data, C.byref(st)))
    Z = None
    if dendrogram:
        m = merges[:max(int(n_genomes) - 1, 0)]
        Z = np.stack([m["a"].astype(np.float64), m["b"].astype(np.float64), m["height"], m["size"].astype(np.float64)], 1).reshape(-1, 4)
    return rep[:n_genomes], cl[:n_genomes], edge[:n_genomes], Z, st


NJ_JOIN_DTYPE = np.dtype([("a", np.uint32), ("b", np.uint32), ("len_a", np.float64), ("len_b", np.float64)])   # sk_nj_join


def neighbor_joining(ctx, n_genomes, results):
    """sk_neighbor_joining: the neighbour-joining tree of triangle results (a RESULT_DTYPE array) over the rows with ani > 0.1,
    distance 1 - ani, 1.0 for pairs without a row.  Returns (joins, stats): joins an NJ_JOIN_DTYPE array of n - 1 rows (a, b,
    len_a, len_b), nodes numbered the scipy way (leaves 0..n-1, row t creates n + t), the last row joining the final two nodes
    at half their distance each; stats the sk_nj_stats struct."""
    res = np.ascontiguousarray(results)
    if res.dtype != RESULT_DTYPE:
        raise TypeError("results must be a RESULT_DTYPE array")
    n = int(n_genomes)
    joins = np.zeros(max(n - 1, 1), NJ_JOIN_DTYPE)
    st = NjStats()
    ctx.check(ctx.L.sk_neighbor_joining(ctx.h, n, res.ctypes.data if len(res) else None, len(res), joins.ctypes.data, C.byref(st)))
    return joins[:max(n - 1, 0)], st


def neighbor_joining_multi(ctxs, n_genomes, results):
    """sk_neighbor_joining_multi: neighbor_joining with the distance matrix split over the contexts ctxs (one band of rows
    each).  Returns (joins, stats) equal to neighbor_joining(ctxs[0], ...)'s; errors are reported on ctxs[0]."""
    res = np.ascontiguousarray(results)
    if res.dtype != RESULT_DTYPE:
        raise TypeError("results must be a RESULT_DTYPE array")
    n = int(n_genomes)
    joins = np.zeros(max(n - 1, 1), NJ_JOIN_DTYPE)
    st = NjStats()
    hs = (C.c_void_p * len(ctxs))(*[None if c is None else c.h for c in ctxs])
    c0 = ctxs[0]
    c0.check(c0.L.sk_neighbor_joining_multi(hs, len(ctxs), n, res.ctypes.data if len(res) else None, len(res), joins.ctypes.data, C.byref(st)))
    return joins[:max(n - 1, 0)], st


def dereplicate(ctx, sset, rank, min_ani=0.95, mp=None, wave=0):
    """sk_dereplicate: greedy ANI dereplication of a sketch set, equal to cluster() (greedy) on the rows of screen_triangle +
    chain_pairs over the same set and mp, but screening and chaining only genome x representative pairs.  rank[g] is a
    permutation, rank 0 the first choice as a representative; wave = genomes per wave (0 = library default), which never
    changes the result.  Returns (rep, cluster, join, stats): join[g] is the chained row (RESULT_DTYPE) joining member g to
    rep[g], for a representative a row with ani = NaN and ref_id = query_id = g; stats the sk_derep_stats struct."""
    mp = mp or map_params()
    n = len(sset)
    rk = np.ascontiguousarray(rank, np.uint32)
    if len(rk) != n:
        raise ValueError("rank needs one entry per genome")
    m = max(n, 1)
    rep = np.zeros(m, np.uint32); cl = np.zeros(m, np.uint32); join = np.zeros(m, RESULT_DTYPE)
    dp = DerepParams(float(min_ani), int(wave)); st = DerepStats()
    ctx.check(ctx.L.sk_dereplicate(ctx.h, sset.h, C.byref(mp), rk.ctypes.data if n else None, C.byref(dp), rep.ctypes.data,
                                   cl.ctypes.data, join.ctypes.data, C.byref(st)))
    return rep[:n], cl[:n], join[:n], st


def dereplicate_store(ctxs, store, rank, min_ani=0.95, mp=None, wave=0, device_budget=0):
    """sk_dereplicate_store: dereplicate() over every genome of a SketchStore, with rep, cluster and join byte for byte what
    dereplicate() returns on one in-memory set of the same genomes and name ranks.  The markers are gathered on ctxs[0]; each
    chain step's pairs are chained in working sets of at most device_budget bytes per context (0 = derived from free device
    memory).  ctxs: one Context or a list (two on one device overlap gather and chain).  Returns (rep, cluster, join, stats,
    store_stats): stats the sk_derep_stats struct, store_stats the StoreStats summed over the chain steps."""
    ctxs = list(ctxs) if isinstance(ctxs, (list, tuple)) else [ctxs]
    mp = mp or map_params()
    n = store.n_genomes()
    rk = np.ascontiguousarray(rank, np.uint32)
    if len(rk) != n:
        raise ValueError("rank needs one entry per genome")
    m = max(n, 1)
    rep = np.zeros(m, np.uint32); cl = np.zeros(m, np.uint32); join = np.zeros(m, RESULT_DTYPE)
    dp = DerepParams(float(min_ani), int(wave)); st = DerepStats(); sst = StoreStats()
    hs = (C.c_void_p * len(ctxs))(*[c.h for c in ctxs])
    c0 = ctxs[0]
    c0.check(c0.L.sk_dereplicate_store(hs, len(ctxs), store.h, C.byref(mp), rk.ctypes.data if n else None, C.byref(dp), int(device_budget),
                                       rep.ctypes.data, cl.ctypes.data, join.ctypes.data, C.byref(st), C.byref(sst)))
    return rep[:n], cl[:n], join[:n], st, sst


def dereplicate_fixed(ctx, sset, rank, n_fixed, min_ani=0.95, mp=None, wave=0):
    """sk_dereplicate_fixed: dereplicate() with the genomes of rank < n_fixed fixed as representatives, equal to cluster()
    (greedy) on the rows of screen_triangle + chain_pairs without the rows between two fixed genomes.  No pair of two fixed
    genomes is screened or chained; n_fixed = 0 is dereplicate().  Returns (rep, cluster, join, stats) as dereplicate()."""
    mp = mp or map_params()
    n = len(sset)
    rk = np.ascontiguousarray(rank, np.uint32)
    if len(rk) != n:
        raise ValueError("rank needs one entry per genome")
    m = max(n, 1)
    rep = np.zeros(m, np.uint32); cl = np.zeros(m, np.uint32); join = np.zeros(m, RESULT_DTYPE)
    dp = DerepParams(float(min_ani), int(wave)); st = DerepStats()
    ctx.check(ctx.L.sk_dereplicate_fixed(ctx.h, sset.h, C.byref(mp), rk.ctypes.data if n else None, int(n_fixed), C.byref(dp),
                                         rep.ctypes.data, cl.ctypes.data, join.ctypes.data, C.byref(st)))
    return rep[:n], cl[:n], join[:n], st


def dereplicate_store_fixed(ctxs, store, rank, n_fixed, min_ani=0.95, mp=None, wave=0, device_budget=0):
    """sk_dereplicate_store_fixed: dereplicate_fixed() over every genome of a SketchStore, equal to dereplicate_fixed() on one
    in-memory set of the same genomes and name ranks; the contexts and device_budget as in dereplicate_store().  Returns
    (rep, cluster, join, stats, store_stats) as dereplicate_store()."""
    ctxs = list(ctxs) if isinstance(ctxs, (list, tuple)) else [ctxs]
    mp = mp or map_params()
    n = store.n_genomes()
    rk = np.ascontiguousarray(rank, np.uint32)
    if len(rk) != n:
        raise ValueError("rank needs one entry per genome")
    m = max(n, 1)
    rep = np.zeros(m, np.uint32); cl = np.zeros(m, np.uint32); join = np.zeros(m, RESULT_DTYPE)
    dp = DerepParams(float(min_ani), int(wave)); st = DerepStats(); sst = StoreStats()
    hs = (C.c_void_p * len(ctxs))(*[c.h for c in ctxs])
    c0 = ctxs[0]
    c0.check(c0.L.sk_dereplicate_store_fixed(hs, len(ctxs), store.h, C.byref(mp), rk.ctypes.data if n else None, int(n_fixed), C.byref(dp),
                                             int(device_budget), rep.ctypes.data, cl.ctypes.data, join.ctypes.data, C.byref(st), C.byref(sst)))
    return rep[:n], cl[:n], join[:n], st, sst
