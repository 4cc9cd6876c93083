"""ctypes binding of the CPU oracle (oracle/liboracle.so).  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
LIB_PATH = os.path.join(ORACLE_DIR, "liboracle.so")


class OrcResult(C.Structure):
    _fields_ = [(n, C.c_float) for n in
                ("ani", "af_query", "af_ref", "ci_lower", "ci_upper", "std",
                 "q90_q", "q90_r", "q50_q", "q50_r", "q10_q", "q10_r")] + \
               [(n, C.c_uint32) for n in
                ("num_contigs_q", "num_contigs_r", "avg_chain_int_len", "total_bases_covered", "ref_id", "query_id")]


class OrcCmd(C.Structure):
    _fields_ = [("screen_val", C.c_double), ("min_aligned_frac", C.c_double), ("both_min_aligned_frac", C.c_double),
                ("robust", C.c_int32), ("median", C.c_int32), ("learned_ani", C.c_int32), ("rescue_small", C.c_int32)]


def cmd(screen_val=0.0, min_af=0.15, both_min_af=-0.01, robust=False, median=False, learned_ani=True,
        rescue_small=True):
    return OrcCmd(screen_val, min_af, both_min_af, int(robust), int(median), int(learned_ani), int(rescue_small))


_lib = None


def build():
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR])


def build_native(out_dir):
    """-march=native build for the CPU baseline (out_dir/liboracle.so); returns its path or None."""
    try:
        subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "native", "NATIVE_DIR=" + os.path.abspath(out_dir)])
        return os.path.join(out_dir, "liboracle.so")
    except Exception:
        return None


def use_library(path):
    """Bind a specific build of the oracle (bench.py --impl reference: the -march=native one). Call before lib()."""
    global LIB_PATH, _lib
    LIB_PATH, _lib = path, None


def set_avx2_intrinsics(on=True):
    """Seeding with the reference's 4-lane AVX2 instruction mix (baseline timing); returns whether it is active."""
    return bool(lib().orc_set_avx2_intrinsics(int(on)))


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        build()
    L = C.CDLL(LIB_PATH)
    vp, u64, u32, i32, dbl = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_double
    L.orc_mm_hash64.restype = u64; L.orc_mm_hash64.argtypes = [u64]
    L.orc_set_avx2_intrinsics.restype = i32; L.orc_set_avx2_intrinsics.argtypes = [i32]
    L.orc_sketch_files.restype = i32
    L.orc_sketch_files.argtypes = [C.POINTER(C.c_char_p), i32, u64, u64, u64, i32, i32, i32,
                                   C.POINTER(C.POINTER(vp)), C.POINTER(i32), C.POINTER(i32)]
    L.orc_free_array.argtypes = [vp]
    L.orc_sketch_from_contigs.restype = vp
    L.orc_sketch_from_contigs.argtypes = [C.c_char_p, vp, vp, u32, u64, u64, u64, i32]
    L.orc_sketch_free.argtypes = [vp]
    L.orc_sketch_many.restype = i32
    L.orc_sketch_many.argtypes = [vp, vp, vp, u32, u32, u64, u64, u64, i32, C.POINTER(vp)]
    L.orc_seed_one_contig.restype = vp
    L.orc_seed_one_contig.argtypes = [vp, u64, u64, u64, u64, i32]
    L.orc_time_seeding.restype = dbl
    L.orc_time_seeding.argtypes = [vp, vp, u32, u64, u64, u64, i32]
    for f in ("n_records", "n_kmers", "n_markers", "n_contigs", "total_len", "contig_order"):
        fn = getattr(L, "orc_sketch_" + f); fn.restype = u64; fn.argtypes = [vp]
    L.orc_sketch_file_name.restype = C.c_char_p; L.orc_sketch_file_name.argtypes = [vp]
    L.orc_sketch_contig_name.restype = C.c_char_p; L.orc_sketch_contig_name.argtypes = [vp, u64]
    L.orc_sketch_export.argtypes = [vp] * 6
    L.orc_check_markers_quickly.restype = i32; L.orc_check_markers_quickly.argtypes = [vp, vp, dbl, i32]
    L.orc_screen_triangle.restype = i32
    L.orc_screen_triangle.argtypes = [C.POINTER(vp), i32, dbl, i32, C.POINTER(C.POINTER(u64)), C.POINTER(C.POINTER(u32))]
    L.orc_sketches_from_markers.restype = i32
    L.orc_sketches_from_markers.argtypes = [i32, vp, vp, C.POINTER(vp)]
    L.orc_screen_query_ref.restype = i32
    L.orc_screen_query_ref.argtypes = [C.POINTER(vp), i32, C.POINTER(vp), i32, dbl, i32, i32, C.POINTER(C.POINTER(u64)), C.POINTER(u64)]
    L.orc_chain.restype = i32; L.orc_chain.argtypes = [vp, vp, C.POINTER(OrcCmd), C.POINTER(OrcResult)]
    L.orc_chain_debug.restype = vp; L.orc_chain_debug.argtypes = [vp, vp, C.POINTER(OrcCmd)]
    L.orc_debug_free.argtypes = [vp]
    L.orc_debug_result.argtypes = [vp, C.POINTER(OrcResult)]
    L.orc_debug_switched.restype = i32; L.orc_debug_switched.argtypes = [vp]
    for f in ("n_anchors", "n_chunks", "n_intervals", "n_ests"):
        fn = getattr(L, "orc_debug_" + f); fn.restype = u64; fn.argtypes = [vp]
    L.orc_debug_anchors.argtypes = [vp] * 4
    L.orc_debug_chunks.argtypes = [vp] * 3
    L.orc_debug_intervals.argtypes = [vp] * 2
    L.orc_debug_ests.argtypes = [vp] * 3
    L.orc_debug_chunk_stats.argtypes = [vp] * 2
    L.orc_chunk_estimate.restype = i32
    L.orc_chunk_estimate.argtypes = [u64, vp, u32, u32, vp, vp, vp]
    L.orc_chain_chunks.restype = i32
    L.orc_chain_chunks.argtypes = [u32, u32, i32, u64, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.orc_select_intervals.restype = i32
    L.orc_select_intervals.argtypes = [u32, u32, i32, u64, u64, vp, vp, vp, vp, vp]
    L.orc_gbdt_predict.restype = C.c_float; L.orc_gbdt_predict.argtypes = [i32, vp]
    L.orc_final_estimate.restype = i32
    L.orc_final_estimate.argtypes = [vp, vp, u64, u32, u32, u64, u64, vp, vp, C.POINTER(OrcCmd), i32, C.POINTER(OrcResult)]
    L.orc_triangle.restype = i32
    L.orc_triangle.argtypes = [C.POINTER(vp), i32, C.POINTER(OrcCmd), i32, C.POINTER(C.POINTER(OrcResult)),
                               C.POINTER(u64), C.POINTER(u64), C.POINTER(dbl), C.POINTER(dbl)]
    for f in ("orc_dist", "orc_search"):
        fn = getattr(L, f); fn.restype = i32
        fn.argtypes = [C.POINTER(vp), i32, C.POINTER(vp), i32, C.POINTER(OrcCmd), i32, i32,
                       C.POINTER(C.POINTER(OrcResult)), C.POINTER(u64)]
    _lib = L
    return L


class Sketch:
    def __init__(self, handle):
        self.h = C.c_void_p(handle)

    def __del__(self):
        try:
            lib().orc_sketch_free(self.h)
        except Exception:
            pass

    @property
    def file_name(self): return lib().orc_sketch_file_name(self.h).decode()
    def contig_name(self, i=0): return lib().orc_sketch_contig_name(self.h, i).decode()
    @property
    def n_records(self): return lib().orc_sketch_n_records(self.h)
    @property
    def n_kmers(self): return lib().orc_sketch_n_kmers(self.h)
    @property
    def n_markers(self): return lib().orc_sketch_n_markers(self.h)
    @property
    def n_contigs(self): return lib().orc_sketch_n_contigs(self.h)
    @property
    def total_len(self): return lib().orc_sketch_total_len(self.h)

    def export(self):
        n, m, nc = self.n_records, self.n_markers, self.n_contigs
        kmer = np.zeros(n, np.uint32); pos = np.zeros(n, np.uint32); cc = np.zeros(n, np.uint32)
        mk = np.zeros(m, np.uint64); cl = np.zeros(nc, np.uint32)
        lib().orc_sketch_export(self.h, kmer.ctypes.data, pos.ctypes.data, cc.ctypes.data, mk.ctypes.data, cl.ctypes.data)
        return dict(kmer=kmer, pos=pos, cc=cc, markers=mk, contig_lengths=cl)


def sketch_files(paths, c=125, k=15, marker_c=1000, individual=False, avx2sem=True, threads=4):
    L = lib()
    arr = (C.c_char_p * len(paths))(*[p.encode() for p in paths])
    out = C.POINTER(C.c_void_p)(); n = C.c_int(); nw = C.c_int()
    rc = L.orc_sketch_files(arr, len(paths), c, k, marker_c, int(individual), int(avx2sem), threads,
                            C.byref(out), C.byref(n), C.byref(nw))
    if rc != 0:
        raise ValueError("orc_sketch_files rc=%d" % rc)
    sk = [Sketch(out[i]) for i in range(n.value)]
    L.orc_free_array(out)
    return sk, nw.value


def sketch_from_contigs(name, seqs, c=125, k=15, marker_c=1000, avx2sem=True):
    """seqs: list of bytes/np.uint8 arrays (ASCII)."""
    arrs = [np.frombuffer(s, np.uint8) if isinstance(s, (bytes, bytearray)) else np.asarray(s, np.uint8) for s in seqs]
    off = np.zeros(len(arrs) + 1, np.uint64)
    off[1:] = np.cumsum([len(a) for a in arrs])
    buf = np.concatenate(arrs) if arrs else np.zeros(0, np.uint8)
    buf = np.ascontiguousarray(buf)
    h = lib().orc_sketch_from_contigs(name.encode(), buf.ctypes.data, off.ctypes.data, len(arrs), c, k, marker_c, int(avx2sem))
    return Sketch(h)


def sketch_many(bases, contig_off, genome_of_contig, n_genomes, c=125, k=15, marker_c=1000, threads=4):
    """Oracle sketches of genomes laid out like sk_sketch_batch's input; OpenMP threads over genomes."""
    bases = np.ascontiguousarray(bases, np.uint8)
    off = np.ascontiguousarray(contig_off, np.uint64); goc = np.ascontiguousarray(genome_of_contig, np.uint32)
    out = (C.c_void_p * n_genomes)()
    lib().orc_sketch_many(bases.ctypes.data, off.ctypes.data, goc.ctypes.data, len(goc), n_genomes, c, k, marker_c, threads, out)
    return [Sketch(out[i]) for i in range(n_genomes)]


def chain(ref, query, cp=None):
    cp = cp or cmd()
    r = OrcResult()
    lib().orc_chain(ref.h, query.h, C.byref(cp), C.byref(r))
    return r


def chain_debug(ref, query, cp=None):
    cp = cp or cmd()
    L = lib()
    d = C.c_void_p(L.orc_chain_debug(ref.h, query.h, C.byref(cp)))
    try:
        res = OrcResult(); L.orc_debug_result(d, C.byref(res))
        na, nc, ni, ne = (L.orc_debug_n_anchors(d), L.orc_debug_n_chunks(d), L.orc_debug_n_intervals(d), L.orc_debug_n_ests(d))
        a5 = np.zeros((na, 5), np.uint32); score = np.zeros(na, np.int64); ptr = np.zeros(na, np.uint32)
        L.orc_debug_anchors(d, a5.ctypes.data, score.ctypes.data, ptr.ctypes.data)
        first = np.zeros(nc + 1, np.uint32); nseeds = np.zeros(nc, np.uint32)
        if nc:
            L.orc_debug_chunks(d, first.ctypes.data, nseeds.ctypes.data)
        iv = np.zeros((ni, 11), np.int64)
        L.orc_debug_intervals(d, iv.ctypes.data)
        est = np.zeros(ne, np.float64); w = np.zeros(ne, np.uint64)
        L.orc_debug_ests(d, est.ctypes.data, w.ctypes.data)
        cs = np.zeros((nc, 9), np.uint32)
        L.orc_debug_chunk_stats(d, cs.ctypes.data)
        return dict(result=res, switched=bool(L.orc_debug_switched(d)), anchors=a5, score=score, pointer=ptr,
                    chunk_first=first, chunk_nseeds=nseeds, intervals=iv, est=est, weight=w, chunk_stats=cs)
    finally:
        L.orc_debug_free(d)


def final_estimate(est, weight, total_bases_covered, avg_chain_int_len, query_total_len, ref_total_len, quant_q, quant_r,
                   cp=None, model=0):
    """The final estimate (trimmed mean, std, bootstrap CI, AF cutoffs, learned ANI) of a sorted (est, weight) list, as
    calculate_ani + predict_from_ani_res compute it; quant_q / quant_r = (q10, q50, q90); model -1 none, 0 C125, 1 C200.
    num_contigs_* of the result are 0."""
    cp = cp or cmd()
    e = np.ascontiguousarray(est, np.float64)
    w = np.ascontiguousarray(weight, np.uint64)
    assert len(e) == len(w)
    qq = np.ascontiguousarray(quant_q, np.float32); qr = np.ascontiguousarray(quant_r, np.float32)
    r = OrcResult()
    lib().orc_final_estimate(e.ctypes.data, w.ctypes.data, len(e), int(total_bases_covered), int(avg_chain_int_len),
                             int(query_total_len), int(ref_total_len), qq.ctypes.data, qr.ctypes.data, C.byref(cp), model,
                             C.byref(r))
    return r


def chunk_estimate(inputs, c, k):
    """The oracle's chunk_estimate over rows (total_anchors, rq0, rq1, tbcq, n_int, n_seeds, num_in, upper_lower): (est f64,
    weight u32, valid u32: 0 no estimate, 1 estimate, 3 estimate with the putative-ANI filter applied)."""
    x = np.ascontiguousarray(inputs, np.uint32).reshape(-1, 8)
    n = len(x)
    est = np.zeros(max(n, 1), np.float64); w = np.zeros(max(n, 1), np.uint32); v = np.zeros(max(n, 1), np.uint32)
    lib().orc_chunk_estimate(n, x.ctypes.data, c, k, est.ctypes.data, w.ctypes.data, v.ctypes.data)
    return est[:n], w[:n], v[:n]


def _selection(iv, hits, acc, sums):
    return dict(intervals=iv, hits=hits, chunk_acc=acc, pair_sumlen=int(sums[0]), pair_nchains=int(sums[1]))


def chain_chunks(chunks, c, k, switched=False):
    """chain_anchors_ani + get_chain_intervals + get_nonoverlapping_chains on given chunks of one pair (each an (n, 5) array
    of (query_contig, query_pos, ref_contig, ref_pos, reverse), sorted as get_anchors sorts them).  Returns score (i64) and
    chunk-local pointer per anchor, the sorted intervals (n, 11: the chain_debug fields with kept), hits (n, 2: kept
    intervals overlapping each one on the ref / query axis), chunk_acc (per chunk: total_anchors, rq0, rq1, tbcq, n_int) and
    the pair's pair_sumlen / pair_nchains (avg_chain_int_len = sumlen / nchains)."""
    chunks = [np.asarray(ch, np.uint32).reshape(-1, 5) for ch in chunks]
    off = np.zeros(len(chunks) + 1, np.uint64); off[1:] = np.cumsum([len(ch) for ch in chunks])
    a = np.ascontiguousarray(np.concatenate(chunks) if chunks else np.zeros((1, 5), np.uint32))
    na, nc = int(off[-1]), len(chunks)
    cap = na // 3 + 1
    score = np.zeros(max(na, 1), np.int64); ptr = np.zeros(max(na, 1), np.uint32)
    iv = np.zeros((cap, 11), np.int64); hits = np.zeros((cap, 2), np.uint32)
    acc = np.zeros((max(nc, 1), 5), np.uint32); sums = np.zeros(2, np.uint32); n_iv = C.c_uint64()
    lib().orc_chain_chunks(c, k, int(switched), nc, off.ctypes.data, a.ctypes.data, score.ctypes.data, ptr.ctypes.data,
                           iv.ctypes.data, hits.ctypes.data, C.byref(n_iv), acc.ctypes.data, sums.ctypes.data)
    n = n_iv.value
    return dict(score=score[:na], pointer=ptr[:na], **_selection(iv[:n], hits[:n], acc[:nc], sums))


def select_intervals(intervals, n_chunks, c, k, switched=False):
    """get_nonoverlapping_chains on given intervals ((n, 10): score, num_anchors, q0, q1, r0, r1, ref_contig, query_contig,
    chunk, reverse) of one pair with n_chunks chunks; outputs as chain_chunks without score / pointer."""
    x = np.ascontiguousarray(np.asarray(intervals, np.int64).reshape(-1, 10))
    n = len(x)
    iv = np.zeros((max(n, 1), 11), np.int64); hits = np.zeros((max(n, 1), 2), np.uint32)
    acc = np.zeros((max(n_chunks, 1), 5), np.uint32); sums = np.zeros(2, np.uint32)
    lib().orc_select_intervals(c, k, int(switched), n_chunks, n, x.ctypes.data, iv.ctypes.data, hits.ctypes.data,
                               acc.ctypes.data, sums.ctypes.data)
    return _selection(iv[:n], hits[:n], acc[:n_chunks], sums)


def _results(out, n):
    res = [OrcResult.from_buffer_copy(out[i]) for i in range(n.value)]
    lib().orc_free_array(out)
    return res


def triangle(sketches, cp=None, threads=4):
    cp = cp or cmd()
    L = lib()
    hs = (C.c_void_p * len(sketches))(*[s.h for s in sketches])
    out = C.POINTER(OrcResult)(); n = C.c_uint64(); nch = C.c_uint64(); ts = C.c_double(); tc = C.c_double()
    L.orc_triangle(hs, len(sketches), C.byref(cp), threads, C.byref(out), C.byref(n), C.byref(nch), C.byref(ts), C.byref(tc))
    return _results(out, n), dict(n_chained=nch.value, t_screen=ts.value, t_chain=tc.value)


def _qr(fn, refs, queries, cp, use_index, threads):
    cp = cp or cmd()
    hr = (C.c_void_p * len(refs))(*[s.h for s in refs])
    hq = (C.c_void_p * len(queries))(*[s.h for s in queries])
    out = C.POINTER(OrcResult)(); n = C.c_uint64()
    fn(hr, len(refs), hq, len(queries), C.byref(cp), int(use_index), threads, C.byref(out), C.byref(n))
    return _results(out, n)


def dist(refs, queries, cp=None, use_index=False, threads=4):
    return _qr(lib().orc_dist, refs, queries, cp, use_index, threads)


def search(refs, queries, cp=None, use_index=False, threads=4):
    return _qr(lib().orc_search, refs, queries, cp, use_index, threads)


def screen_triangle(sketches, screen_val=0.0, rescue_small=True):
    L = lib()
    hs = (C.c_void_p * len(sketches))(*[s.h for s in sketches])
    ro = C.POINTER(C.c_uint64)(); cols = C.POINTER(C.c_uint32)()
    L.orc_screen_triangle(hs, len(sketches), screen_val, int(rescue_small), C.byref(ro), C.byref(cols))
    n = len(sketches)
    row_off = np.ctypeslib.as_array(ro, shape=(n + 1,)).astype(np.uint64)
    c = np.ctypeslib.as_array(cols, shape=(int(row_off[-1]),)).astype(np.uint32) if row_off[-1] else np.zeros(0, np.uint32)
    L.orc_free_array(ro); L.orc_free_array(cols)
    return row_off, c


def sketches_from_markers(mk_off, markers):
    """Markers-only oracle sketches, built in one call: genome g holds markers[mk_off[g]:mk_off[g + 1]]."""
    n = len(mk_off) - 1
    off = np.ascontiguousarray(mk_off, np.uint64)
    mk = np.ascontiguousarray(np.concatenate([np.asarray(markers, np.uint64), np.zeros(1, np.uint64)]))
    out = (C.c_void_p * max(n, 1))()
    lib().orc_sketches_from_markers(n, off.ctypes.data, mk.ctypes.data, out)
    return [Sketch(out[i]) for i in range(n)]


def screen_query_ref(refs, queries, screen_val=0.0, mode=0, rescue_small=True):
    """Sorted (ref << 32 | query) list of the query x ref screen in mode 0-3 (see orc_screen_query_ref)."""
    L = lib()
    hr = (C.c_void_p * max(len(refs), 1))(*[s.h for s in refs])
    hq = (C.c_void_p * max(len(queries), 1))(*[s.h for s in queries])
    pp = C.POINTER(C.c_uint64)(); n = C.c_uint64()
    rc = L.orc_screen_query_ref(hr, len(refs), hq, len(queries), screen_val, mode, int(rescue_small), C.byref(pp), C.byref(n))
    if rc != 0:
        raise ValueError("orc_screen_query_ref rc=%d" % rc)
    arr = np.ctypeslib.as_array(pp, shape=(n.value,)).copy() if n.value else np.zeros(0, np.uint64)
    L.orc_free_array(pp)
    return arr


def screen_triangle_pairs(sketches, screen_val=0.0, rescue_small=True):
    """screen_triangle as a sorted (i << 32 | j) list, the form sk_screen_triangle returns."""
    row_off, cols = screen_triangle(sketches, screen_val, rescue_small)
    rows = np.repeat(np.arange(len(sketches), dtype=np.uint64), np.diff(row_off).astype(np.int64))
    return np.sort((rows << np.uint64(32)) | cols.astype(np.uint64))
