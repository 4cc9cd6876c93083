"""ctypes loader for libskani_b200.so (the CUDA product library).  There is no CPU fallback: if the
library is missing or no CUDA device is usable, importing/creating a context raises."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libskani_b200.so")


class SketchParams(C.Structure):
    _fields_ = [("c", C.c_uint32), ("k", C.c_uint32), ("marker_c", C.c_uint32)]


class MapParams(C.Structure):
    _fields_ = [("screen_val", C.c_double), ("min_aligned_frac", C.c_double), ("both_min_aligned_frac", C.c_double),
                ("robust", C.c_int32), ("median", C.c_int32), ("learned_ani", C.c_int32), ("rescue_small", C.c_int32)]


class AniResult(C.Structure):
    _fields_ = [(n, C.c_float) for n in
                ("ani", "af_query", "af_ref", "ci_lower", "ci_upper", "std",
                 "q90_q", "q90_r", "q50_q", "q50_r", "q10_q", "q10_r")] + \
               [(n, C.c_uint32) for n in
                ("num_contigs_q", "num_contigs_r", "avg_chain_int_len", "total_bases_covered", "ref_id", "query_id")]


class ChainDebug(C.Structure):
    _fields_ = [("result", AniResult), ("switched", C.c_int32),
                ("n_anchors", C.c_uint64), ("n_chunks", C.c_uint64), ("n_intervals", C.c_uint64), ("n_ests", C.c_uint64),
                ("anchors", C.POINTER(C.c_uint32)), ("chunk_first", C.POINTER(C.c_uint32)),
                ("chunk_nseeds", C.POINTER(C.c_uint32)), ("score", C.POINTER(C.c_int64)),
                ("pointer", C.POINTER(C.c_uint32)), ("intervals", C.POINTER(C.c_int64)),
                ("est", C.POINTER(C.c_double)), ("weight", C.POINTER(C.c_uint64)), ("chunk_stats", C.POINTER(C.c_uint32))]


class TriangleStats(C.Structure):
    _fields_ = [("t_sketch", C.c_double), ("t_screen", C.c_double), ("t_chain", C.c_double), ("t_total", C.c_double),
                ("n_pairs_screened", C.c_uint64), ("n_pairs_kept", C.c_uint64)]


class StoreStats(C.Structure):
    _fields_ = [("n_working_sets", C.c_uint32), ("n_split_components", C.c_uint32), ("gathered_bytes", C.c_uint64),
                ("max_working_set_bytes", C.c_uint64), ("t_screen", C.c_double), ("t_gather", C.c_double), ("t_chain", C.c_double)]


# every symbol include/skani_b200.h declares: (name, restype, argtypes)
vp, u64, u32, i32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int
PP = C.POINTER
SYMBOLS = [
    ("sk_device_count", i32, []),
    ("sk_device_memory", i32, [i32, PP(u64), PP(u64)]),
    ("sk_ctx_create", i32, [i32, PP(vp)]),
    ("sk_ctx_destroy", i32, [vp]),
    ("sk_ctx_set_seeding_semantics", i32, [vp, i32]),
    ("sk_last_error", C.c_char_p, [vp]),
    ("sk_ctx_launch_count", u64, [vp]),
    ("sk_ctx_stream", vp, [vp]),
    ("sk_ctx_set_timing", i32, [vp, i32]),
    ("sk_ctx_get_timing", i32, [vp, C.c_char_p, u64, i32]),
    ("sk_sketch_batch", i32, [vp, vp, vp, u32, vp, u32, PP(SketchParams), PP(vp)]),
    ("sk_pack_contig", i32, [vp, u64, vp, vp]),
    ("sk_pack_impl", C.c_char_p, []),
    ("sk_sketch_batch_2bit", i32, [vp, vp, vp, vp, u32, vp, u32, PP(SketchParams), PP(vp)]),
    ("sk_ctx_last_pack_share", C.c_double, [vp]),
    ("sk_sketch_batch_dev", i32, [vp, vp, vp, u32, vp, u32, PP(SketchParams), PP(vp)]),
    ("sk_sketch_set_free", i32, [vp]),
    ("sk_sketch_set_append", i32, [vp, vp]),
    ("sk_sketch_set_n_genomes", u32, [vp]),
    ("sk_sketch_set_genome_info", i32, [vp, u32, PP(u64), PP(u64), PP(u64), PP(u64), PP(u64)]),
    ("sk_sketch_set_export", i32, [vp, u32, vp, vp, vp, vp, vp]),
    ("sk_sketch_set_import", i32, [vp, PP(SketchParams), vp, vp, vp, u64, vp, u64, vp, u32, PP(vp)]),
    ("sk_sketch_set_import_batch", i32, [vp, PP(SketchParams), u32, vp, vp, vp, vp, vp, vp, vp, vp, vp, PP(vp)]),
    ("sk_sketch_set_blob_size", i32, [vp, PP(u64), PP(u64)]),
    ("sk_sketch_set_pack", i32, [vp, vp, vp]),
    ("sk_sketch_set_unpack", i32, [vp, u32, vp, vp, PP(vp)]),
    ("sk_sketch_set_subset_blob_size", i32, [vp, vp, u32, i32, PP(u64), PP(u64)]),
    ("sk_sketch_set_pack_subset", i32, [vp, vp, u32, i32, vp, vp]),
    ("sk_screen_triangle", i32, [vp, vp, PP(MapParams), PP(PP(u64)), PP(u64)]),
    ("sk_screen_triangle_rows", i32, [vp, vp, PP(MapParams), u32, u32, PP(PP(u64)), PP(u64)]),
    ("sk_screen_triangle_block", i32, [vp, vp, u32, u32, PP(MapParams), PP(PP(u64)), PP(u64)]),
    ("sk_screen_query_ref", i32, [vp, vp, vp, PP(MapParams), i32, PP(PP(u64)), PP(u64)]),
    ("sk_free", None, [vp]),
    ("sk_chain_pairs", i32, [vp, vp, vp, vp, u64, PP(MapParams), vp]),
    ("sk_sketch_set_set_name_ranks", i32, [vp, vp]),
    ("sk_chain_pair_debug", i32, [vp, vp, vp, u64, PP(MapParams), PP(ChainDebug)]),
    ("sk_chain_pairs_debug", i32, [vp, vp, vp, vp, u64, PP(MapParams), vp]),
    ("sk_chain_debug_free", None, [PP(ChainDebug)]),
    ("sk_debug_chunk_estimate", i32, [vp, u64, vp, u32, u32, vp, vp, vp]),
    ("sk_debug_chain_anchors", i32, [vp, u32, u32, u64, vp, vp, vp, vp, vp, vp]),
    ("sk_debug_select_intervals", i32, [vp, u32, u32, u64, vp, vp, vp, vp, vp, vp]),
    ("sk_triangle", i32, [vp, vp, vp, u32, vp, u32, PP(SketchParams), PP(MapParams), PP(PP(AniResult)), PP(u64),
                          PP(TriangleStats)]),
    ("sk_triangle_local", i32, [vp, vp, vp, u32, vp, u32, PP(SketchParams), PP(MapParams), vp, PP(PP(AniResult)), PP(u64),
                                PP(TriangleStats), PP(vp)]),
    ("sk_triangle_2bit", i32, [vp, vp, vp, vp, u32, vp, u32, PP(SketchParams), PP(MapParams), vp, PP(PP(AniResult)), PP(u64),
                               PP(TriangleStats), PP(vp)]),
    ("sk_triangle_multi", i32, [vp, u32, vp, vp, u32, vp, u32, PP(SketchParams), PP(MapParams), vp, PP(PP(AniResult)), PP(u64),
                                PP(TriangleStats)]),
    ("sk_sketch_set_copy", i32, [vp, vp, PP(vp)]),
    ("sk_screen_query_ref_multi", i32, [vp, u32, vp, vp, vp, PP(MapParams), i32, PP(PP(u64)), PP(u64)]),
    ("sk_chain_pairs_multi", i32, [vp, u32, vp, vp, vp, vp, u64, PP(MapParams), vp]),
    ("sk_sketch_store_create", i32, [PP(SketchParams), PP(vp)]),
    ("sk_sketch_store_add", i32, [vp, vp]),
    ("sk_sketch_store_n_genomes", u32, [vp]),
    ("sk_sketch_store_genome_bytes", u64, [vp, u32]),
    ("sk_sketch_store_set_name_ranks", i32, [vp, vp]),
    ("sk_sketch_store_gather", i32, [vp, vp, vp, u32, i32, PP(vp)]),
    ("sk_sketch_store_free", i32, [vp]),
    ("sk_triangle_store", i32, [vp, u32, vp, PP(MapParams), u64, PP(PP(AniResult)), PP(u64), PP(StoreStats)]),
    ("sk_query_ref_store", i32, [vp, u32, vp, vp, PP(MapParams), i32, u64, PP(PP(AniResult)), PP(u64), PP(StoreStats)]),
]

_lib = None


def load():
    """Load the shared library and bind every declared symbol (raises if the .so or a symbol is missing)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError("libskani_b200.so not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    for name, res, args in SYMBOLS:
        fn = getattr(L, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L
