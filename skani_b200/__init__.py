"""skani_b200 -- H100 (sm_90a) CUDA implementation of skani's ANI hot path.

Host-side mirror of the reference's public API for the path (fastx_to_sketches -> screen -> chain_seeds,
reference tests/tests.rs:42-60) over the C ABI in include/skani_b200.h.  No CPU fallback exists."""
from .host import (Context, SketchSet, sketch_params, map_params, sketch_contigs, sketch_sequences,
                   screen_triangle, screen_triangle_rows, screen_triangle_block, screen_query_ref, RefIndex, chain_pairs, chain_pair_debug, chain_pairs_debug, triangle, import_sketches, import_blobs, BlobError,
                   pack_contigs, sketch_contigs_2bit, triangle_local, triangle_multi, triangle_2bit,
                   screen_query_ref_multi, chain_pairs_multi, SketchStore, triangle_store, query_ref_store, cluster, cluster_linkage, neighbor_joining, neighbor_joining_multi,
                   dereplicate, dereplicate_store, dereplicate_fixed, dereplicate_store_fixed, chain_pairs_mappings, chain_pairs_multi_mappings, MAPPING_DTYPE)  # noqa: F401
