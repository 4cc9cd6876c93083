"""skani_b200 -- H100 (sm_90a) CUDA implementation of skani's ANI hot path.

Host-side mirror of the reference's public API for the path (fastx_to_sketches -> screen -> chain_seeds,
reference tests/tests.rs:42-60) over the C ABI in include/skani_b200.h.  No CPU fallback exists."""
from .host import (Context, SketchSet, sketch_params, map_params, sketch_contigs, sketch_sequences,
                   screen_triangle, screen_triangle_rows, screen_triangle_block, screen_query_ref, chain_pairs, chain_pair_debug, chain_pairs_debug, triangle, import_sketches,
                   pack_contigs, sketch_contigs_2bit, triangle_local, triangle_multi, triangle_2bit,
                   screen_query_ref_multi, chain_pairs_multi, SketchStore, triangle_store)  # noqa: F401
