"""GPU parity of the chain front end's compacted hit stream against the CPU oracle, per pair and bit-exact through
sk_chain_pairs_debug: pairs whose query-role hits are sparse (one step's 1,024 hits span many probe tiles), dense (every record of a tile hits), or few and ending at the genome's last record, through the hash-table
probe and the bucket-search probe.  Each case asserts from the data that it reached its edge."""
import numpy as np
import pytest

from chain_testlib import make_sets, rand_seq
from test_gpu_chain_batch import check_batch, record_index, roles

pytestmark = pytest.mark.gpu
TILE = 1024                     # query-role records per probe tile, hit records per chunk_anchor_kernel step


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def hit_genomes():
    rng = np.random.default_rng(20261017)
    base = rand_seq(rng, 1_500_000)
    same = base.copy()                                    # every record hits: full tiles
    sparse = rand_seq(rng, len(base))                     # 4 kb of `base` every 20 kb: a step's hits span many tiles
    for p in range(0, len(base), 20_000):
        sparse[p:p + 4_000] = base[p:p + 4_000]
    # only the first and last 3 kb shared, 1 Mbp of other sequence between: few hits, the last on the last record
    tail = np.concatenate([base[:3_000], rand_seq(rng, 1_000_000), base[-3_000:]])
    return [[base], [same], [sparse], [tail]]


@pytest.mark.parametrize("env", [{}, {"SK_FORCE_BUCKET_PROBE": "1"}], ids=["hash_probe", "bucket_probe"])
def test_hit_stream_edges_bit_exact(ctx, monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    kw = dict(c=125, k=15, marker_c=1000)
    gs, osk = make_sets(ctx, hit_genomes(), kw)
    pairs = [(0, 1), (1, 0), (0, 2), (2, 0), (0, 3), (3, 0)]
    gds = check_batch(ctx, gs, osk, pairs)
    full_tile = multi_tile_step = last_record = 0
    for (r, q), gd in zip(pairs, gds):
        if not len(gd["anchors"]):
            continue
        qr, _ = roles(gd, r, q)
        exp = osk[qr].export()
        ri = np.unique(record_index(exp, gd["anchors"]))     # hit records, in record order
        n_rec = len(exp["pos"])
        per_tile = np.bincount(ri // TILE, minlength=(n_rec + TILE - 1) // TILE)
        full_tile += int(np.any(per_tile == TILE))
        step_tiles = ri[::TILE] // TILE                      # probe tile of the first hit of every step
        last_tiles = ri[TILE - 1::TILE] // TILE
        multi_tile_step += int(np.any(last_tiles - step_tiles[:len(last_tiles)] > 4))
        last_record += int(ri[-1] == n_rec - 1 and len(ri) < TILE)   # one partial step ending at the last record
    assert full_tile >= 1, "no probe tile in which every record hits"
    assert multi_tile_step >= 1, "no step whose hits span several probe tiles"
    assert last_record >= 1, "no pair with fewer than 1,024 hits whose last hit is its last record"
