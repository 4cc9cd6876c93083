"""dp_group_kernel on chunks of DP_SMEM_ANCHORS - 1, DP_SMEM_ANCHORS and DP_SMEM_ANCHORS + 1 anchors sharing warps (the
largest chunks on chip next to ones that keep their chain bookkeeping in global memory), under every group-kernel
instantiation sk_chain_pairs can choose: score and pointer of every anchor, every interval with its kept flag and the
per-chunk and per-pair sums equal the oracle's.  See tests/test_emu_dp_onchip.py for the emulated edges."""
import numpy as np
import pytest

import oracle_py as O
from test_emu_dp_onchip import bound_chunks, dp_smem_anchors
from test_gpu_dp_select import CONFIGS, compare_selection

pytestmark = pytest.mark.gpu
K = 15
GROUP = [cfg for cfg in CONFIGS if cfg[3].startswith("group")]


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("c,hooks,band,kernel", GROUP, ids=["c%d_%s" % (c, k.replace(" ", "_")) for c, _, _, k in GROUP])
def test_dp_onchip_bound_against_oracle(ctx, monkeypatch, c, hooks, band, kernel):
    import skani_b200 as sk
    for var in ("SK_DP_GL", "SK_DP_WARP", "SK_DP_MINB"):
        monkeypatch.delenv(var, raising=False)
    for var, v in hooks.items():
        monkeypatch.setenv(var, v)
    bound = dp_smem_anchors()
    chunks = bound_chunks(bound, seed=c)
    assert {len(x) for x in chunks} >= {bound - 1, bound, bound + 1}
    pairs = [chunks, chunks[::-1]]
    switched = [0, 1]
    got = sk.host.debug_chain_anchors(ctx, c, K, pairs, switched)
    for pi, (p, g) in enumerate(zip(pairs, got)):
        o = O.chain_chunks(p, c, K, switched[pi])
        for key in ("score", "pointer"):
            bad = np.nonzero(g[key].astype(np.int64) != o[key].astype(np.int64))[0]
            assert len(bad) == 0, "%s pair %d: anchor %d, field %s: device %d, oracle %d" % (
                kernel, pi, bad[0], key, g[key][bad[0]], o[key][bad[0]])
        compare_selection("%s pair %d" % (kernel, pi), g, o)
        assert len(o["intervals"]) > 0
