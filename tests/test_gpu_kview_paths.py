"""GPU: the k-mer view built through (key, record index) pairs -- the sort used when genome, k-mer and record index do not
fit one 64-bit key (forced here with SK_KVIEW_SORT_PAIRS) -- gives byte for byte the same sketch set as the keys-only sort,
on a sub-batch with genomes without records between genomes with records (their group sentinels and offsets), and both
match the CPU oracle."""
import numpy as np
import pytest

import oracle_py as O
from bench_support import synth

pytestmark = pytest.mark.gpu


def blob(s):
    import torch
    nb, nw = s.subset_blob_size(None, 0)
    t = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    meta = s.pack_subset(None, 0, t.data_ptr(), nw)
    return t.cpu().numpy(), np.asarray(meta)


@pytest.mark.parametrize("c,k,mc", [(125, 15, 1000), (10, 16, 40)])
def test_kview_pair_sort_equals_key_sort(monkeypatch, c, k, mc):
    import skani_b200 as sk
    ctx = sk.Context(0)
    try:
        bases, off, goc = synth.generate(0, 4, 300_000, G=2)
        gen = [[bases[int(off[i]):int(off[i + 1])] for i in np.nonzero(goc == g)[0]] for g in range(4)]
        # genome 1: one contig too short to seed; genome 3: no contigs; genome 5: records again
        genomes = [gen[0], [gen[1][0][:30]], gen[1], [], gen[2], gen[3]]
        contigs = [x for g in genomes for x in g]
        o = np.concatenate([[0], np.cumsum([len(x) for x in contigs])]).astype(np.uint64)
        gc = np.concatenate([np.full(len(g), i, np.uint32) for i, g in enumerate(genomes)])
        sp = sk.sketch_params(c, k, mc)
        seq = np.concatenate(contigs)
        keys = sk.sketch_contigs(ctx, seq, o, gc, len(genomes), sp)
        monkeypatch.setenv("SK_KVIEW_SORT_PAIRS", "1")
        pairs = sk.sketch_contigs(ctx, seq, o, gc, len(genomes), sp)
        monkeypatch.delenv("SK_KVIEW_SORT_PAIRS")
        assert keys.info(1)["n_records"] == 0 and keys.info(3)["n_contigs"] == 0
        a, am = blob(keys)
        b, bm = blob(pairs)
        assert np.array_equal(am, bm) and np.array_equal(a, b)
        for g, ctgs in enumerate(genomes):
            e, x = pairs.export(g), O.sketch_from_contigs("g%d" % g, ctgs, c=c, k=k, marker_c=mc).export()
            for key in ("kmer", "pos", "cc", "markers"):
                assert np.array_equal(e[key], x[key]), (g, key)
        keys.free()
        pairs.free()
    finally:
        ctx.close()
