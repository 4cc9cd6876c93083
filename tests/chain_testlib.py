"""Shared helpers of the GPU chaining tests: sketch sets built on the GPU and in the CPU oracle from the same sequences,
and the parity assertions (integer stages bit-exact, ANI / AF floats within 1e-4)."""
import numpy as np

import oracle_py as O
from bench_support import synth

TOL = 1e-4
ACGT = np.frombuffer(b"ACGT", np.uint8)
_COMP = np.zeros(256, np.uint8)
_COMP[ACGT] = np.frombuffer(b"TGCA", np.uint8)


def assert_result_close(g, o, tol=TOL):
    if np.isnan(o.ani):
        assert np.isnan(g.ani)
        return
    for f in ("ani", "af_query", "af_ref", "std", "ci_lower", "ci_upper"):
        assert abs(getattr(g, f) - getattr(o, f)) <= tol, (f, getattr(g, f), getattr(o, f))
    for f in ("q90_q", "q90_r", "q50_q", "q50_r", "q10_q", "q10_r", "num_contigs_q", "num_contigs_r",
              "avg_chain_int_len", "total_bases_covered"):
        assert getattr(g, f) == getattr(o, f), (f, getattr(g, f), getattr(o, f))


def assert_debug_equal(gd, od):
    assert gd["switched"] == od["switched"]
    assert np.array_equal(gd["anchors"], od["anchors"]), "anchors"
    assert np.array_equal(gd["chunk_first"], od["chunk_first"]), "chunk_first"
    assert np.array_equal(gd["chunk_nseeds"], od["chunk_nseeds"]), "chunk_nseeds"
    assert np.array_equal(gd["score"], od["score"]), "score"
    assert np.array_equal(gd["pointer"], od["pointer"]), "pointer"
    assert np.array_equal(gd["intervals"], od["intervals"]), "intervals"
    assert np.array_equal(gd["weight"], od["weight"]), "weights"
    assert np.allclose(gd["est"], od["est"], rtol=0, atol=1e-12), "ests"
    assert_result_close(gd["result"], od["result"])


def make_sets(ctx, genomes, sp_kw, individual=False):
    """genomes: list of lists of contig byte arrays -> (gpu set, [oracle sketches])"""
    import skani_b200 as sk
    gs = sk.sketch_sequences(ctx, genomes, sk.sketch_params(**sp_kw), individual_contig=individual)
    osk = []
    for gi, ctgs in enumerate(genomes):
        kept = [c for c in ctgs if len(c) >= 500]
        if not kept:
            continue
        if individual:
            for j, c in enumerate(kept):
                osk.append(O.sketch_from_contigs("g%06d" % gi, [c], **sp_kw))
        else:
            osk.append(O.sketch_from_contigs("g%06d" % gi, kept, **sp_kw))
    assert len(gs) == len(osk)
    return gs, osk


def synth_genomes(n, L, G):
    bases, off, goc = synth.generate(0, n, L, G=G)
    out = []
    for g in range(n):
        idx = np.nonzero(goc == g)[0]
        out.append([bases[int(off[i]):int(off[i + 1])] for i in idx])
    return out


def rand_seq(rng, n):
    return ACGT[rng.integers(0, 4, n)]


def mutate(rng, s, rate):
    s = np.array(s, np.uint8)
    m = rng.random(len(s)) < rate
    s[m] = ACGT[rng.integers(0, 4, int(m.sum()))]
    return s


def revcomp(s):
    return _COMP[np.asarray(s, np.uint8)[::-1]]
