"""GPU: sk_sketch_set_encode writes skani v0.3 entries byte for byte as the host writer does (skani-db-tool write:
put_params + put_sketch, and put_sketch(markers_only(s)) for markers.bin) for the same sketches -- the golden E. coli pair,
viruses.fna -i, o157_reads.fa.gz -i, a zero-record genome (all_ns.fa) with test.fasta, and repeat-rich synthetic genomes
with multi-position lists of hundreds to thousands of records.  Names are chosen so that entries start at every offset
mod 16; sub-ranges (n = 0, the last genome, a middle run), pinned and pageable output, the sizes call, and import_blobs
of the encoded entries rebuilding the same set are covered.  Out-of-range genomes and short buffers are refused."""
import os
import subprocess

import numpy as np
import pytest

import fasta_py
from conftest import db_tool

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
EXPORT_KEYS = ("kmer", "pos", "cc", "markers", "contig_lengths")


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def records(path):
    return [seq for _, seq in fasta_py.read_fastx(path)], [name for name, _ in fasta_py.read_fastx(path)]


def repeat_genomes():
    rng = np.random.default_rng(11)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    out = []
    for copies in (2, 40, 700, 2500):
        unit = acgt[rng.integers(0, 4, 700)]
        flank = acgt[rng.integers(0, 4, 30000)]
        out.append([np.concatenate([flank, np.tile(unit, copies), flank[::-1]]).tobytes()])
    return out


def build_input(ctx, which):
    """(set, names, contigs, contig_order): one genome per file, or per record with individual contigs"""
    import skani_b200 as sk
    ind = False
    if which == "ecoli":
        files = ["e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz"]
        ind = False
    elif which in ("viruses", "o157"):
        files = ["viruses.fna" if which == "viruses" else "o157_reads.fa.gz"]
        ind = True
    elif which == "ns":
        files = ["all_ns.fa", "test.fasta"]
        ind = False
    if which == "repeats":
        genomes = repeat_genomes()
        heads = [["rep%d contig" % i] for i in range(len(genomes))]
        s = sk.sketch_sequences(ctx, genomes)
        kept = [(i, 0) for i in range(len(genomes))]
    else:
        genomes, heads = zip(*[records(os.path.join(GOLD, f)) for f in files])
        s = sk.sketch_sequences(ctx, list(genomes), individual_contig=ind)
        kept = s.names
    names, contigs, order = [], [], []
    for g, (fi, j) in enumerate(kept):
        names.append("x" * ((g * 7 + fi) % 17) + "/g%d" % g)    # lengths vary so that entry starts cover every offset mod 16
        hs = [h for h, q in zip(heads[fi], genomes[fi]) if len(q) >= 500]
        contigs.append([hs[j]] if ind else hs)
        order.append(j)
    return s, names, contigs, order


def host_writer(tmp, s, names, contigs, order):
    """the host writer's (full entries, markers-only entries) for the sketches of s, via skani-db-tool write"""
    lines = []
    for g in range(len(s)):
        e, i = s.export(g), s.info(g)
        lines.append("S %d %d %s" % (order[g], i["total_len"], names[g]))
        lines += ["C " + c for c in contigs[g]]
        lines.append("L %d %s" % (len(e["contig_lengths"]), " ".join(map(str, e["contig_lengths"].tolist()))))
        r = np.stack([e["kmer"], e["pos"], e["cc"]], 1).ravel().tolist()
        lines.append("R %d %s" % (len(e["kmer"]), " ".join(map(str, r))))
        lines.append("M %d %s" % (len(e["markers"]), " ".join(map(str, e["markers"].tolist()))))
        lines.append("E")
    d = str(tmp)
    os.makedirs(d)
    subprocess.run([db_tool(), "write", d, "125", "15", "1000"], input="\n".join(lines) + "\n", text=True, check=True)
    full = open(os.path.join(d, "sketches.db"), "rb").read()
    mk = open(os.path.join(d, "markers.bin"), "rb").read()[626 + 8:]
    return full, mk


def same_sets(a, b):
    assert len(a) == len(b)
    for g in range(len(a)):
        ea, eb = a.export(g), b.export(g)
        for key in EXPORT_KEYS:
            assert np.array_equal(ea[key], eb[key]), (key, g)
        assert a.info(g) == b.info(g), g


@pytest.mark.parametrize("which", ["ecoli", "viruses", "o157", "ns", "repeats"])
def test_encode_equals_host_writer(ctx, tmp_path, which):
    import skani_b200 as sk
    import torch
    s, names, contigs, order = build_input(ctx, which)
    n = len(s)
    full_ref, mk_ref = host_writer(tmp_path / "host", s, names, contigs, order)
    full, flen = s.encode(names, contigs, order)
    mk, mlen = s.encode(names, contigs, order, markers_only=True)
    assert full.tobytes() == full_ref and mk.tobytes() == mk_ref
    assert np.array_equal(s.encode_sizes(names, contigs, order), flen)
    assert np.array_equal(s.encode_sizes(names, contigs, order, markers_only=True), mlen)
    starts = np.concatenate([[0], np.cumsum(flen)[:-1]]).astype(np.int64)
    if n >= 32:
        assert set((starts % 16).tolist()) == set(range(16))
    if which == "repeats":         # long multi-position lists really occur
        assert max(np.bincount(s.export(g)["kmer"]).max() for g in range(n)) >= 1000
    if which == "ns":
        assert s.info(0)["n_records"] == 0
    # pinned output, and a pageable one at an odd address
    pin = torch.empty(len(full) + 64, dtype=torch.uint8, pin_memory=True).numpy()
    got, _ = s.encode(names, contigs, order, out=pin[:len(full)])
    assert got.tobytes() == full_ref
    odd = np.zeros(len(full) + 8, np.uint8)
    got, _ = s.encode(names, contigs, order, out=odd[3:3 + len(full)])
    assert got.tobytes() == full_ref
    # sub-ranges
    for g0, k in ((0, 0), (n - 1, 1), (n // 3, max(1, n // 2))):
        k = min(k, n - g0)
        sl = slice(g0, g0 + k)
        got, ln = s.encode(names[sl], contigs[sl], order[sl], g0=g0, n=k)
        a = int(starts[g0]) if k else 0
        assert got.tobytes() == (full_ref[a:a + int(flen[sl].sum())] if k else b"") and np.array_equal(ln, flen[sl])
    # the entries decode on the device to the same set
    back = sk.import_blobs(ctx, full, starts, flen)
    same_sets(back, s)
    back.free()
    s.free()


def test_encode_refusals(ctx):
    from skani_b200.host import SkaniError
    s, names, contigs, order = build_input(ctx, "ecoli")
    n = len(s)
    for g0, k in ((n, 1), (n + 1, 0), (1, n), (0, n + 1)):
        with pytest.raises(SkaniError, match="rc=-2"):
            s.encode(["a"] * k, [[]] * k, [0] * k, g0=g0, n=k)
        with pytest.raises(SkaniError, match="rc=-2"):
            s.encode_sizes(["a"] * k, [[]] * k, [0] * k, g0=g0, n=k)
    need = int(s.encode_sizes(names, contigs, order).sum())
    with pytest.raises(SkaniError, match="rc=-2"):
        s.encode(names, contigs, order, out=np.zeros(need - 1, np.uint8))
    got, ln = s.encode([], [], [], g0=n, n=0)
    assert len(got) == 0 and len(ln) == 0
    s.free()
