"""GPU: sk_sketch_set_import_blobs (skani v0.3 sketch entries as stored, expanded on the device) builds the same set as
sk_sketch_set_import_batch from the host-decoded records -- export and info per genome, and chain_pairs byte for byte over
all pairs -- for databases of the golden E. coli, viruses -i and reads -i sketches, synthetic blobs with heavy
multi-position lists, blobs at every offset mod 16, marker-only and zero-record genomes, pinned and pageable input.
Blobs that do not decode are refused with SK_ERR_PARAM naming the blob; the CLI ends every database path, search -d
included, with `ERROR Failed to load sketch <name>` when only the device can see the fault (a multi-position index past
the entry's lists)."""
import os
import struct
import subprocess

import numpy as np
import pytest

import skani_db_py as D

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")
EC, K12, VIR, TEST, O157 = (os.path.join(GOLD, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "viruses.fna", "test.fasta",
                                                            "o157_reads.fa.gz"))
EXPORT_KEYS = ("kmer", "pos", "cc", "markers", "contig_lengths")


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def cli(args, cwd, env=None):
    e = {k: v for k, v in os.environ.items() if k not in ("SK_DEVICE_BUDGET_MB", "SK_SKETCH_GROUP_RECORDS")}
    e.update(env or {})
    os.makedirs(cwd, exist_ok=True)
    return subprocess.run([BIN] + args, capture_output=True, text=True, timeout=900, env=e, cwd=cwd)


@pytest.fixture(scope="module")
def golden_blobs(tmp_path_factory):
    """blobs of three databases written by `sketch`: (all bytes, offsets, lengths, names)"""
    d = tmp_path_factory.mktemp("dbs")
    data, off, ln, names = b"", [], [], []
    for name, args in (("ecoli", [EC, K12]), ("vir", [VIR, "-i"]), ("reads", [O157, "-i"])):
        assert cli(["sketch"] + args + ["-o", str(d / name)], str(d)).returncode == 0
        raw = open(str(d / name / "sketches.db"), "rb").read()
        for nm, o, n in D.read_db(str(d / name))[3]:
            off.append(len(data) + o); ln.append(n); names.append(nm)
        data += raw
    return data, off, ln, names


def decoded(data, off, ln):
    """the blobs decoded on the host (independent decoder) in import_sketches' form"""
    out = []
    for o, n in zip(off, ln):
        c = D.Cur(data, o)
        D.params(c)
        s = D.sketch(c)
        r = np.array(s["records"], np.uint64).reshape(-1, 3)
        out.append(dict(kmer=r[:, 0].astype(np.uint32), pos=r[:, 1].astype(np.uint32), cc=r[:, 2].astype(np.uint32),
                        markers=np.array(s["markers"], np.uint64), contig_lengths=np.array(s["contig_lengths"], np.uint32),
                        total_len=s["total_len"]))
    return out


def same_sets(ctx, a, b, chain=True):
    import skani_b200 as sk
    assert len(a) == len(b)
    for g in range(len(a)):
        ea, eb = a.export(g), b.export(g)
        for key in EXPORT_KEYS:
            assert np.array_equal(ea[key], eb[key]), (key, g)
        assert a.info(g) == b.info(g), g
    if chain and len(a) > 1:
        n = len(a)
        pairs = np.array([(i << 32) | j for i in range(n) for j in range(n) if i != j], np.uint64)
        mp = sk.map_params()
        assert sk.chain_pairs(ctx, a, a, pairs, mp, as_array=True).tobytes() == sk.chain_pairs(ctx, b, b, pairs, mp, as_array=True).tobytes()


def check(ctx, data, off, ln, sp=None, chain=True):
    import skani_b200 as sk
    got = sk.import_blobs(ctx, data, off, ln, sp)
    want = sk.import_sketches(ctx, decoded(bytes(data), off, ln), sp)
    same_sets(ctx, got, want, chain)
    got.free(); want.free()


# ---- a writer for synthetic blobs: groups = [(k-mer, [(pos, cc), ...]), ...] in file order
def params_bytes(c=125, k=15, m=1000, use_aa=0):
    b = bytearray(D.expected_params_bytes(c, k, m))
    b[25] = use_aa
    return bytes(b)


def blob(name, groups, contig_lengths, markers, c=125, k=15, m=1000, seeds=True, use_aa=0, bad_index=None):
    q = lambda v: struct.pack("<Q", v)                       # noqa: E731
    out = [params_bytes(c, k, m, use_aa), q(len(name)), name.encode()]
    multi = [g for g in groups if len(g[1]) > 1]
    if not seeds:
        out += [b"\x00", q(0)]
    else:
        out += [b"\x01", q(len(groups))]
        j = 0
        for km, recs in groups:
            if len(recs) == 1:
                v = ((((recs[0][0] << 31) | recs[0][1]) << 1) | 1)
            else:
                v = (len(multi) if bad_index == km else j) << 1
                j += 1
            out.append(struct.pack("<IQ", km, v))
        out.append(q(len(multi)))
        for _, recs in multi:
            out.append(q(len(recs)) + b"".join(struct.pack("<II", p, cc) for p, cc in recs))
    out += [q(len(contig_lengths))] + [q(3) + b"ctg" for _ in contig_lengths]
    out += [q(int(sum(contig_lengths))), q(len(contig_lengths)), np.array(contig_lengths, "<u4").tobytes(), q(0), q(len(markers)),
            np.array(markers, "<u8").tobytes(), q(c), q(c), q(k), q(0), b"\x00\x00"]
    return b"".join(out)


def synthetic(rng, name, n_keys, n_contigs, list_lens=(), n_markers=50, **kw):
    """random k-mers with unique (contig, pos); list_lens: extra multi-position k-mers of these lengths"""
    lens = [1] * n_keys + list(list_lens)
    rng.shuffle(lens)
    kmers = rng.choice(4 ** 15, len(lens), replace=False)
    total = int(sum(lens))
    slots = rng.choice(n_contigs * 2_000_000, total, replace=False)
    recs = [(int(s % 2_000_000), int((s // 2_000_000) << 1 | rng.integers(2))) for s in slots]
    groups, at = [], 0
    for km, n in zip(kmers, lens):
        groups.append((int(km), recs[at:at + n]))
        at += n
    markers = np.unique(rng.integers(0, 1 << 42, n_markers, dtype=np.uint64))
    return blob(name, groups, [2_000_000] * n_contigs, markers, **kw)


def packed(blobs, pad=lambda i: 0, mod16=False):
    """blobs back to back with pad(i) bytes before blob i, or (mod16) each blob i at an offset = i mod 16"""
    data, off, ln = b"", [], []
    for i, b in enumerate(blobs):
        data += b"\xee" * ((i - len(data)) % 16 if mod16 else pad(i))
        off.append(len(data)); ln.append(len(b))
        data += b
    return data, off, ln


def test_golden_databases(ctx, golden_blobs):
    data, off, ln, names = golden_blobs
    assert len(off) > 300 and {os.path.basename(n) for n in names[:2]} == {"e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz"}
    check(ctx, data, off, ln)
    # the same blobs at every offset mod 16, and the E. coli pair alone from pinned and pageable memory
    blobs = [data[o:o + n] for o, n in zip(off, ln)][:24]
    d16, o16, l16 = packed(blobs, mod16=True)
    assert [o % 16 for o in o16] == [i % 16 for i in range(24)]
    check(ctx, d16, o16, l16)
    import torch
    d2, o2, l2 = packed(blobs[:2], pad=lambda i: 5 + i)
    pinned = torch.empty(len(d2), dtype=torch.uint8).pin_memory()
    pinned.numpy()[:] = np.frombuffer(d2, np.uint8)
    check(ctx, pinned.numpy(), o2, l2)
    check(ctx, np.frombuffer(d2, np.uint8).copy(), o2, l2)


def test_synthetic_blobs(ctx):
    import skani_b200 as sk
    rng = np.random.default_rng(7)
    blobs = [synthetic(rng, "heavy", 3000, 3, list_lens=[2, 3, 50, 999, 1000, 1000] + [2] * 200),
             synthetic(rng, "zero-keys", 0, 2),
             blob("markers-only", [], [], np.arange(10, 200, 7, dtype=np.uint64), seeds=False),
             synthetic(rng, "plain", 5000, 1, list_lens=[2] * 40),
             blob("nothing", [], [], [], seeds=True),
             synthetic(rng, "many-contigs", 2000, 60, list_lens=[4, 17]),
             synthetic(rng, "one-key", 0, 1, list_lens=[1000], n_markers=1)]
    for pad in (lambda i: 0, lambda i: 1 + 3 * i, lambda i: 15 - i % 16):
        check(ctx, *packed(blobs, pad), chain=False)          # chained: the real sketches of test_golden_databases
    s = sk.import_blobs(ctx, *packed(blobs))
    assert s.info(1)["n_records"] == 0 and s.info(2)["n_records"] == 0 and s.info(4)["n_records"] == 0
    assert s.info(0)["n_records"] == 3000 + 2 + 3 + 50 + 999 + 2000 + 400 and s.info(6)["n_records"] == 1000
    s.free()


def test_beyond_one_staging_chunk(ctx, golden_blobs):
    """more bytes than one 64 MiB staging chunk, pageable and pinned: the E. coli pair repeated"""
    import torch
    import skani_b200 as sk
    data, off, ln, _ = golden_blobs
    pair = [data[o:o + n] for o, n in zip(off[:2], ln[:2])]
    reps = (70 << 20) // (len(pair[0]) + len(pair[1])) + 1
    big, o2, l2 = packed(pair * reps, pad=lambda i: i % 11)
    assert len(big) > 64 << 20
    pinned = torch.empty(len(big), dtype=torch.uint8).pin_memory()
    pinned.numpy()[:] = np.frombuffer(big, np.uint8)
    want = sk.import_sketches(ctx, decoded(big, o2[:2], l2[:2]) * reps)
    for src in (big, pinned.numpy()):
        got = sk.import_blobs(ctx, src, o2, l2)
        same_sets(ctx, got, want, chain=False)
        got.free()
    want.free()


def test_refused_blobs(ctx):
    import skani_b200 as sk
    rng = np.random.default_rng(9)
    good = [synthetic(rng, "g%d" % i, 500, 2, list_lens=[2, 3]) for i in range(4)]
    groups = [(7, [(1, 2), (5, 2)]), (9, [(3, 0)]), (11, [(8, 0), (9, 0)])]
    cases = {"multi-position index out of range": blob("bad", groups, [100], [1, 2], bad_index=11),
             "truncated sketch data": good[0][:-5],
             "sketch parameters differ": blob("c30", groups, [100], [1, 2], c=30),
             "amino-acid sketches are not supported": blob("aa", groups, [100], [1, 2], use_aa=1)}
    for why, bad in cases.items():
        for at in (0, 2):
            blobs = good[:at] + [bad] + good[at:]
            with pytest.raises(sk.BlobError) as e:
                sk.import_blobs(ctx, *packed(blobs, pad=lambda i: i))
            assert e.value.blob == at and why in str(e.value), (why, at, str(e.value))
    # the context stays usable
    check(ctx, *packed(good), chain=False)


# ---- the CLI: an entry whose fault only the device sees
GROUPS = {"SK_DEVICE_BUDGET_MB": "8", "SK_SKETCH_GROUP_RECORDS": "3000"}
MEM_GROUPS = {"SK_SKETCH_GROUP_RECORDS": "3000"}
STORE = {"SK_DEVICE_BUDGET_MB": "8"}


def test_cli_entry_with_bad_multi_index(tmp_path):
    db = str(tmp_path / "db")
    assert cli(["sketch", EC, K12, VIR, TEST, "-o", db], str(tmp_path)).returncode == 0
    index = D.read_db(db)[3]
    name, off, _ = index[1]
    assert name == K12
    raw = bytearray(open(os.path.join(db, "sketches.db"), "rb").read())
    keys = off + 626 + 8 + len(name) + 1
    n_keys = struct.unpack_from("<Q", raw, keys)[0]
    n_multi = struct.unpack_from("<Q", raw, keys + 8 + 12 * n_keys)[0]
    struct.pack_into("<Q", raw, keys + 8 + 4, n_multi << 1)            # first key -> the list after the last one
    open(os.path.join(db, "sketches.db"), "wb").write(bytes(raw))
    t = str(tmp_path / "run")
    for args, env in ((["triangle", db], None), (["triangle", db], MEM_GROUPS), (["triangle", db], GROUPS),
                      (["triangle", db, "--gpus", "3"], None), (["dist", "-q", EC, "-r", db], MEM_GROUPS),
                      (["dist", "-q", EC, "-r", db, "--gpus", "3"], None), (["dist", "-q", EC, "-r", db], STORE),
                      (["dist", "-q", db, "-r", EC], None), (["search", "-d", db, EC], None), (["search", "-d", db, EC, "--gpus", "2"], None)):
        p = cli(args, t, env)
        assert p.returncode == 1 and "ERROR Failed to load sketch %s" % K12 in p.stderr, (args, env, p.stderr)
        rows = [ln for ln in p.stdout.split("\n") if ln and not ln.startswith("Ref_file")]
        assert not rows and "INFO Screen + chain" not in p.stderr, (args, env, p.stdout)
        if args[0] != "search":
            assert "Ref_file" not in p.stdout
