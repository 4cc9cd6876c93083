"""`skani-b200 dereplicate --fixed-reps / --fixed-reps-list`: a round trip (an earlier run's --representatives file passed
back as --fixed-reps-list keeps its clusters' ids, and every row equals sk_dereplicate_fixed computed here on the same
genomes, name ranks and ranks); a catalogue given as a sketch database with new FASTA files prints what the same catalogue
given as FASTA prints; --host-store (small and derived budgets) and --gpus 2 print what the in-memory path prints; -i; the
refusals (an explicit -c / -k / -m against a sketch group, two sketch groups with different parameters, a file in both
groups, an empty fixed group, the flags on other commands); dereplicate without the flags is unchanged."""
import os
import subprocess

import numpy as np
import pytest

from fasta_py import read_fastx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")
EC, K12, VIR = (os.path.join(GOLD, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "viruses.fna"))


def run(args, env_add=None, rc=0):
    env = dict(os.environ)
    for k in ("SK_DEVICE_BUDGET_MB", "SK_DEREP_WAVE", "SK_TRACE"):
        env.pop(k, None)
    env.update({k: v for k, v in (env_add or {}).items() if v is not None})
    p = subprocess.run([BIN] + args, capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == rc, p.stderr
    return p.stdout, p.stderr


def ensure_built():
    if not os.path.exists(BIN):
        import __graft_entry__ as g
        g.build()


@pytest.fixture(scope="module")
def synth_files(tmp_path_factory):
    """48 synthetic 120 kbp genomes in families of 8, one FASTA file each, of slightly different lengths"""
    from bench_support import synth
    d = tmp_path_factory.mktemp("synth")
    n, L = 48, 120_000
    bases, off, goc = synth.generate(0, n, L, G=8)
    files = []
    for g in range(n):
        path = str(d / ("g%02d.fa" % g))
        idx = np.nonzero(goc == g)[0]
        with open(path, "wb") as f:
            for k, i in enumerate(idx):
                end = int(off[i + 1]) - (g * 97 if k == len(idx) - 1 else 0)     # distinct lengths: a visible length rank
                f.write(b">g%02d_c%d synthetic\n" % (g, i) + bases[int(off[i]):end].tobytes() + b"\n")
        files.append(path)
    return files


def rows_of(tsv):
    return [ln.split("\t") for ln in tsv.rstrip("\n").split("\n")[1:]]


def contract(fixed, new, ani):
    """sk_dereplicate_fixed on the genomes of the fixed files (sorted) then the new ones (sorted), name ranks over all file
    names, ranks: the fixed genomes longest first, then the new ones; the TSV's first six columns"""
    import skani_b200 as sk
    files = sorted(fixed) + sorted(new)
    genomes = [[seq for _, seq in read_fastx(f)] for f in files]
    ctx = sk.Context(0)
    try:
        s = sk.sketch_sequences(ctx, genomes)
        names = sorted(set(files))
        s.set_name_ranks(np.array([names.index(f) for f in files], np.uint64))
        total = np.array([sum(len(c) for c in g if len(c) >= 500) for g in genomes], np.int64)
        nf = len(fixed)
        order = np.concatenate([np.lexsort((np.arange(nf), -total[:nf])), nf + np.lexsort((np.arange(len(new)), -total[nf:]))])
        rank = np.empty(len(files), np.uint32)
        rank[order] = np.arange(len(files))
        rep, cl, join, _ = sk.dereplicate_fixed(ctx, s, rank, nf, min_ani=ani / 100.0)
    finally:
        ctx.close()
    out = []
    for g in range(len(files)):
        if rep[g] == g:
            vals = ["100.00"] * 3
        else:
            r = join[g]
            is_ref = r["ref_id"] == g
            af_g, af_r = (r["af_ref"], r["af_query"]) if is_ref else (r["af_query"], r["af_ref"])
            vals = ["%.2f" % float(np.float32(v) * np.float32(100)) for v in (r["ani"], af_g, af_r)]
        out.append([files[g], files[rep[g]], str(cl[g])] + vals)
    return out


@pytest.mark.gpu
def test_round_trip(synth_files, tmp_path):
    s1, s2 = synth_files[:32], synth_files[32:]
    reps = str(tmp_path / "reps.txt")
    first, _ = run(["dereplicate", "--representatives", reps] + s1)
    old = {r[0]: r[2] for r in rows_of(first) if r[0] == r[1]}
    listed = open(reps).read().split("\n")[:-1]
    assert listed == sorted(old, key=lambda f: int(old[f]))
    base, err = run(["dereplicate", "--fixed-reps-list", reps, "-o", str(tmp_path / "o.tsv")] + s2)
    assert base == "" and "%d fixed representatives" % len(listed) in err
    out = open(str(tmp_path / "o.tsv")).read()
    rows = rows_of(out)
    assert [r[0] for r in rows] == sorted(listed) + sorted(s2)
    for r in rows[:len(listed)]:
        assert r[1] == r[0] and r[2] == old[r[0]]
    assert [r[:6] for r in rows] == contract(listed, s2, 95.0)
    for env in ({"SK_DEREP_WAVE": "1"}, {"SK_DEREP_WAVE": "3"}):
        assert run(["dereplicate", "--fixed-reps-list", reps] + s2, env)[0] == out
    # a catalogue with edges inside it (every genome of s1 fixed): each stays a representative of its own cluster
    inside = rows_of(run(["dereplicate", "--ani", "90"] + [a for f in s1[:16] for a in ("--fixed-reps", f)] + s2)[0])
    assert all(r[0] == r[1] for r in inside[:16]) and sorted(int(r[2]) for r in inside[:16]) == list(range(16))
    assert [r[:6] for r in inside] == contract(s1[:16], s2, 90.0)


@pytest.mark.gpu
def test_database_catalogue(synth_files, tmp_path):
    cat, new = synth_files[:24] + [EC], synth_files[24:] + [K12]
    db = str(tmp_path / "catalogue")
    run(["sketch"] + cat + ["-o", db])
    as_fasta, _ = run(["dereplicate", "--ani", "97"] + new + [a for f in cat for a in ("--fixed-reps", f)])
    as_db, err = run(["dereplicate", "--ani", "97", "--fixed-reps", db] + new)
    assert as_db == as_fasta and "%d fixed representatives" % len(cat) in err
    sep = str(tmp_path / "sep")
    run(["sketch"] + new + ["-o", sep, "--separate-sketches"])
    sketches = sorted(os.path.join(sep, f) for f in os.listdir(sep) if f.endswith(".sketch"))
    assert run(["dereplicate", "--ani", "97", "--fixed-reps", db] + sketches)[0] == as_fasta      # both groups sketches
    listing = tmp_path / "cat.txt"
    listing.write_text("\n".join(cat) + "\n")
    db_new = str(tmp_path / "new_db")
    run(["sketch"] + new + ["-o", db_new])
    assert run(["dereplicate", "--ani", "97", "--fixed-reps-list", str(listing), db_new])[0] == as_fasta   # FASTA catalogue, new db


@pytest.mark.gpu
@pytest.mark.parametrize("individual", [False, True])
def test_host_store_and_gpus(synth_files, tmp_path, individual):
    flags = ["-i"] if individual else []
    fixed = synth_files[:20] + ([VIR] if individual else [EC])
    new = synth_files[20:] + ([EC] if individual else [K12])
    args = ["dereplicate"] + flags + [a for f in fixed for a in ("--fixed-reps", f)] + new
    reps = str(tmp_path / "r.txt")
    base, err = run(args + ["--representatives", reps])
    base_reps = open(reps).read()
    rows = rows_of(base)
    nf = sum(r[0] in fixed for r in rows)
    assert all(r[0] in fixed for r in rows[:nf]) and "%d fixed representatives" % nf in err
    assert all(r[0] == r[1] and (not individual or r[6] == r[7]) for r in rows[:nf])
    assert sorted(int(r[2]) for r in rows[:nf]) == list(range(nf))
    for budget, gpus, wave in ((None, "1", None), ("8", "1", "1"), ("8", "2", None), (None, "2", "3")):
        out, err = run(args + ["--host-store", "--gpus", gpus, "--representatives", reps], {"SK_DEVICE_BUDGET_MB": budget, "SK_DEREP_WAVE": wave})
        assert out == base, (budget, gpus, wave)
        assert open(reps).read() == base_reps and "Store path" in err
    if not individual:
        assert [r[:6] for r in rows] == contract(fixed, new, 95.0)


@pytest.mark.gpu
def test_without_the_flags_unchanged(synth_files):
    out, err = run(["dereplicate"] + synth_files[:24])
    assert out == run(["cluster"] + synth_files[:24])[0] and "fixed" not in err


@pytest.mark.gpu
def test_sketch_parameter_refusals(synth_files, tmp_path):
    db, db30 = str(tmp_path / "db"), str(tmp_path / "db30")
    run(["sketch"] + synth_files[:8] + ["-o", db])
    run(["sketch", "-c", "30"] + synth_files[8:16] + ["-o", db30])
    for flag in (["-c", "100"], ["-k", "13"], ["-m", "500"]):
        _, err = run(["dereplicate"] + flag + ["--fixed-reps", db] + synth_files[16:20], rc=1)
        assert "ERROR %s %s differs from the sketch parameter" % tuple(flag) in err and "WARN" not in err, err
        _, err = run(["dereplicate"] + flag + ["--fixed-reps", synth_files[16], db], rc=1)
        assert "of the new genomes" in err, err
    assert run(["dereplicate", "-c", "125", "--fixed-reps", db] + synth_files[16:20])[0]    # equal to the sketches' c: accepted
    _, err = run(["dereplicate", "--fixed-reps", db, db30], rc=1)
    assert "\nERROR Sketch parameters of %s (c = 30, " % db30 in err and "differ from those of %s (c = 125, " % db in err, err


def test_input_refusals(tmp_path):
    ensure_built()
    _, err = run(["dereplicate", "--fixed-reps", VIR, VIR, EC], rc=1)
    assert err.startswith("ERROR %s is both a fixed representative and a new genome" % VIR)
    empty = tmp_path / "empty.txt"
    empty.write_text("")
    _, err = run(["dereplicate", "--fixed-reps-list", str(empty), EC], rc=1)
    assert err.startswith("ERROR --fixed-reps") and "no fixed representatives" in err
    _, err = run(["dereplicate", "--fixed-reps", EC], rc=1)
    assert err.startswith("ERROR No reference inputs found")
    db = tmp_path / "db"
    db.mkdir()
    (db / "index.db").write_bytes(b"")
    (db / "sketches.db").write_bytes(b"")
    _, err = run(["dereplicate", "--fixed-reps", str(db), "--fixed-reps", VIR, EC], rc=1)
    assert err.startswith("ERROR Sketch database") and "cannot be mixed" in err


@pytest.mark.parametrize("cmd", ["triangle", "cluster", "tree", "dist", "search", "sketch"])
@pytest.mark.parametrize("flag", ["--fixed-reps", "--fixed-reps-list"])
def test_other_commands_reject_the_flags(cmd, flag):
    ensure_built()
    _, err = run([cmd, flag, VIR, EC], rc=2)
    assert "ERROR unknown option %s" % flag in err
