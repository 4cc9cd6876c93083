"""`skani-b200 triangle` on the store path (sketches kept in a host sketch store, chained in working sets; forced here with a
small SK_DEVICE_BUDGET_MB): stdout and the .af matrix must equal the default in-memory run byte for byte in every output
mode, for FASTA inputs, -i and .sketch inputs, and stderr must name the store path."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")
EC, K12, VIR, TEST = (os.path.join(GOLD, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "viruses.fna", "test.fasta"))
BUDGET_MB = "8"      # about 2 MB per E. coli sketch: the pair fits one working set, the viruses spread over others


def run(args, out_dir, budget=None):
    env = dict(os.environ)
    env.pop("SK_DEVICE_BUDGET_MB", None)
    if budget:
        env["SK_DEVICE_BUDGET_MB"] = budget
    out = os.path.join(out_dir, "store" if budget else "mem")
    p = subprocess.run([BIN, "triangle"] + args + ["-o", out], capture_output=True, text=True, timeout=600, env=env)
    assert p.returncode == 0, p.stderr
    text = open(out).read()
    af = open(out + ".af").read() if os.path.exists(out + ".af") else None
    return text, af, p.stderr


def same_on_store_path(args, tmp_path, min_lines=2):
    mem = run(args, str(tmp_path))
    store = run(args, str(tmp_path), BUDGET_MB)
    assert "INFO Store path" in store[2] and "INFO Store path" not in mem[2]
    assert store[0] == mem[0] and store[1] == mem[1]
    assert len(mem[0].strip().split("\n")) >= min_lines
    return mem


MODES = {"sparse": ["-E"], "sparse_ci_diagonal": ["-E", "--ci", "--diagonal"], "sparse_detailed": ["-E", "--detailed"],
         "matrix": [], "full_matrix": ["--full-matrix"], "diagonal": ["--diagonal"], "distance": ["--distance", "--full-matrix"]}
INPUTS = {"files": [EC, K12, VIR, TEST], "individual": [VIR, TEST, EC, "-i"]}


@pytest.mark.parametrize("inputs", sorted(INPUTS))
@pytest.mark.parametrize("mode", sorted(MODES))
def test_store_path_output_identical(tmp_path, mode, inputs):
    text, af, _ = same_on_store_path(INPUTS[inputs] + MODES[mode], tmp_path)
    assert (af is None) == mode.startswith("sparse")
    if mode.startswith("sparse"):
        assert len(text.strip().split("\n")) >= 2          # header and at least one related pair


@pytest.fixture(scope="module")
def sketches(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("sk") / "sep")
    p = subprocess.run([BIN, "sketch", EC, K12, VIR, "-o", d, "--separate-sketches"], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    return [os.path.join(d, os.path.basename(f) + ".sketch") for f in (EC, K12, VIR)]


@pytest.mark.parametrize("mode", ["sparse", "matrix", "full_matrix"])
def test_store_path_sketch_inputs(tmp_path, sketches, mode):
    _, _, err = same_on_store_path(sketches + MODES[mode], tmp_path)
    assert "INFO Sketches detected" in err
