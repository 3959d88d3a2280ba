"""The predict CLI's score dumps on the CPU: the dump kernels' arithmetic (vaporetto_b200/csrc/dump.hpp) under g++, and
the dump oracle (tests/native/dump_oracle.cpp, main.rs:125-181 restated) against a composition of the per-sentence
oracles, with the --no-norm glue and deviation 1 written out by hand."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from golden import reference_kat as kat
from test_gpu_parity import _random_model, read
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.dump_oracle import DumpOracle, compose
from vpt_testlib.oracle import OraclePredictor
from vpt_testlib.tag_scores_oracle import TagScoresOracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dump_arithmetic_on_the_host():
    exe = os.path.join(tempfile.mkdtemp(), "dump_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include"),
                           "-o", exe, os.path.join(ROOT, "tests", "native", "dump_test.cpp")])
    assert subprocess.run([exe], capture_output=True, text=True, check=True).stdout.strip() == "ok"


def _lines(rng, alpha, n):
    out = []
    for _ in range(n):
        k = int(rng.integers(0, 14))
        out.append("".join(rng.choice(list(alpha), size=k)) if k else "")
    out += ["人", "a", "\0x", b"\xff\xfe"]
    return out


def _data(lines):
    return b"".join((ln.encode() if isinstance(ln, str) else ln) + b"\n" for ln in lines)


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("no_norm", [False, True])
def test_oracle_vs_composition(seed, no_norm):
    rng = np.random.default_rng(seed)
    model, alpha = _random_model(rng, 3, 3, tags=3)
    mb = encode_model(model)
    o, so, d = OraclePredictor(mb, predict_tags=True), TagScoresOracle(mb), DumpOracle(mb, predict_tags=True)
    lines = _lines(rng, alpha + "ａＢ１", 120)
    data = _data(lines)
    for scores, tag_scores in ((True, False), (False, True), (True, True)):
        got = d.dump_lines(data, no_norm=no_norm, scores=scores, tag_scores=tag_scores)
        assert got == compose(o, so, model, lines, no_norm=no_norm, scores=scores, tag_scores=tag_scores, predict_tags=True)


def test_bundled_model_scores():
    mb = read("model.bin")
    o, so, d = OraclePredictor(mb), None, DumpOracle(mb)
    lines = ["まぁ社長は火星猫だ", "ABC１２３", "", "x"]
    for no_norm in (False, True):
        got = d.dump_lines(_data(lines), no_norm=no_norm, scores=True)
        assert got == compose(o, so, {}, lines, no_norm=no_norm, scores=True)


def test_no_norm_glue_and_deviation_1():
    """The reference's tag test model, --no-norm --predict-tags --scores --tag-scores, worked out by hand: "この" gets
    the model bias 5 at its one boundary and no tag model, "人" is a known one-character token (bias 40..43 plus no
    weights that reach it alone), and the empty line after it is rejected.  --no-norm writes each score block before
    the line's own "\n", so "こ の" is glued to "0:この 5".  The rejected line prints " " and two newlines; the reference
    would print " \t名詞:40,接尾辞:41\tジン:42,ヒト:43", the stale entry 0 of the line before, which set_default
    leaves in place (sentence.rs:140-158, 1234)."""
    d = DumpOracle(encode_model(kat.PREDICTOR_TEST_MODEL), predict_tags=True)
    out = d.dump_lines("この\n人\n\n".encode(), no_norm=True, scores=True, tag_scores=True).decode()
    assert out == ("こ の0:この 5\n\n\n" "こ\nの\n\n"
                   "人/接尾辞/ヒト\n\n" "人\t名詞:40,接尾辞:41\tジン:42,ヒト:43\n\n"
                   "\n" " \n\n")
