"""vpt_evaluate_lines (the reference's `evaluate` command, evaluate/src/main.rs:69-195) on the device against the CPU
oracle's restatement (vpt_testlib/eval_oracle.py): totals and every per-line count."""
import itertools
import os
import random
import subprocess
import sys

import pytest

import vaporetto_b200 as vb
from vpt_testlib import eval_oracle as eo
from vpt_testlib.oracle import OraclePredictor

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CLI = os.path.join(os.path.dirname(HERE), "tools", "evaluate_cli.py")
MODEL = os.path.join(HERE, "golden", "model.bin")
DOCS = os.path.join(HERE, "golden", "docs.tok")
KEYS = ("tp", "tn", "fp", "fn", "n_sys", "n_ref", "n_cor")


def _check(p, o, data, no_norm, wsconst, predict_tags):
    want, rows = eo.evaluate_lines(o, data, no_norm=no_norm, wsconst=wsconst, predict_tags=predict_tags)
    got, lc = p.evaluate_lines(data, no_norm=no_norm, wsconst=wsconst, predict_tags=predict_tags, per_line=True)
    assert got == want, (no_norm, wsconst, predict_tags)
    assert lc.tolist() == rows, (no_norm, wsconst, predict_tags)
    assert p.evaluate_lines(data, no_norm=no_norm, wsconst=wsconst, predict_tags=predict_tags) == want
    return got


@pytest.fixture(scope="module")
def docs():
    data = open(MODEL, "rb").read()
    return vb.Predictor(vb.Model.read(data), predict_tags=True), OraclePredictor(data, predict_tags=True)


@pytest.mark.parametrize("no_norm,predict_tags,wsconst", list(itertools.product((False, True), (False, True),
                                                                                ("", "K", "GD"))))
def test_docs_tok(docs, no_norm, predict_tags, wsconst):
    p, o = docs
    got = _check(p, o, open(DOCS, "rb").read(), no_norm, wsconst, predict_tags)
    assert got["n_lines"] == got["n_sentences"] == 2
    if wsconst == "":
        assert (got["tp"], got["tn"], got["fp"], got["fn"]) == (7, 7, 0, 0)
        word_ok = predict_tags or no_norm  # normalised without tags: the gold's tag fields meet empty system tags
        assert (got["n_sys"], got["n_ref"], got["n_cor"]) == (9, 9, 9 if word_ok else 0)
    if wsconst == "K":
        assert (got["tp"], got["tn"], got["fn"]) == (6, 7, 1)  # the boundary 星|猫 is cleared


def _gold_line(rng, raw, bounds, tags, k):
    """A gold line for `raw` with perturbed boundaries and tag fields and gratuitous escapes."""
    def esc(c, tag):
        if c in " /\\" or rng.random() < 0.04:
            return "\\" + c
        return c
    b = [x if rng.random() > 0.08 else 1 - x for x in bounds]  # merge and split tokens
    out = []
    for i, c in enumerate(raw):
        if i and b[i - 1]:
            out.append(" ")
        out.append(esc(c, False))
        if i + 1 == len(raw) or b[i]:
            fields = list(tags[i]) if tags else []
            u = rng.random()
            if u < 0.6:
                fields = fields + [None] * (k - len(fields))
            elif u < 0.7:
                fields = fields[:-1]
            elif u < 0.8:
                fields = fields + ["x/y z\\"]
            if fields and rng.random() < 0.1:
                fields[rng.randrange(len(fields))] = rng.choice(["名詞", "a b", None, "\\/"])
            while fields and fields[-1] is None and rng.random() < 0.5:
                fields.pop()
            for f in fields:
                out.append("/" + ("".join(esc(ch, True) for ch in f) if f else ""))
    return "".join(out)


@pytest.fixture(scope="module")
def synthetic():
    from vpt_testlib import synth
    mb = synth.gen_model_bccwj_shaped(n_patterns=30_000, sample_sentences=50_000, tag_models=1_500)
    p, o = vb.Predictor(vb.Model.read(mb), predict_tags=True), OraclePredictor(mb, predict_tags=True)
    text, offs, _ = synth.gen_text(1500, 40, seed=synth.TEXT_SEED + 21)
    raw_lines = [text[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)]
    rng = random.Random(7)
    # add spaces, slashes and backslashes to some surfaces: they are escaped in the gold
    raw_lines = [r.replace(b"a", b" ", 1).replace(b"b", b"/", 1).replace(b"c", b"\\", 1) if i % 5 == 0 else r
                 for i, r in enumerate(raw_lines)]
    tagged, _ = o.tokenize_lines(b"\n".join(raw_lines) + b"\n", predict_tags=True)
    gold = []
    for line in tagged.decode().split("\n")[:-1]:
        if not line:
            continue
        raw, bounds, tags = eo.parse_tokenized(line)
        gold.append(_gold_line(rng, raw, bounds, tags, o.n_tags))
    long_line = " ".join(gold[:1200])  # over 64 KiB
    assert len(long_line.encode()) > 65536
    parts = []
    for i, g in enumerate(gold[1200:]):
        parts.append(g + ("\r\n" if i % 7 == 0 else "\n"))
        if i % 11 == 0:
            parts.append("\n" if i % 2 else "\r\n")  # empty lines
    data = ("".join(parts[:100]) + long_line + "\n" + "".join(parts[100:])).encode()
    data = data.rstrip(b"\n")  # an unterminated last line
    return p, o, data


@pytest.mark.parametrize("chunk", ["64", "1000", "65536", "300000"])
def test_synthetic_corpus(synthetic, monkeypatch, chunk):
    p, o, data = synthetic
    assert data.count(b"/") > 1000 and data.count(b"\\") > 100 and b"\r\n" in data
    monkeypatch.setenv("VPT_CHUNK_BYTES", chunk)
    for no_norm, predict_tags in itertools.product((False, True), (False, True)):
        got = _check(p, o, data, no_norm, "", predict_tags)
        assert got["fp"] > 0 and got["fn"] > 0
        assert got["n_cor"] < got["n_sys"]


def test_predict_output_evaluates_perfectly(monkeypatch):
    """The tokenized output of vpt_tokenize_lines, evaluated with the same flags, is the system's own prediction."""
    from vpt_testlib import synth
    mb = synth.gen_model_bccwj_shaped(n_patterns=5000, sample_sentences=20000)
    p = vb.Predictor(vb.Model.read(mb))
    text, offs, _ = synth.gen_text(4000, 40, seed=synth.TEXT_SEED + 5)
    data = b"\n".join(text[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)) + b"\nA b/c\\d\n"
    assert b"\r" not in data
    monkeypatch.setenv("VPT_CHUNK_BYTES", "20000")
    for no_norm, wsconst in itertools.product((False, True), ("", "KG")):
        out, nl = p.tokenize_lines(data, no_norm=no_norm, wsconst=wsconst)
        got = p.evaluate_lines(out.tobytes(), no_norm=no_norm, wsconst=wsconst)
        assert got["n_lines"] == nl and got["n_sentences"] == nl
        assert got["fp"] == got["fn"] == 0 and got["tp"] > 0
        assert got["n_cor"] == got["n_sys"] == got["n_ref"]


BAD_LINES = [" a", "a  b", "/a", "a /b", "a\0b", "a/b\0", "a\\\0", "ab ", "\\", b"a\xffb", b"\xe3\x81", b"\\\xe3\\\x81\x82"]


@pytest.mark.parametrize("bad", BAD_LINES)
def test_first_error_in_a_later_chunk(docs, monkeypatch, bad):
    p, o = docs
    good = open(DOCS, "rb").read().split(b"\n")[0]
    bad = bad.encode() if isinstance(bad, str) else bad
    lines = [good] * 40 + [b""] + [good] * 9 + [bad] + [good] * 5 + [b"a  b"] + [good] * 3
    data = b"\n".join(lines) + b"\n"
    with pytest.raises(eo.GoldError) as want:
        eo.evaluate_lines(o, data)
    assert want.value.line == 50
    monkeypatch.setenv("VPT_CHUNK_BYTES", "1000")
    for predict_tags in (False, True):
        with pytest.raises(vb.VaporettoError) as got:
            p.evaluate_lines(data, predict_tags=predict_tags)
        assert got.value.code == want.value.code and str(got.value) == want.value.msg


def test_rejected_flags(docs):
    p, _ = docs
    with pytest.raises(vb.VaporettoError) as e:
        vb.Predictor(vb.Model.read(open(MODEL, "rb").read())).evaluate_lines(b"a b\n", predict_tags=True)
    assert e.value.code == 2
    with pytest.raises(vb.VaporettoError):
        p.evaluate_lines(b"a b\n", wsconst="X")
    rc = vb.lib().vpt_evaluate_lines(p._h, b"a", 1, 0, 1, 0, None, None, 0)
    assert rc == 2


def test_empty_input(docs):
    p, _ = docs
    zero = dict.fromkeys(("n_lines", "n_sentences") + KEYS, 0)
    assert p.evaluate_lines(b"") == zero
    got, lc = p.evaluate_lines(b"\n\r\n", per_line=True)
    assert got == dict(zero, n_lines=2) and lc.tolist() == [[0] * 7] * 2
    for metric in ("char", "word"):
        out = subprocess.run([sys.executable, CLI, "--model", MODEL, "--metric", metric], input=b"", capture_output=True)
        assert out.returncode == 0, out.stderr.decode()
        assert out.stdout.decode().split("\n")[:3] == ["Precision: NaN", "Recall: NaN", "F1: NaN"]


def test_cli_end_to_end():
    docs = open(DOCS, "rb").read()

    def run(*args):
        out = subprocess.run([sys.executable, CLI, "--model", MODEL, *args], input=docs, capture_output=True)
        assert out.returncode == 0, out.stderr.decode()
        assert out.stderr.decode().splitlines() == ["Loading model file...", "Start tokenization"]
        return out.stdout.decode()

    perfect = "Precision: 1\nRecall: 1\nF1: 1\n"
    assert run() == perfect + "TP: 7, TN: 7, FP: 0, FN: 0\n"
    assert run("--no-norm", "--predict-tags") == perfect + "TP: 7, TN: 7, FP: 0, FN: 0\n"
    assert run("--metric", "word", "--predict-tags") == perfect
    assert run("--metric", "word", "--no-norm") == perfect
    assert run("--metric", "word") == "Precision: 0\nRecall: 0\nF1: NaN\n"
    assert run("--wsconst", "K") == "Precision: 1\nRecall: 0.8571428571428571\nF1: 0.923076923076923\nTP: 6, TN: 7, FP: 0, FN: 1\n"
    bad = subprocess.run([sys.executable, CLI, "--model", MODEL], input=b"a  b\n", capture_output=True)
    assert bad.returncode == 1 and b"consecutive whitespaces (line 0)" in bad.stderr
