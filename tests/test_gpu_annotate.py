"""Partially annotated output on the device (vpt_annotate_lines, the annotate line stream, tools/predict_cli.py
--write-partial-annotation, the C++ wrapper), byte for byte against the CPU oracle of tests/native/annotate_oracle.cpp:
predict, the margin, the wsconst post-filters, fill_tags, PatternMatchTagger over iter_tokens and
write_partial_annotation_text over the oracle's Sentence and Predictor."""
import ctypes as C
import os
import random
import subprocess
import sys
import tempfile
import zlib

import numpy as np
import pytest

import vaporetto_b200 as vb
from vpt_testlib import synth
from vpt_testlib import tag_rules as tr
from vpt_testlib import weight_windows as ww
from vpt_testlib.annotate_oracle import AnnotateOracle
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.oracle import OraclePredictor

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MAXM = 2**31 - 1
GRID = [(n, w, t, r) for n in (False, True) for w in ("", "K", "GD") for t in (False, True) for r in (False, True)]
GRID_IDS = ["%s-%s-%s-%s" % ("nonorm" if n else "norm", w or "none", "tags" if t else "notags", "rules" if r else "norules")
            for n, w, t, r in GRID]


def _synth():
    mb = synth.gen_model_bccwj_shaped(n_patterns=30_000, sample_sentences=50_000, tag_models=1_500)
    text, offs, _ = synth.gen_text(400, 40, seed=synth.TEXT_SEED + 7)
    return mb, [bytes(text[int(offs[i]):int(offs[i + 1])]).decode() for i in range(len(offs) - 1)]


MODELS = {
    "model.bin": lambda: (open(os.path.join(HERE, "golden", "model.bin"), "rb").read(),
                          ["まぁ社長は火星猫だ", "まぁ良いだろう", "火星", "社長は社長だ" * 30, "Vaporetto 1.5 と猫",
                           "a-b|c d/e\\f", "東京特許許可局", "ＡＢＣ１２３漢字かなカナ", "ｶﾞｷﾞ゛ー〜 👍🏽 é"] * 12),
    "synth": _synth,
}


@pytest.fixture(scope="module", params=sorted(MODELS))
def setup(request):
    mb, sents = MODELS[request.param]()
    o = OraclePredictor(mb)
    sc = np.concatenate([o.predict(s)[0] for s in sents[:50]])
    mid = int(np.median(np.abs(sc)))  # about half of the boundaries inside the margin
    return (request.param, vb.Predictor(vb.Model.read(mb), predict_tags=True), AnnotateOracle(mb, predict_tags=True),
            sents, mid)


def shaped(sents, rng) -> bytes:
    """The sentences with one- and many-window lines, a line longer than a scoring tile, empty, NUL and invalid UTF-8
    lines, CRLF and an unterminated last line."""
    lines = list(sents) + ["あ" * 3000, "猫", "", "a\0b", "\xff"]
    rng.shuffle(lines)
    data = "\n".join(lines[:len(lines) // 2]) + "\n" + "\r\n".join(lines[len(lines) // 2:]) + "\r\n" + "最後の行"
    return data.encode("utf-8", "surrogateescape").replace("\xff".encode(), b"\xff")


def rules_for(p, data: bytes, no_norm: bool):
    """Rules for tokens the tagged output holds, plus one that never matches."""
    out, _ = p.tokenize_lines(data, no_norm=no_norm, predict_tags=True)
    seen = []
    for line in out.tobytes().decode(errors="replace").split("\n"):
        for s, _ in tr.parse_tokenized_line(line) if line else []:
            if s not in seen:
                seen.append(s)
    fw = lambda s: "".join(chr(vb.lib().vpt_kytea_fullwidth(ord(c))) for c in s)
    rules = {(s if no_norm else fw(s)): ["R" + str(k % 3), None, "ル-ル|/"][: 1 + k % 3] for k, s in enumerate(seen[:40])}
    rules["nomatch"] = ["z"]
    return rules


@pytest.mark.parametrize("no_norm,wsconst,tags,use_rules", GRID, ids=GRID_IDS)
def test_oracle(setup, no_norm, wsconst, tags, use_rules):
    name, p, o, sents, mid = setup
    rng = random.Random(zlib.crc32(f"{name} {no_norm} {wsconst} {tags} {use_rules}".encode()))
    data = shaped(sents, rng)
    rules = rules_for(p, data, no_norm) if use_rules else None
    tagger = vb.PatternMatchTagger(p, rules) if rules else None
    for m in (0, 1, mid, MAXM):
        got, nl = p.annotate_lines(data, m, no_norm=no_norm, wsconst=wsconst, predict_tags=tags, tag_rules=tagger)
        want, wl = o.lines(data, m, no_norm=no_norm, wsconst=wsconst, predict_tags=tags, rules=rules)
        assert nl == wl and got == want, m


def test_margin_zero_is_tokenize_lines(setup):
    """margin 0 leaves nothing Unknown: tokenize_lines' segmentation in the other format."""
    name, p, o, sents, mid = setup
    data = ("\n".join(sents) + "\n").encode()
    got, _ = p.annotate_lines(data, 0)
    ref, _ = p.tokenize_lines(data)
    for g, line in zip(got.decode().split("\n"), ref.tobytes().decode().split("\n")):
        toks = [s for s, _ in tr.parse_tokenized_line(line)] if line else []
        assert g == "|".join("-".join(t) for t in toks)


def test_from_raw_doctest_on_device(setup):
    name, p, o, sents, mid = setup
    if name != "model.bin":
        pytest.skip("the doctest's text")
    for tags in (False, True):
        got, _ = p.annotate_lines("まぁ良いだろう\n".encode(), MAXM, no_norm=True, predict_tags=tags)
        assert got.decode() == "ま ぁ 良 い だ ろ う\n"


def test_host_sentence_path(setup):
    """Every line as the host Sentence API writes it: predict, the margin through boundaries_mut, fill_tags (which skips
    the tokens next to an Unknown boundary), write_partial_annotation_text.  Some tokens lose the tags
    tokenize_lines_tags gives them, the known ones keep theirs."""
    name, p, o, sents, mid = setup
    uniq = list(dict.fromkeys(sents))[:60]
    data = ("\n".join(uniq) + "\n").encode()
    got, _ = p.annotate_lines(data, mid, no_norm=True, predict_tags=True)
    zero, _ = p.annotate_lines(data, 0, no_norm=True, predict_tags=True)
    for g, line in zip(got.decode().split("\n"), uniq):
        s = vb.Sentence.from_raw(line)
        p.predict(s)
        sc = s.boundary_scores()
        bd = s.boundaries_mut()
        for i in range(len(bd)):
            if -mid < int(sc[i]) < mid:
                bd[i] = vb.CharacterBoundary.Unknown
        s.fill_tags()
        assert s.write_partial_annotation_text() == g
    assert got.count(b"/") < zero.count(b"/")
    assert got.count(b"/") > 0 or name != "model.bin"


@pytest.mark.parametrize("bias", [0, 2**31 - 40, -2**31 + 40], ids=["bias0", "wrap_hi", "wrap_lo"])
def test_margin_edges(bias):
    """Models whose scores land on +-margin, +-(margin - 1), 0 and on wrapped i32 sums: every margin taken from the
    scores, against the oracle."""
    md = ww.build_model(3, rows=((-3, 0),), bias=bias, seed=abs(bias) % 97, n_per_len=8)
    mb = encode_model(md)
    o, ao = OraclePredictor(mb), AnnotateOracle(mb)
    p = vb.Predictor(vb.Model.read(mb))
    rng = random.Random(bias)
    sents = ["".join(rng.choice(ww.PAT + ww.FILL) for _ in range(rng.randint(1, 60))) for _ in range(80)]
    data = ("\n".join(sents) + "\n").encode()
    scores = sorted({int(x) for s in sents for x in o.predict(s)[0]})
    margins = {0, 1, MAXM}
    for s in scores[:: max(len(scores) // 12, 1)] + [0]:
        a = abs(s) if s != -2**31 else MAXM
        margins |= {a, min(a + 1, MAXM)}
    for m in sorted(margins):
        got, _ = p.annotate_lines(data, m, no_norm=True)
        want, _ = ao.lines(data, m, no_norm=True)
        assert got == want, m
    if bias:
        assert any(abs(s) > 2**30 for s in scores)


@pytest.mark.parametrize("wsconst", ["", "K"])
def test_round_trip(setup, wsconst):
    """tokenize_partial_lines(annotate_lines(x, m)) == tokenize_lines(x) for every m (with tags on model.bin; the
    synthetic model's tag strings hold marker characters, so it runs without tags)."""
    name, p, o, sents, mid = setup
    tags = name == "model.bin"
    data = ("\n".join(sents) + "\n\n").encode()
    ref, _ = p.tokenize_lines(data, predict_tags=tags)
    for m in (0, 1, mid, MAXM):
        ann, _ = p.annotate_lines(data, m, predict_tags=tags)
        back, _ = p.tokenize_partial_lines(ann, predict_tags=tags)
        assert back.tobytes() == ref.tobytes(), m
    if wsconst:
        # the post-filters decide what they clear in both calls alike
        ref, _ = p.tokenize_lines(data, wsconst=wsconst)
        ann, _ = p.annotate_lines(data, mid, wsconst=wsconst)
        back, _ = p.tokenize_partial_lines(ann, wsconst=wsconst)
        assert back.tobytes() == ref.tobytes()


def test_stream_cuts_capacity_and_cli(setup, tmp_path):
    name, p, o, sents, mid = setup
    rng = random.Random(13)
    data = shaped(sents, rng)
    whole, nl = p.annotate_lines(data, mid, predict_tags=True)
    for trial in range(3):
        cuts = sorted(set(rng.sample(range(1, len(data)), 40)))
        out = b""
        with p.line_stream("annotate", predict_tags=True, margin=mid) as s:
            lo = 0
            for c in cuts + [len(data)]:
                out += s.feed(data[lo:c])
                lo = c
            rest, sl = s.finish()
        assert out + rest == whole and sl == nl
    # too small an out_capacity: the size needed, and the same bytes with it
    n, k = C.c_uint64(), C.c_uint64()
    small = np.empty(16, np.uint8)
    rc = vb.lib().vpt_annotate_lines(p._h, None, data, len(data), 0, 0, 1, mid, small.ctypes.data, small.size,
                                     C.byref(n), C.byref(k))
    assert rc == 2 and n.value == len(whole)
    rc = vb.lib().vpt_annotate_lines(p._h, None, data, len(data), 0, 0, 1, -1, small.ctypes.data, small.size,
                                     C.byref(n), C.byref(k))
    assert rc == 2 and n.value == 0 and "margin" in vb.lib().vpt_last_error().decode()
    if name != "model.bin":
        return
    f = tmp_path / "in.txt"
    f.write_bytes(data)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "predict_cli.py"), "--model",
                        os.path.join(HERE, "golden", "model.bin"), "--write-partial-annotation", "--margin", str(mid),
                        "--predict-tags"], stdin=open(f, "rb"), capture_output=True, check=True)
    assert r.stdout == whole


def test_cpp_wrapper(setup, tmp_path):
    name, p, o, sents, mid = setup
    if name != "model.bin":
        pytest.skip("one model is enough for the wrapper")
    src = os.path.join(HERE, "native", "annotate_cpp_test.cpp")
    exe = os.path.join(tempfile.mkdtemp(), "annotate_cpp_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-o", exe, src,
                           "-L" + os.path.join(ROOT, "vaporetto_b200"), "-lvaporetto_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "vaporetto_b200")])
    model = os.path.join(HERE, "golden", "model.bin")
    r = subprocess.run([exe, model], capture_output=True, text=True)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr
    inp = tmp_path / "in.txt"
    text = ("\n".join(sents) + "\n").encode()
    inp.write_bytes(text)
    r = subprocess.run([exe, model, "gpu", str(inp), str(mid)], capture_output=True)
    assert r.returncode == 0, r.stderr
    want, _ = p.annotate_lines(text, mid, predict_tags=True)
    assert r.stdout == want
