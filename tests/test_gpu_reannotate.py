"""Re-annotation on the device (vpt_reannotate_lines, the reannotate line stream, tools/predict_cli.py
--partial-annotation --write-partial-annotation, the C++ wrapper), byte for byte against the CPU oracle of
tests/native/reannotate_oracle.cpp, and the properties that tie it to annotate_lines: its output is a fixed point, an
unannotated input is annotate_lines of its raw text, and fully given markers come out as given."""
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
from vpt_testlib.oracle import OracleError, OraclePredictor
from vpt_testlib.reannotate_oracle import ReannotateOracle

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MAXM = 2**31 - 1
GRID = [(n, w, t, r) for n in (False, True) for w in ("", "K", "GD") for t in (False, True) for r in (False, True)]
GRID_IDS = ["%s-%s-%s-%s" % ("nonorm" if n else "norm", w or "none", "tags" if t else "notags", "rules" if r else "norules")
            for n, w, t, r in GRID]
TAG_CHARS = ["x", "名詞", " ", "-", "|", "/", "\\", "é", "𠮷"]


def _synth():
    mb = synth.gen_model_bccwj_shaped(n_patterns=30_000, sample_sentences=50_000, tag_models=1_500)
    text, offs, _ = synth.gen_text(300, 40, seed=synth.TEXT_SEED + 11)
    return mb, [bytes(text[int(offs[i]):int(offs[i + 1])]).decode() for i in range(len(offs) - 1)]


MODELS = {
    "model.bin": lambda: (open(os.path.join(HERE, "golden", "model.bin"), "rb").read(),
                          ["まぁ社長は火星猫だ", "まぁ良いだろう", "火星", "社長は社長だ" * 30, "Vaporetto 1.5 と猫",
                           "東京特許許可局", "ＡＢＣ１２３漢字かなカナ", "ｶﾞｷﾞ゛ー〜 👍🏽 é"] * 10),
    "synth": _synth,
}


@pytest.fixture(scope="module", params=sorted(MODELS))
def setup(request):
    mb, sents = MODELS[request.param]()
    o = OraclePredictor(mb)
    sc = np.concatenate([o.predict(s)[0] for s in sents[:50]])
    mid = int(np.median(np.abs(sc)))  # about half of the boundaries inside the margin
    return (request.param, vb.Predictor(vb.Model.read(mb), predict_tags=True), ReannotateOracle(mb, predict_tags=True),
            sents, mid)


def esc(s: str) -> str:
    return "".join("\\" + c if c in " -|/\\" else c for c in s)


def annotate(sent: str, frac: float, rng, tag_share: float = 0.2) -> str:
    """A partially annotated line of `sent`: a share `frac` of the markers given ('|' or '-'), the rest ' ', random
    input tag fields (escapes, empty and trailing-empty fields), sometimes a trailing '\\'."""
    out = []
    for i, c in enumerate(sent):
        out.append(c)
        if rng.random() < tag_share:
            for _ in range(rng.randint(1, 3)):
                out.append("/" + esc("".join(rng.choice(TAG_CHARS) for _ in range(rng.randint(0, 3)))))
        if i + 1 < len(sent):
            out.append(rng.choice("|-") if rng.random() < frac else " ")
    if rng.random() < 0.05:
        out.append("\\")
    return "".join(out)


def shaped(sents, rng) -> bytes:
    """Given-marker shares 0, 0.3 and 1 with random tag fields, a line longer than a scoring tile, empty lines, CRLF
    and an unterminated last line."""
    lines = [annotate(s, frac, rng) for frac in (0.0, 0.3, 1.0) for s in sents]
    lines += [annotate("あ" * 3000, 0.3, rng), "猫", "", "", "猫/x\\/y//"]
    rng.shuffle(lines)
    h = len(lines) // 2
    return ("\n".join(lines[:h]) + "\n" + "\r\n".join(lines[h:]) + "\r\n" + "最-後/z の 行").encode()


def rules_for(p, sents, no_norm: bool, plain: bool = False):
    """Rules for tokens the tagged output of the sentences holds, plus one that never matches; `plain`: tags without
    ' ', '-', '|', '/' and '\\'."""
    out, _ = p.tokenize_lines(("\n".join(sents) + "\n").encode(), no_norm=no_norm, predict_tags=True)
    seen = []
    for line in out.tobytes().decode(errors="replace").split("\n"):
        for s, _ in tr.parse_tokenized_line(line) if line else []:
            if s not in seen:
                seen.append(s)
    fw = lambda s: "".join(chr(vb.lib().vpt_kytea_fullwidth(ord(c))) for c in s)
    third = "ルール" if plain else "ル-ル|/"
    rules = {(s if no_norm else fw(s)): ["R" + str(k % 3), None, third][: 1 + k % 3] for k, s in enumerate(seen[:40])}
    rules["nomatch"] = ["z"]
    return rules


@pytest.mark.parametrize("keep_tags", [True, False], ids=["keep", "drop"])
@pytest.mark.parametrize("no_norm,wsconst,tags,use_rules", GRID, ids=GRID_IDS)
def test_oracle(setup, no_norm, wsconst, tags, use_rules, keep_tags):
    name, p, o, sents, mid = setup
    rng = random.Random(zlib.crc32(f"{name} {no_norm} {wsconst} {tags} {use_rules} {keep_tags}".encode()))
    data = shaped(sents, rng)
    rules = rules_for(p, sents, no_norm) if use_rules else None
    tagger = vb.PatternMatchTagger(p, rules) if rules else None
    for m in (0, 1, mid, MAXM):
        got, nl = p.reannotate_lines(data, m, keep_tags, no_norm=no_norm, wsconst=wsconst, predict_tags=tags,
                                     tag_rules=tagger)
        want, wl = o.lines(data, m, keep_tags, no_norm=no_norm, wsconst=wsconst, predict_tags=tags, rules=rules)
        assert nl == wl and got == want, m


def test_windows(setup, monkeypatch):
    """Tag regions and escape pairs across bytes 126-129 of a line at every start offset mod 4 (the 128-byte steps and
    4-byte words of k_part_tags and k_pa_rewrite), lines of one character and of many steps, chunks cut everywhere."""
    name, p, o, sents, mid = setup
    snippets = ["/\\/x\\\\\\|y|", "//a//|", "/é/𠮷\\\\ ", "/\\\\\\\\-", "/あ/é/𠮷|", "/\\-\\|\\ -", "/ab/cd/ef "]
    lines = []
    for head in ("a\n", "a\\\n", "a-b\n", "a-b\\\n"):  # the line starts at every offset mod 4
        for pad in range(110, 132):
            for snip in snippets:
                body = ("é-" if pad % 2 else "a-") + "a-" * (pad // 2 - 1) + "猫" + snip + "c"
                lines.append(head + body)
    lines += ["a", "猫/x", "a/b/c", "あ-" * 400 + "い/y", "𠮷|" * 300 + "a/\\/"]
    data = "\n".join(lines).encode() + b"\n"
    for chunk in (None, "64", "1000", "8191"):
        if chunk:
            monkeypatch.setenv("VPT_CHUNK_BYTES", chunk)
        for tags in (False, True):
            for m in (0, mid):
                got, nl = p.reannotate_lines(data, m, predict_tags=tags)
                want, wl = o.lines(data, m, predict_tags=tags)
                assert nl == wl and got == want, (chunk, tags, m)


BAD = [("nul", "猫-\0|だ", 2), ("boundary", "猫?だ", 2), ("boundary_wide", "猫𠮷だ", 2),
       ("escaped_marker", "猫\\|だ", 2), ("end", "猫|だ|", 2), ("utf8", b"\xe7\x8c|\xff", 5)]


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("bad", BAD, ids=[b[0] for b in BAD])
def test_errors(setup, monkeypatch, bad, where):
    """A malformed line stops the call with tokenize_partial_lines' error and line number."""
    name, p, o, sents, mid = setup
    monkeypatch.setenv("VPT_CHUNK_BYTES", "4096")
    rng = random.Random(7)
    good = [annotate(s, 0.3, rng).encode() for s in sents] * 3
    line = bad[1] if isinstance(bad[1], bytes) else bad[1].encode()
    k = {"first": 0, "middle": len(good) // 2, "last": len(good)}[where]
    data = b"\n".join(good[:k] + [line] + good[k:]) + b"\n"
    with pytest.raises(vb.VaporettoError) as ref:
        p.tokenize_partial_lines(data, predict_tags=True)
    assert ref.value.code == bad[2] and str(ref.value).endswith(f" (line {k})")
    for keep in (True, False):
        with pytest.raises(vb.VaporettoError) as e:
            p.reannotate_lines(data, mid, keep, predict_tags=True)
        assert e.value.code == bad[2] and str(e.value) == str(ref.value)
    # the stream delivers a line-aligned prefix of the output, then the same error
    got = b""
    with p.line_stream("reannotate", predict_tags=True, margin=mid) as s:
        with pytest.raises(vb.VaporettoError) as e2:
            for i in range(0, len(data), 1000):
                got += s.feed(data[i:i + 1000])
            s.finish()
    assert str(e2.value) == str(ref.value)
    with pytest.raises(OracleError) as oe:
        o.lines(data, mid, predict_tags=True)
    assert oe.value.message == str(ref.value)
    assert oe.value.output.startswith(got) and (got == b"" or got.endswith(b"\n"))


@pytest.mark.parametrize("wsconst", ["", "K"])
def test_fixed_point(setup, wsconst):
    """reannotate_lines(annotate_lines(x, m), m) == annotate_lines(x, m), with the input tags kept or predicted again
    (tags on model.bin only: the synthetic model's tag strings hold marker characters; rules with plain tags)."""
    name, p, o, sents, mid = setup
    tags = name == "model.bin"
    data = ("\n".join(sents) + "\n\n").encode()
    tagger = vb.PatternMatchTagger(p, rules_for(p, sents, False, plain=True)) if tags else None
    tagged = False
    for m in (0, 1, mid, MAXM):
        ann, _ = p.annotate_lines(data, m, wsconst=wsconst, predict_tags=tags, tag_rules=tagger)
        tagged |= b"/" in ann
        for keep in (True, False):
            again, _ = p.reannotate_lines(ann, m, keep, wsconst=wsconst, predict_tags=tags, tag_rules=tagger)
            assert again == ann, (m, keep)
    assert tagged or not tags


def test_unannotated_input(setup):
    """An all-' ' untagged input is annotate_lines of its raw text."""
    name, p, o, sents, mid = setup
    raw = ("\n".join(sents) + "\n").encode()
    pa = ("\n".join(" ".join(s) for s in sents) + "\n").encode()
    for m in (0, 1, mid, MAXM):
        for wsconst in ("", "K"):
            want, _ = p.annotate_lines(raw, m, wsconst=wsconst, predict_tags=True)
            got, _ = p.reannotate_lines(pa, m, wsconst=wsconst, predict_tags=True)
            assert got == want, (m, wsconst)


def test_fully_given_input(setup):
    """With every marker given the markers come out exactly as given, whatever the margin and post-filters."""
    name, p, o, sents, mid = setup
    rng = random.Random(5)
    lines = [annotate(s, 1.0, rng, tag_share=0.0) for s in sents]
    lines = [ln[:-1] if ln.endswith("\\") else ln for ln in lines]
    data = ("\n".join(lines) + "\n").encode()
    for m in (0, mid, MAXM):
        for wsconst in ("", "K", "GD"):
            got, _ = p.reannotate_lines(data, m, wsconst=wsconst)
            assert got == data, (m, wsconst)
    # with tags: the markers are unchanged
    got, _ = p.reannotate_lines(data, mid, predict_tags=True)
    strip = lambda b: [("".join(c for c in ln if c in " |-")) for ln in b.decode().split("\n")]
    if name == "model.bin":
        assert strip(got) == strip(data)


def test_stream_pieces_and_cli(setup, tmp_path):
    name, p, o, sents, mid = setup
    rng = random.Random(13)
    data = shaped(sents, rng)
    whole, nl = p.reannotate_lines(data, mid, predict_tags=True)
    for trial in range(3):
        cuts = sorted(set(rng.sample(range(1, len(data)), 40)))
        out = b""
        with p.line_stream("reannotate", predict_tags=True, margin=mid) as s:
            lo = 0
            for c in cuts + [len(data)]:
                out += s.feed(data[lo:c])
                lo = c
            rest, sl = s.finish()
        assert out + rest == whole and sl == nl
    dropped, _ = p.reannotate_lines(data, mid, False, predict_tags=True)
    with p.line_stream("reannotate", predict_tags=True, margin=mid, keep_tags=False) as s:
        out = b"".join(s.feed(data[i:i + 999]) for i in range(0, len(data), 999))
        rest, _ = s.finish()
    assert out + rest == dropped
    with pytest.raises(vb.VaporettoError):
        p.reannotate_lines(data, -1)
    if name != "model.bin":
        return
    f = tmp_path / "in.txt"
    f.write_bytes(data)
    cli = [sys.executable, os.path.join(ROOT, "tools", "predict_cli.py"), "--model",
           os.path.join(HERE, "golden", "model.bin"), "--partial-annotation", "--write-partial-annotation", "--margin",
           str(mid), "--predict-tags"]
    r = subprocess.run(cli, stdin=open(f, "rb"), capture_output=True, check=True)
    assert r.stdout == whole
    r = subprocess.run(cli + ["--drop-input-tags"], stdin=open(f, "rb"), capture_output=True, check=True)
    assert r.stdout == dropped


def test_cpp_wrapper(setup, tmp_path):
    name, p, o, sents, mid = setup
    if name != "model.bin":
        pytest.skip("one model is enough for the wrapper")
    src = os.path.join(HERE, "native", "reannotate_cpp_test.cpp")
    exe = os.path.join(tempfile.mkdtemp(), "reannotate_cpp_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-o", exe, src,
                           "-L" + os.path.join(ROOT, "vaporetto_b200"), "-lvaporetto_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "vaporetto_b200")])
    rng = random.Random(3)
    text = ("\n".join(annotate(s, 0.3, rng) for s in sents) + "\n").encode()
    inp = tmp_path / "in.txt"
    inp.write_bytes(text)
    r = subprocess.run([exe, os.path.join(HERE, "golden", "model.bin"), str(inp), str(mid)], capture_output=True)
    assert r.returncode == 0, r.stderr
    keep, _ = p.reannotate_lines(text, mid, True, predict_tags=True)
    drop, _ = p.reannotate_lines(text, mid, False, predict_tags=True)
    assert r.stdout == keep + drop
