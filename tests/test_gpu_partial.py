"""Partially annotated lines on the device (vpt_tokenize_partial_lines, the partial line stream, tools/predict_cli.py
--partial-annotation), byte for byte against the CPU oracle of tests/native/partial_oracle.cpp: the reference's
from_partial_annotation restated, then predict, the wsconst post-filters, the caller's markers, fill_tags and
PatternMatchTagger over the oracle's Sentence and Predictor."""
import os
import random
import subprocess
import sys
import zlib

import pytest

import vaporetto_b200 as vb
from vpt_testlib import synth
from vpt_testlib import tag_rules as tr
from vpt_testlib.partial_oracle import PartialOracle

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GRID = [(n, w, t, r) for n in (False, True) for w in ("", "K", "GD") for t in (False, True) for r in (False, True)]
GRID_IDS = ["%s-%s-%s-%s" % ("nonorm" if n else "norm", w or "none", "tags" if t else "notags", "rules" if r else "norules")
            for n, w, t, r in GRID]
TAG_CHARS = ["x", "名詞", " ", "-", "|", "/", "\\", "é", "𠮷"]


def _synth():
    mb = synth.gen_model_bccwj_shaped(n_patterns=30_000, sample_sentences=50_000, tag_models=1_500)
    text, offs, _ = synth.gen_text(400, 40, seed=synth.TEXT_SEED + 7)
    return mb, [bytes(text[int(offs[i]):int(offs[i + 1])]).decode() for i in range(len(offs) - 1)]


MODELS = {
    "model.bin": lambda: (open(os.path.join(HERE, "golden", "model.bin"), "rb").read(),
                          ["まぁ社長は火星猫だ", "まぁ良いだろう", "火星", "社長は社長だ" * 30, "Vaporetto 1.5 と猫",
                           "a-b|c d/e\\f", "東京特許許可局", "ＡＢＣ１２３漢字かなカナ"] * 12),
    "synth": _synth,
}


@pytest.fixture(scope="module", params=sorted(MODELS))
def setup(request):
    mb, sents = MODELS[request.param]()
    assert tr.model_tags_nonempty(mb)
    return request.param, vb.Predictor(vb.Model.read(mb), predict_tags=True), PartialOracle(mb, predict_tags=True), sents


def esc(s: str) -> str:
    return "".join("\\" + c if c in " -|/\\" else c for c in s)


def annotate(sent: str, frac: float, rng, tag_fields: bool = True) -> str:
    """A partially annotated line of `sent`: a share `frac` of the markers given ('|' or '-'), the rest ' ', random
    escaped input tag fields, sometimes a trailing '\\'."""
    out = []
    for i, c in enumerate(sent):
        out.append(c)
        if tag_fields and rng.random() < 0.15:
            for _ in range(rng.randint(1, 3)):
                out.append("/" + esc("".join(rng.choice(TAG_CHARS) for _ in range(rng.randint(0, 3)))))
        if i + 1 < len(sent):
            out.append(rng.choice("|-") if rng.random() < frac else " ")
    if rng.random() < 0.05:
        out.append("\\")
    return "".join(out)


def rules_for(o, data: bytes, no_norm: bool):
    """Rules for tokens the oracle's tagged output holds, plus one that never matches."""
    out, _, _ = o.lines(data, no_norm=no_norm, predict_tags=True)
    seen = []
    for line in out.decode().split("\n"):
        for s, _ in tr.parse_tokenized_line(line) if line else []:
            if s not in seen:
                seen.append(s)
    fw = lambda s: "".join(chr(vb.lib().vpt_kytea_fullwidth(ord(c))) for c in s)
    rules = {(s if no_norm else fw(s)): ["R" + str(k % 3), None, "ルール"][: 1 + k % 3] for k, s in enumerate(seen[:40])}
    rules["nomatch"] = ["z"]
    return rules


def run(p, o, data, no_norm, wsconst, tags, rules):
    tagger = vb.PatternMatchTagger(p, rules) if rules else None
    got, nl = p.tokenize_partial_lines(data, no_norm=no_norm, wsconst=wsconst, predict_tags=tags, tag_rules=tagger)
    want, wl, err = o.lines(data, no_norm=no_norm, wsconst=wsconst, predict_tags=tags, rules=rules)
    assert err is None, err
    return got.tobytes(), nl, want, wl


@pytest.mark.parametrize("no_norm,wsconst,tags,use_rules", GRID, ids=GRID_IDS)
def test_oracle(setup, no_norm, wsconst, tags, use_rules):
    name, p, o, sents = setup
    rng = random.Random(zlib.crc32(f"{name} {no_norm} {wsconst} {tags} {use_rules}".encode()))
    lines = [annotate(s, frac, rng) for frac in (0.0, 0.3, 1.0) for s in sents]
    rng.shuffle(lines)
    data = ("\n".join(lines[:100]) + "\n\n" + "\r\n".join(lines[100:]) + "\r\n" + "猫|だ").encode()
    rules = rules_for(o, data, no_norm) if use_rules else None
    got, nl, want, wl = run(p, o, data, no_norm, wsconst, tags, rules)
    assert nl == wl == len(lines) + 2
    assert got == want


@pytest.mark.parametrize("no_norm,wsconst,tags,use_rules", GRID, ids=GRID_IDS)
def test_unknown_markers_are_plain_prediction(setup, no_norm, wsconst, tags, use_rules):
    name, p, o, sents = setup
    rng = random.Random(zlib.crc32(f"u {name} {no_norm} {wsconst}".encode()))
    raw = "\n".join(sents).encode() + b"\n"
    data = "\n".join(annotate(s, 0.0, rng) for s in sents).encode() + b"\n"
    rules = rules_for(o, data, no_norm) if use_rules else None
    tagger = vb.PatternMatchTagger(p, rules) if rules else None
    got, nl = p.tokenize_partial_lines(data, no_norm=no_norm, wsconst=wsconst, predict_tags=tags, tag_rules=tagger)
    plain, pl = p.tokenize_lines(raw, no_norm=no_norm, wsconst=wsconst, predict_tags=tags, tag_rules=tagger)
    assert nl == pl and got.tobytes() == plain.tobytes()


@pytest.mark.parametrize("no_norm", [False, True])
@pytest.mark.parametrize("wsconst", ["", "K", "GD", "DRHTKO"])
def test_round_trip(setup, no_norm, wsconst):
    """Every marker given from a tokenize_lines_tags output reproduces it, whatever post-filters the call runs."""
    name, p, o, sents = setup
    raw = "\n".join(sents).encode() + b"\n"
    ref, _ = p.tokenize_lines(raw, no_norm=no_norm, predict_tags=True)
    lines = []
    for line in ref.tobytes().decode().split("\n")[:-1]:
        toks = tr.parse_tokenized_line(line)
        parts = []
        for k, (surface, tags) in enumerate(toks):
            parts.append("-".join(surface) + "".join("/" + esc(t or "") for t in tags))
        lines.append("|".join(parts))
    got, nl = p.tokenize_partial_lines(("\n".join(lines) + "\n").encode(), no_norm=no_norm, wsconst=wsconst,
                                       predict_tags=True)
    assert nl == len(sents) and got.tobytes() == ref.tobytes()


BAD = [("nul", "猫-\0|だ", 2, "must not contain NULL"),
       ("boundary", "猫?だ", 2, "contains an invalid boundary character: '?'"),
       ("boundary_wide", "猫𠮷だ", 2, "contains an invalid boundary character: '𠮷'"),
       ("escaped_marker", "猫\\|だ", 2, "contains an invalid boundary character: '|'"),
       ("end", "猫|だ|", 2, "invalid annotation"),
       ("utf8", b"\xe7\x8c|\xff", 5, "stream did not contain valid UTF-8")]


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("bad", BAD, ids=[b[0] for b in BAD])
def test_errors(setup, monkeypatch, bad, where):
    name, p, o, sents = setup
    monkeypatch.setenv("VPT_CHUNK_BYTES", "4096")
    rng = random.Random(7)
    good = [annotate(s, 0.3, rng).encode() for s in sents] * 4
    line = bad[1] if isinstance(bad[1], bytes) else bad[1].encode()
    k = {"first": 0, "middle": len(good) // 2, "last": len(good)}[where]
    lines = good[:k] + [line] + good[k:]
    data = b"\n".join(lines) + b"\n"
    want, _, err = o.lines(data, predict_tags=True)
    assert err is not None and err[0] == bad[2] and err[1].endswith(f" (line {k})")
    with pytest.raises(vb.VaporettoError) as e:
        p.tokenize_partial_lines(data, predict_tags=True)
    assert e.value.code == bad[2] and str(e.value) == err[1]
    if bad[2] == 2:
        assert str(e.value) == "InvalidArgumentError: partial_annotation_text: " + bad[3] + f" (line {k})"
    # the stream delivers a line-aligned prefix of the output, then the same error
    got = b""
    with p.line_stream("partial", predict_tags=True) as s:
        with pytest.raises(vb.VaporettoError) as e2:
            for i in range(0, len(data), 1000):
                got += s.feed(data[i:i + 1000])
            s.finish()
    assert str(e2.value) == err[1]
    assert want.startswith(got) and (got == b"" or got.endswith(b"\n"))


def test_edges(setup, monkeypatch):
    """Escape runs, '/', markers and 2-, 3-, 4-byte characters across bytes 126-129 of a line at every start offset
    mod 4, lines of one character and of many 128-byte steps, and groups and chunks cut everywhere."""
    name, p, o, sents = setup
    # each starts in character position and ends with a marker
    snippets = ["\\/x\\\\\\|y|", "/-/|\\ //\\-|", "é-あ|𠮷 ", "𠮷/é/𠮷\\\\|", "a/\\\\\\\\-", "あ/é/𠮷 ",
                "\\-\\|\\ "]
    lines = []
    for head in ("a\n", "a\\\n", "a-b\n", "a-b\\\n"):  # the line starts at every offset mod 4
        for pad in range(110, 132):
            for snip in snippets:
                # the snippet starts at byte `pad` of its line ("é-" is one byte longer than "a-")
                body = ("é-" if pad % 2 else "a-") + "a-" * (pad // 2 - 1) + snip + "c"
                lines.append(head + body)
    lines += ["a", "猫", "\\", "-"] + ["あ-" * 400 + "い", "𠮷|" * 300 + "a"]
    data = "\n".join(lines).encode() + b"\n"
    for chunk in (None, "64", "1000", "8191"):
        if chunk:
            monkeypatch.setenv("VPT_CHUNK_BYTES", chunk)
        for tags in (False, True):
            got, nl, want, wl = run(p, o, data, False, "", tags, None)
            assert nl == wl and got == want


def test_stream_cuts_and_cli(setup, tmp_path):
    name, p, o, sents = setup
    rng = random.Random(11)
    data = ("\r\n".join(annotate(s, 0.5, rng) for s in sents) + "\r\n\nl-a-s-t|行").encode()
    whole, nl = p.tokenize_partial_lines(data, predict_tags=True)
    for trial in range(4):
        cuts = sorted(rng.sample(range(1, len(data)), 40))
        cuts += [i for i in range(1, len(data)) if data[i - 1:i] == b"\r"][:5]  # between '\r' and '\n'
        cuts = sorted(set(cuts))
        out = b""
        with p.line_stream("partial", predict_tags=True) as s:
            lo = 0
            for c in cuts + [len(data)]:
                out += s.feed(data[lo:c])
                lo = c
            rest, sl = s.finish()
        assert out + rest == whole.tobytes() and sl == nl
    if name != "model.bin":
        return
    f = tmp_path / "in.txt"
    f.write_bytes(data)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "predict_cli.py"), "--model",
                        os.path.join(HERE, "golden", "model.bin"), "--partial-annotation", "--predict-tags"],
                       stdin=open(f, "rb"), capture_output=True, check=True)
    assert r.stdout == whole.tobytes()


def test_flags_refused(setup):
    name, p, o, sents = setup
    with pytest.raises(vb.VaporettoError) as e:
        vb._check(vb.lib().vpt_tokenize_partial_lines(p._h, None, b"a|b", 3, 0, 1, 0, None, 0, None, None))
    assert e.value.kind == "InvalidArgument" and "wsconst_types" in str(e.value)
    untagged = vb.Predictor(vb.Model.read(open(os.path.join(HERE, "golden", "model.bin"), "rb").read()))
    with pytest.raises(vb.VaporettoError) as e:
        untagged.tokenize_partial_lines(b"a|b\n", predict_tags=True)
    assert e.value.kind == "InvalidArgument" and "predict_tags = false" in str(e.value)
    with pytest.raises(vb.VaporettoError):
        p.line_stream("partial", scores=True)
