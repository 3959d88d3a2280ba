"""PatternMatchTagger rules in the tagged line path on the device (vpt_tokenize_lines_tags_rules, the line stream with
rules, tools/predict_cli.py --tag-rules), byte for byte against the filter restated from the reference source over the
oracle's tagged output (vpt_testlib.tag_rules.oracle_tokenize_lines).  Rules are drawn from the tokens the models actually produce: unknown tokens, known
tokens with empty tag slots and fully tagged ones, plus rules that never match."""
import ctypes as C
import os
import random
import subprocess
import sys
import zlib

import numpy as np
import pytest

import vaporetto_b200 as vb
from golden import reference_kat as kat
from vpt_testlib import synth, tag_edges as te
from vpt_testlib import tag_rules as tr
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.oracle import OraclePredictor

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(ROOT := os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import predict_cli  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
TAGS = ["", "x", "名詞", "a b", "s/l", "b\\s", "ｶﾅ/ 😀", "固有名詞-人名"]


def split_tokens(line: str):
    """The tokens of one output line (an unescaped ' ' separates them) as (surface, [tag or None])."""
    out, cur, esc = [], [], False
    for c in line:
        if esc:
            cur.append("\\" + c)
            esc = False
        elif c == "\\":
            esc = True
        elif c == " ":
            out.append("".join(cur))
            cur = []
        else:
            cur.append(c)
    if cur:
        out.append("".join(cur))
    return [predict_cli.parse_tag_rule(t, 1) for t in out]


def fullwidth(s: str) -> str:
    return "".join(chr(vb.lib().vpt_kytea_fullwidth(ord(c))) for c in s)


def draw_rules(o, data: bytes, n_tags: int, no_norm: bool, rng, n_pick=60):
    """Rules for tokens the oracle's tagged output holds (keys as the filter sees them), classes mixed, plus misses."""
    out, _ = o.tokenize_lines(data, no_norm=no_norm, predict_tags=True)
    toks = {}
    for line in out.decode().split("\n"):
        for s, tags in split_tokens(line):
            toks[s] = tags
    unknown = [s for s, t in toks.items() if not t]
    partial = [s for s, t in toks.items() if t and (len(t) < n_tags or None in t)]
    full = [s for s, t in toks.items() if t and len(t) == n_tags and None not in t]
    picked = set()
    for pool in (unknown, partial, full):
        picked |= set(rng.sample(pool, min(len(pool), n_pick // 3)))
    rules = {}
    for s in sorted(picked):
        key = s if no_norm else fullwidth(s)
        rules[key] = [rng.choice([None] + TAGS) for _ in range(rng.randint(0, n_tags + 1))]
    for k in range(10):  # never produced
        rules["nomatch%d" % k] = ["z"]
    rules["ABC"] = ["half"]  # a half-width key: matches only with no_norm
    return rules, (len(unknown), len(partial), len(full))


def lines_of(sents):
    """The sentences as lines, then half-width text, an empty line, rejected lines (invalid UTF-8, U+0000), "\r\n" and
    an unterminated last line."""
    return "\n".join(sents).encode() + "\nABC 123 ＡＢＣ★\n\n".encode() + b"\xffbad\na\x00b\r\n" + "猫★\r\nlast".encode()


def _synth():
    mb = synth.gen_model_bccwj_shaped(n_patterns=30_000, sample_sentences=50_000, tag_models=1_500)
    text, offs, _ = synth.gen_text(600, 40, seed=synth.TEXT_SEED + 5)
    return mb, [bytes(text[int(offs[i]):int(offs[i + 1])]).decode() for i in range(len(offs) - 1)]


def _edges():
    cases = te.edge_cases()
    return encode_model(te.model(cases)), [c.sentence for c in cases[:80]]


MODELS = {
    "predictor_test": lambda: (encode_model(kat.PREDICTOR_TEST_MODEL), ["この人は地球人だ", "地球人", "この人", "ABCは人"] * 20),
    "model.bin": lambda: (open(os.path.join(HERE, "golden", "model.bin"), "rb").read(),
                          ["まぁ社長は火星猫だ", "まぁ良いだろう", "火星", "社長は社長だ" * 30, "Vaporetto 1.5 と猫"] * 20),
    "synth": _synth,
    "tag_edges": _edges,
}


@pytest.fixture(scope="module", params=sorted(MODELS))
def setup(request):
    mb, sents = MODELS[request.param]()
    assert tr.model_tags_nonempty(mb)  # (the restated filter reads the oracle's output back)
    return request.param, vb.Predictor(vb.Model.read(mb), predict_tags=True), OraclePredictor(mb, predict_tags=True), sents


@pytest.mark.parametrize("no_norm", [False, True])
@pytest.mark.parametrize("wsconst", ["", "D", "KH", "G"])
def test_tokenize_lines_with_rules(setup, no_norm, wsconst):
    name, p, o, sents = setup
    rng = random.Random(zlib.crc32(f"{name} {no_norm} {wsconst}".encode()))
    data = lines_of(sents)
    rules, classes = draw_rules(o, data, o.n_tags, no_norm, rng)
    assert classes[0] > 0, classes  # unknown tokens are always there
    tagger = vb.PatternMatchTagger(p, rules)
    got, nl = p.tokenize_lines(data, no_norm=no_norm, wsconst=wsconst, predict_tags=True, tag_rules=tagger)
    want, wl = tr.oracle_tokenize_lines(o, data, rules, no_norm=no_norm, wsconst=wsconst)
    assert nl == wl
    assert got.tobytes() == want
    # (the rules supplied tags the model's output does not have)
    assert want != o.tokenize_lines(data, no_norm=no_norm, wsconst=wsconst, predict_tags=True)[0]


def test_no_rules_and_no_tags_change_nothing(setup):
    name, p, o, sents = setup
    data = lines_of(sents)
    plain, nl = p.tokenize_lines(data, predict_tags=True)
    empty = vb.PatternMatchTagger(p, {})
    got, gl = p.tokenize_lines(data, predict_tags=True, tag_rules=empty)
    assert got.tobytes() == plain.tobytes() and gl == nl
    rules, _ = draw_rules(o, data, o.n_tags, False, random.Random(2))
    tagger = vb.PatternMatchTagger(p, rules)
    untagged, _ = p.tokenize_lines(data)
    assert p.tokenize_lines(data, tag_rules=tagger)[0].tobytes() == untagged.tobytes()
    with p.line_stream(tag_rules=tagger) as s:
        out = s.feed(data) + s.finish()[0]
    assert out == untagged.tobytes()
    # the evaluate stream ignores them too
    with p.line_stream(kind="evaluate", predict_tags=True, tag_rules=tagger) as s:
        s.feed(b"\xe7\x8c\xab/x\n")
        assert s.finish() == p.evaluate_lines(b"\xe7\x8c\xab/x\n", predict_tags=True)
    # rules bound to another predictor are refused
    other = vb.Predictor(vb.Model.read(open(os.path.join(HERE, "golden", "model.bin"), "rb").read()), predict_tags=True)
    with pytest.raises(vb.VaporettoError) as e:
        other.tokenize_lines(data, predict_tags=True, tag_rules=tagger)
    assert e.value.kind == "InvalidArgument" and "another predictor" in str(e.value)


def test_predictor_without_tag_models():
    """n_tags == 0: the rules do nothing (predictor.rs:553-555)."""
    mb = encode_model(dict(kat.PREDICTOR_TEST_MODEL, tag_models=[]))
    p = vb.Predictor(vb.Model.read(mb), predict_tags=True)
    data = "この人は地球人だ\n人\n".encode()
    tagger = vb.PatternMatchTagger(p, {"人": ["x", "y"]})
    assert p.tokenize_lines(data, predict_tags=True, tag_rules=tagger)[0].tobytes() == \
        p.tokenize_lines(data, predict_tags=True)[0].tobytes()


@pytest.mark.parametrize("chunk", [None, "2048"])
def test_line_stream_with_rules(setup, chunk, monkeypatch):
    name, p, o, sents = setup
    if chunk:
        monkeypatch.setenv("VPT_CHUNK_BYTES", chunk)
    rng = random.Random(7)
    data = lines_of(sents * 3)
    rules, _ = draw_rules(o, data, o.n_tags, False, rng)
    tagger = vb.PatternMatchTagger(p, rules)
    whole, nl = p.tokenize_lines(data, predict_tags=True, tag_rules=tagger)
    parts = []
    with p.line_stream(predict_tags=True, tag_rules=tagger) as s:
        i = 0
        while i < len(data):
            k = rng.choice([1, 3, 17, 200, 4096])
            parts.append(s.feed(data[i:i + k]))
            i += k
            if rng.random() < 0.05:
                parts.append(s.flush())
        rest, sl = s.finish()
    assert b"".join(parts) + rest == whole.tobytes() and sl == nl


def test_long_surfaces_and_long_tags(monkeypatch):
    """Rules on tokens longer than any tag-model token, and a 64 KiB tag on a one-character surface over many chunks:
    the output is the oracle's, and each chunk's device output buffer is sized by the rule tags it matched."""
    mb = open(os.path.join(HERE, "golden", "model.bin"), "rb").read()
    p, o = vb.Predictor(vb.Model.read(mb), predict_tags=True), OraclePredictor(mb, predict_tags=True)
    line = "まぁ社長は火星猫だ★"  # (★: an unknown one-character token)
    long_lines = ["ヴァポレットヴァポレットヴァポレットヴァポレット" * 20, "x" * 3000]
    data = ("\n".join([line] * 300 + long_lines) + "\n").encode()
    out, _ = o.tokenize_lines(data, predict_tags=True)
    longest = max((s for ln in out.decode().split("\n") for s, _ in split_tokens(ln)), key=len)
    assert len(longest) > 100
    big = "猫" * (65536 // 3) + "x"
    rules = {"★": [None, big], fullwidth(longest): ["長い", "ナガイ"]}
    monkeypatch.setenv("VPT_CHUNK_BYTES", "4096")
    tagger = vb.PatternMatchTagger(p, rules)
    got, nl = p.tokenize_lines(data, predict_tags=True, tag_rules=tagger)
    want, wl = tr.oracle_tokenize_lines(o, data, rules)
    assert nl == wl and got.tobytes() == want
    assert want.count(big.encode()) == 300
    # exact output of the largest chunk plus fixed slack: the chunk cut at <= 4096 + one line, its lines carry at most
    # one 64 KiB tag each; sizing by the longest rule suffix would need 4096 x 64 KiB = 268 MB
    c = 4096 + len(line.encode()) + 1
    per_line = len(line.encode()) + 1 + 1 + len(big.encode()) + 1
    bound = 1.125 * (3 * c + c + 4 + c * 64 + (c // len(line.encode()) + 1) * per_line) + 256
    assert 0 < tagger.max_output() <= bound, (tagger.max_output(), bound)
    # the whole-buffer call reports the size it needs when the buffer is too small
    small = np.empty(1000, np.uint8)
    n, k = C.c_uint64(), C.c_uint64()
    t = np.frombuffer(data, np.uint8)
    rc = vb.lib().vpt_tokenize_lines_tags_rules(p._h, tagger._h, t.ctypes.data, t.size, 0, 0, small.ctypes.data,
                                                small.size, C.byref(n), C.byref(k))
    assert rc == 2 and n.value == len(want)


def test_predict_cli_with_rules(tmp_path):
    mb = os.path.join(HERE, "golden", "model.bin")
    o = OraclePredictor(open(mb, "rb").read(), predict_tags=True)
    data = ("まぁ社長は火星猫だ★\nまぁ良いだろう\nVaporetto 1.5 と猫\n\n火星猫★\n").encode()
    f = tmp_path / "rules.txt"
    f.write_text("猫//ネ\\/コ\n★/記号/ホ\\ シ\n良い/形容詞\n", encoding="utf-8")
    rules = {"猫": [None, "ネ/コ"], "★": ["記号", "ホ シ"], "良い": ["形容詞"]}
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "predict_cli.py"), "--model", mb, "--predict-tags",
                        "--tag-rules", str(f)], input=data, capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    want, _ = tr.oracle_tokenize_lines(o, data, rules)
    assert r.stdout == want and want.count("★/記号/ホ\\ シ".encode()) == 2
