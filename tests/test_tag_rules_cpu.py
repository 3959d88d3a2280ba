"""PatternMatchTagger rules on the CPU: the reference's own test of the filter as a known answer, the host rule table
(tag_rules.cpp) against a Python dict, the per-token suffix merge the tagged writer runs (tag_rules.hpp, built for the
host by tests/native/tag_rules_test.cpp) against a restatement of the filter from the reference source, the validation of
vpt_tag_rules_new, and the rule-file parser of tools/predict_cli.py --tag-rules."""
import ctypes as C
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import vaporetto_b200 as vb
from vpt_testlib import tag_rules as tr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import predict_cli  # noqa: E402

KAT = json.load(open(os.path.join(HERE, "golden", "pattern_match_tagger_kat.json"), encoding="utf-8"))


@pytest.fixture(scope="module")
def L():
    return tr.native_lib()


esc = tr.esc


def parse_tokenized(text: str):
    """Sentence::from_tokenized's tokens and tags (n_tags = the most tag fields of any token, missing ones None)."""
    toks = [predict_cli.parse_tag_rule(t, 1) for t in text.split(" ")]
    n = max(len(t) for _, t in toks)
    return [(s, t + [None] * (n - len(t))) for s, t in toks], n


def test_reference_known_answer(L):
    toks, n = parse_tokenized(KAT["input"])
    rules = {k: v for k, v in KAT["rules"]}
    assert tr.filter_tokens(toks, n, rules) == KAT["expected"]
    h = tr.HostRules(L, rules, n)
    assert " ".join(esc(s) + h.suffix(s, t) for s, t in toks) == KAT["expected"]


def test_oracle_lines_with_rules():
    """The restated filter over the oracle's tagged output: empty slots of unknown and known tokens are filled, predicted
    tags stay, keys match the full-width image unless no_norm, rejected lines stay empty."""
    from vpt_testlib.oracle import OraclePredictor
    mb = open(os.path.join(HERE, "golden", "model.bin"), "rb").read()
    assert tr.model_tags_nonempty(mb)
    o = OraclePredictor(mb, predict_tags=True)
    data = "火星猫だ★\n\xffx\nABC\n".encode("utf-8", "surrogateescape").replace(b"\xc3\xbf", b"\xff")
    rules = {"★": [None, "ホ シ", "x"], "猫": ["動物", "ネ"], "ＡＢＣ": ["全角"], "ABC": ["半角"]}
    out, nl = tr.oracle_tokenize_lines(o, data, rules)
    assert nl == 3 and out == "火星/名詞/カセー 猫/名詞/ネコ だ/助動詞/ダ ★//ホ\\ シ\n\nABC/全角\n".encode()
    out, _ = tr.oracle_tokenize_lines(o, data, rules, no_norm=True)
    assert out.endswith("\nABC/半角\n".encode())


def rand_text(rng, lo=1, hi=6):
    pools = ["abcXYZ019", "éßñΩж", "あいう漢字カナ", "🐈😀🀄"]  # 1- to 4-byte characters
    return "".join(rng.choice(rng.choice(pools)) for _ in range(rng.randint(lo, hi)))


@pytest.mark.parametrize("n_rules", [1, 5, 8, 200, 3000])
def test_host_table_matches_dict(L, n_rules):
    """Keys are found with their rule id, other strings are not; up to 8 rules share the smallest table (32 slots), where
    their home slots collide."""
    rng = random.Random(n_rules)
    keys = []
    seen = set()
    while len(keys) < n_rules:
        k = rand_text(rng)
        if k not in seen:
            seen.add(k)
            keys.append(k)
    h = tr.HostRules(L, [(k, ["t"]) for k in keys], 2)
    if n_rules <= 8:
        assert L.tr_capacity(h.h) == 32
    for i, k in enumerate(keys):
        assert h.find(k) == i
    for _ in range(2000):
        q = rand_text(rng, 1, 7)
        assert h.find(q) == (keys.index(q) if q in seen else -1)


def test_host_table_normalised_matching(L):
    """With norm the token's KyteaFullwidthFilter image is looked up; keys are taken as given."""
    h = tr.HostRules(L, [("ＡＢＣ", ["full"]), ("xyz", ["half"]), ("", ["empty"]), ("a\0b", ["nul"])], 1)
    assert h.find("ABC", norm=True) == 0 and h.find("ABC") == -1 and h.find("ＡＢＣ") == 0
    assert h.find("xyz") == 1 and h.find("xyz", norm=True) == -1
    assert h.find("a\0b") == 3  # (never a token: lines with U+0000 are rejected)


TAGS = ["", "x", "名詞", "a b", "s/l", "b\\s", "ｶﾅ/ 😀"]


@pytest.mark.parametrize("n_tags", range(1, 9))
def test_suffix_merge_matches_oracle(L, n_tags):
    """Every combination per slot of model tag (absent, Some("") or text) and rule slot (absent, None, Some("") or
    text), through the writer's merge and through the restated filter + write_tokenized_text."""
    rng = random.Random(n_tags)
    for trial in range(300):
        surface = rand_text(rng, 1, 3) + ("/ \\"[trial % 3] if trial % 5 == 0 else "")
        model = None if trial % 7 == 0 else [rng.choice([None, None] + TAGS) for _ in range(n_tags)]
        n_rule = rng.randint(0, n_tags + 2)
        rule = [rng.choice([None] + TAGS) for _ in range(n_rule)]
        rules = {surface: rule} if trial % 11 else {surface + "_": rule}
        h = tr.HostRules(L, rules, n_tags)
        got = esc(surface) + h.suffix(surface, model)
        want = tr.filter_tokens([(surface, model or [None] * n_tags)], n_tags, rules)
        assert got == want, (surface, model, rules)


def test_rule_slots_are_clipped_to_n_tags(L):
    h = tr.HostRules(L, {"猫": ["a", "b", "c"]}, 2)
    assert h.suffix("猫", None) == "/a/b"
    h = tr.HostRules(L, {"猫": [None, "", None]}, 3)
    assert h.suffix("猫", None) == "//" and h.suffix("猫", ["m", None, None]) == "/m/"


@pytest.fixture(scope="module")
def host_predictor():
    data = open(os.path.join(HERE, "golden", "model.bin"), "rb").read()
    return vb.Predictor(vb.Model.read(data), predict_tags=True, device=-1)


def rules_new(p, n, surf, soff, qoff, slots, tags, tags_len):
    h = C.c_void_p()
    rc = vb.lib().vpt_tag_rules_new(p, n, surf, soff, qoff, slots, tags, tags_len, C.byref(h))
    return rc, vb.lib().vpt_last_error().decode(), h


@pytest.mark.parametrize("case,msg", [
    ({"a": ["x"], b"\xff": ["y"]}, "rule 1: surface is not valid UTF-8"),
    ({"a": ["x"], "b": [b"\xed\xa0\x80"]}, "rule 1: tag is not valid UTF-8"),        # a surrogate
    ({"a": [b"\xc0\xaf"]}, "rule 0: tag is not valid UTF-8"),                       # an overlong '/'
    ([("a", ["x"]), ("b", []), ("a", ["y"])], "rule 2: duplicate surface (also rule 0)"),
    ([("", []), ("", ["z"])], "rule 1: duplicate surface"),
])
def test_rules_new_rejects(host_predictor, L, case, msg):
    n, surf, soff, qoff, slots, tags, tags_len = tr.encode(case)
    rc, err, h = rules_new(host_predictor._h, n, surf.ctypes.data, soff.ctypes.data, qoff.ctypes.data, slots.ctypes.data,
                           tags.ctypes.data, tags_len)
    assert rc == 2 and msg in err and not h.value, err
    with pytest.raises(ValueError) as e:
        tr.HostRules(L, case, 2)
    assert e.value.args[0] == 2 and msg in e.value.args[1]


def test_rules_new_rejects_bad_arrays(host_predictor):
    n, surf, soff, qoff, slots, tags, tags_len = tr.encode({"ab": ["x", None], "c": ["yz"]})
    p = host_predictor._h
    args = [surf.ctypes.data, soff.ctypes.data, qoff.ctypes.data, slots.ctypes.data, tags.ctypes.data]
    for i, what in ((1, "must not be NULL"), (2, "must not be NULL"), (0, "surfaces must not be NULL"),
                    (3, "slots must not be NULL"), (4, "tags must not be NULL")):
        a = list(args)
        a[i] = None
        rc, err, _ = rules_new(p, n, *a, tags_len)
        assert rc == 2 and what in err, (i, err)
    bad = soff.copy()
    bad[2] = 1
    rc, err, _ = rules_new(p, n, surf.ctypes.data, bad.ctypes.data, *args[2:], tags_len)
    assert rc == 2 and "rule 1: surface_offsets must not decrease" in err
    bad = qoff.copy()
    bad[2] = 1
    rc, err, _ = rules_new(p, n, surf.ctypes.data, soff.ctypes.data, bad.ctypes.data, *args[3:], tags_len)
    assert rc == 2 and "rule 1: slot_offsets must not decrease" in err
    rc, err, _ = rules_new(p, n, *args, tags_len - 1)
    assert rc == 2 and "rule 1: tag outside the tag bytes" in err
    h = C.c_void_p()
    assert vb.lib().vpt_tag_rules_new(None, n, *args, tags_len, C.byref(h)) == 2
    assert vb.lib().vpt_tag_rules_new(p, n, *args, tags_len, None) == 2
    # valid rules on a predictor without a device: checked first, then refused for the missing device
    rc, err, h = rules_new(p, n, *args, tags_len)
    assert rc == 16 and not h.value and "without a CUDA device" in err
    rc, err, h = rules_new(p, 0, None, np.zeros(1, np.uint64).ctypes.data, np.zeros(1, np.uint64).ctypes.data, None, None, 0)
    assert rc == 16


def test_cli_rule_parser(tmp_path):
    P = predict_cli.parse_tag_rule
    assert P("猫/名詞/ネコ", 1) == ("猫", ["名詞", "ネコ"])
    assert P("猫//ネコ/", 1) == ("猫", [None, "ネコ", None])
    assert P("猫", 1) == ("猫", [])
    assert P(r"a\/b\ c/x\/y/\\", 1) == ("a/b c", ["x/y", "\\"])
    for bad, what in (("猫 犬", "line 3: one token per line"), ("/名詞", "line 3: empty surface"), ("", "line 3: empty surface")):
        with pytest.raises(ValueError, match=what):
            P(bad, 3)
    f = tmp_path / "rules.txt"
    f.write_bytes("ＡＢＣ/名詞/エービーシー\r\n猫//ネコ\n".encode())
    assert predict_cli.read_tag_rules(str(f)) == {"ＡＢＣ": ["名詞", "エービーシー"], "猫": [None, "ネコ"]}
    f.write_bytes("猫/a\n犬/b\n猫/c\n".encode())
    with pytest.raises(ValueError, match="line 3: duplicate surface"):
        predict_cli.read_tag_rules(str(f))
    # the option is checked before the model is read
    cli = os.path.join(ROOT, "tools", "predict_cli.py")
    r = subprocess.run([sys.executable, cli, "--model", "missing.bin", "--tag-rules", str(f)], capture_output=True, text=True)
    assert r.returncode == 2 and "--tag-rules needs --predict-tags" in r.stderr
    r = subprocess.run([sys.executable, cli, "--model", "missing.bin", "--predict-tags", "--tag-rules", str(f)],
                       capture_output=True, text=True)
    assert r.returncode == 2 and "line 3: duplicate surface" in r.stderr
    r = subprocess.run([sys.executable, cli, "--help"], capture_output=True, text=True)
    assert "--tag-rules" in r.stdout and "not in the reference CLI" in r.stdout
