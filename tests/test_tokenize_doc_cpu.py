"""The CPU oracle of vpt_tokenize_dev (tests/native/tokenize_doc_oracle.cpp) pinned without a device: for documents
without '\\n' it is the oracle's line loop (ora_tokenize_lines*) minus the '\\n', with and without tags and with
PatternMatchTagger rules, and it reproduces the reference's write_tokenized_text known answers.  The device side is
tests/test_gpu_tokenize_device.py."""
import os
import random

import numpy as np
import pytest

from golden import reference_kat as kat
from vpt_testlib import tag_rules as tr
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.oracle import OraclePredictor
from vpt_testlib.tokenize_doc_oracle import TokenizeDocOracle

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")

# kana, kanji, full-width-mapped ASCII, escaped bytes (' ', '/', '\\'), emoji with ZWJ, combining marks, '\r'
ALPHABET = (list("あいうえおかきアイウエオ東京特許許可局社長火星猫だはまぁ") + list("abcXYZ012789.-,!?()") +
            ["１", "２", "Ａ", "ｶ", "ﾞ", "🤌", "🏿", "‍", "👩", "́", "。", " ", "/", "\\", "é", "\r"])
RULE_TAGS = ["x", "名詞", "a b", "s/l", "b\\s", "ｶﾅ/ 😀"]


def read(fn):
    with open(os.path.join(GOLDEN, fn), "rb") as f:
        return f.read()


def docs_of(rng, n, max_len):
    """Documents without '\n' that do not end in '\r' (the line loop drops a '\r' in front of the '\n')."""
    return [("".join(rng.choice(ALPHABET) for _ in range(rng.randint(1, max_len)))).rstrip("\r") or "猫" for _ in range(n)]


def batch(docs):
    enc = [d if isinstance(d, bytes) else d.encode() for d in docs]
    off = np.zeros(len(enc) + 1, np.uint64)
    np.cumsum([len(e) for e in enc], out=off[1:])
    return b"".join(enc), off


def line_loop(o, docs, no_norm, wsconst, tags, rules=None):
    """The oracle's line loop over the documents joined by '\\n', cut back into one output per document."""
    data = b"".join(d.encode() + b"\n" for d in docs)
    if rules is not None:
        out, nl = tr.oracle_tokenize_lines(o, data, rules, no_norm=no_norm, wsconst=wsconst)
    else:
        out, nl = o.tokenize_lines(data, no_norm=no_norm, wsconst=wsconst, predict_tags=tags)
    assert nl == len(docs)
    lines = out.split(b"\n")
    assert lines[-1] == b""
    return lines[:-1]


@pytest.mark.parametrize("model,tags", [("model.bin", False), ("model.bin", True), ("tantivy_model.bin", False)])
@pytest.mark.parametrize("no_norm", [False, True])
@pytest.mark.parametrize("wsconst", ["", "D", "KHG"])
def test_equals_line_loop(model, tags, no_norm, wsconst):
    mb = read(model)
    rng = random.Random(f"{model} {tags} {no_norm} {wsconst}")
    docs = docs_of(rng, 150, 60)
    text, off = batch(docs)
    got, status = TokenizeDocOracle(mb, predict_tags=tags).tokenize_docs(text, off, no_norm, wsconst, tags)
    assert status.tolist() == [0] * len(docs)
    assert got == line_loop(OraclePredictor(mb, predict_tags=tags), docs, no_norm, wsconst, tags)


@pytest.mark.parametrize("no_norm", [False, True])
def test_equals_line_loop_with_rules(no_norm):
    mb = read("model.bin")
    assert tr.model_tags_nonempty(mb)
    rng = random.Random(f"rules {no_norm}")
    docs = docs_of(rng, 120, 40) + ["まぁ社長は火星猫だ", "火星 猫/社長\\は"]
    o = OraclePredictor(mb, predict_tags=True)
    toks = set()
    for ln in line_loop(o, docs, no_norm, "", True):
        toks.update(s for s, _ in tr.parse_tokenized_line(ln.decode()))
    pick = sorted(toks)
    rng.shuffle(pick)
    fw = lambda s: s if no_norm else "".join(chr(tr.oracle.lib().ora_kytea_fullwidth(ord(c))) for c in s)
    rules = {fw(s): [rng.choice(RULE_TAGS + [None]) for _ in range(rng.randint(1, o.n_tags + 1))] for s in pick[:80]}
    text, off = batch(docs)
    got, _ = TokenizeDocOracle(mb, predict_tags=True).tokenize_docs(text, off, no_norm, "", True, rules=rules)
    assert got == line_loop(o, docs, no_norm, "", True, rules=rules)
    assert got != TokenizeDocOracle(mb, predict_tags=True).tokenize_docs(text, off, no_norm, "", True)[0]


def test_rejected_documents_and_line_breaks():
    """Rejected documents are empty with the from_raw status; '\\r' and '\\n' stay characters of the sentence."""
    mb = read("tantivy_model.bin")
    docs = [b"", b"a\0b", b"\xff\xfe", "東京\n特許\r\n許可局".encode(), b"\n", b"\r\n"]
    text, off = batch(docs)
    got, status = TokenizeDocOracle(mb).tokenize_docs(text, off)
    assert status.tolist() == [1, 2, 3, 0, 0, 0]
    assert got[:3] == [b"", b"", b""]
    assert got[4] == b"\n" and got[5].replace(b" ", b"") == b"\r\n"
    assert got[3].replace(b" ", b"") == "東京\n特許\r\n許可局".encode()


def test_write_tokenized_text_known_answers():
    """write_tokenized_text of the reference's tests: the escape vector and the model.bin / tantivy known answers."""
    e = kat.TOKENIZED_ESCAPE
    got, _ = TokenizeDocOracle(encode_model(e["model"])).tokenize_docs(*batch([e["text"]]), no_norm=True)
    assert got == [e["tokenized"].encode()]
    mb = read("model.bin")
    for text, tags, want in kat.MODEL_BIN_TOKENIZE:
        got, _ = TokenizeDocOracle(mb, predict_tags=tags).tokenize_docs(*batch([text]), predict_tags=tags)
        assert got == [want.encode()]
    mb = read("tantivy_model.bin")
    for text, want in kat.TANTIVY_TOKENIZE:
        got, _ = TokenizeDocOracle(mb).tokenize_docs(*batch([text]))
        assert got == [want.encode()]
