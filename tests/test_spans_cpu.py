"""Token spans (vpt_token_spans) without a device: the kernels' window arithmetic (vaporetto_b200/csrc/spans.hpp) against
a byte-by-byte restatement, and the CPU oracle of vaporetto_tantivy's token_stream against the reference's known answers
and against a composition of ora_predict with literal filters.  The device side is tests/test_gpu_spans.py."""
import ctypes as C
import itertools
import os
import random
import subprocess

import numpy as np
import pytest

import vaporetto_b200 as vb
from golden import tantivy_kat as kat
from vpt_testlib import oracle
from vpt_testlib import spans_oracle as so
from vpt_testlib.bincode_model import encode_model

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
SRC = os.path.join(HERE, "native", "spans_test.cpp")

# characters the random documents are made of: kana, kanji, full-width-mapped ASCII, digits, emoji with ZWJ and skin
# tones, regional indicators, combining marks, and line breaks
ALPHABET = (list("あいうえおかきアイウエオ東京特許許可局社長火星猫") + list("abcXYZ012789.-/,!?()") + ["１", "２", "Ａ", "ｶ", "ﾞ"]
            + ["🤌", "🏿", "‍", "👩", "🇯", "🇵", "́", "。", "、", " ", "é"])
LINEBREAKS = ["\n", "\r", "\r\n", "\n\n", "\r\r\n"]


def random_doc(rng, n):
    out = []
    for _ in range(n):
        out.append(rng.choice(LINEBREAKS) if rng.random() < 0.12 else rng.choice(ALPHABET))
    return "".join(out)


def read(fn):
    with open(os.path.join(GOLDEN, fn), "rb") as f:
        return f.read()


def batch(docs):
    enc = [d if isinstance(d, bytes) else d.encode() for d in docs]
    off = np.zeros(len(enc) + 1, np.uint64)
    np.cumsum([len(e) for e in enc], out=off[1:])
    return b"".join(enc), off


def test_window_arithmetic(tmp_path):
    """The warp loops of k_split_linebreaks and k_token_ends over spans.hpp, lane by lane, equal SplitLinebreaksFilter and
    boundary_pos byte by byte: window edges, characters across them, runs of line breaks, one-character documents and
    tokens over several windows, at every start alignment."""
    exe = str(tmp_path / "spans_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-o", exe, SRC])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.startswith("spans ok")


@pytest.mark.parametrize("text,wsconst,tokens", kat.TANTIVY_TOKEN_STREAMS)
def test_oracle_tantivy_known_answers(text, wsconst, tokens):
    o = so.SpansOracle(read("tantivy_model.bin"))
    b, off = batch([text])
    r = o.token_spans(b, off, wsconst=wsconst)
    assert r["token_ends"].tolist() == [t[2] for t in tokens]
    assert r["n_tokens"].tolist() == [len(tokens)]
    assert r["status"].tolist() == [1 if text == "" else 0]


@pytest.mark.parametrize("text,tokens", kat.SPLIT_LINEBREAKS)
def test_oracle_split_linebreaks_known_answers(text, tokens):
    # a model that predicts no boundary at all: the sentence of Sentence::from_tokenized(text) in the reference's test
    m = dict(char_ngrams=[], type_ngrams=[], dict=[], bias=-1, char_window=1, type_window=1, tag_models=[])
    o = so.SpansOracle(encode_model(m))
    b, off = batch([text])
    r = o.token_spans(b, off, no_norm=True)
    ends = r["token_ends"].tolist()
    assert [b[f:t].decode() for f, t in zip([0] + ends[:-1], ends)] == tokens
    assert so.split_linebreaks(text, [0] * (len(text) - 1)) == [int(text[i] in "\r\n" or text[i + 1] in "\r\n")
                                                               for i in range(len(text) - 1)]


@pytest.mark.parametrize("model", ["tantivy_model.bin", "model.bin"])
def test_oracle_matches_composition(model):
    """ora_token_spans equals ora_predict on the pre-filtered text followed by literal restatements of the line-break
    split, the wsconst filters and boundary_pos, for every wsconst combination, normalised or not."""
    rng = random.Random(7)
    mb = read(model)
    o, ora = so.SpansOracle(mb), oracle.OraclePredictor(mb)
    docs = [random_doc(rng, rng.randrange(1, 60)) for _ in range(12)] + ["\n", "\r\n", "。\n", "a\r\nb", "🤌🏿\n🇯🇵"]
    b, off = batch(docs)
    for k in range(8):
        for combo in itertools.combinations("DRHTKOG", k):
            ws = "".join(combo)
            if k > 2 and rng.random() > 0.2:
                continue  # (a sample of the larger sets; all of them are covered on the device)
            for no_norm in (False, True):
                r = o.token_spans(b, off, no_norm=no_norm, wsconst=ws)
                base = 0
                for d, text in enumerate(docs):
                    want = so.compose(ora, text, no_norm=no_norm, wsconst=ws)
                    n = int(r["n_tokens"][d])
                    assert r["token_ends"][base:base + n].tolist() == want, (text, ws, no_norm)
                    base += n


def test_oracle_rejected_documents():
    o = so.SpansOracle(read("tantivy_model.bin"))
    b, off = batch(["東京", b"", "a\x00b", b"\xe3\x81", "a\x00" .encode() + b"\xff", "局"])
    r = o.token_spans(b, off)
    assert r["status"].tolist() == [0, 1, 2, 3, 3, 0]
    assert r["n_tokens"].tolist()[1:5] == [0, 0, 0, 0]


def test_tokenizer_wsconst_parse_without_device():
    """An unknown wsconst letter is the adapter's error (lib.rs:69-85); it is raised before any device work."""
    with pytest.raises(vb.VaporettoError) as e:
        vb.Tokenizer(None, "DX")
    assert str(e.value) == "Could not parse a wsconst value"
    vb.Tokenizer(None, "DRHTKOG")


def test_token_spans_abi_without_device():
    """The C call rejects a NULL predictor and a host-only one (there is no CPU fallback)."""
    L = vb.lib()
    n = np.zeros(1, np.uint32)
    st = np.zeros(1, np.uint8)
    ends = np.zeros(4, np.uint32)
    off = np.array([0, 3], np.uint64)
    total = C.c_uint64()
    assert L.vpt_token_spans(None, b"abc", off.ctypes.data, 1, 0, 0, n.ctypes.data, st.ctypes.data, ends.ctypes.data,
                             None, None, 4, C.byref(total)) == 2
    host_only = vb.Predictor(vb.Model.read(read("model.bin")), device=-1)
    with pytest.raises(vb.VaporettoError) as e:
        host_only.token_spans(b"abc", off)
    assert e.value.kind == "CudaError"
