"""The byte-window kernels on the device against the CPU oracles, byte for byte, on lines and documents whose features
sit exactly on the 128-byte window and 4-byte lane edges (vpt_testlib.window_edges; test_window_edges_cpu.py checks
that every case lands on its edge and is live).  Each entry point runs on all its cases in one call per flag setting."""
import itertools
import os

import numpy as np
import pytest
import torch

import vaporetto_b200 as vb
from vpt_testlib import eval_oracle as eo
from vpt_testlib import tag_rules as tr
from vpt_testlib import window_edges as we
from vpt_testlib.oracle import OraclePredictor
from vpt_testlib.spans_oracle import SpansOracle
from vpt_testlib.tokenize_doc_oracle import TokenizeDocOracle

pytestmark = pytest.mark.gpu

MODEL_BIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "model.bin")
WSCONST = ["", "DRHTKO", "G", "GD"]


@pytest.fixture(autouse=True)
def one_chunk(monkeypatch):
    # the line layouts are checked against the default chunk size (VPT_CHUNK_BYTES is read at every call)
    monkeypatch.delenv("VPT_CHUNK_BYTES", raising=False)


def _model_bytes(name):
    if name == "model.bin":
        return open(MODEL_BIN, "rb").read()
    return {"all": we.model_all, "none": we.model_none, "tag": we.model_tag}[name]()


TAGGED = {"tag", "model.bin"}


@pytest.fixture(scope="module", params=["all", "none", "tag", "model.bin"])
def model(request):
    mb = _model_bytes(request.param)
    tags = request.param in TAGGED
    return request.param, mb, vb.Predictor(vb.Model.read(mb), predict_tags=tags), OraclePredictor(mb, predict_tags=tags)


def _rules(no_norm):
    fw = (lambda s: s) if no_norm else (lambda s: "".join(chr(vb.lib().vpt_kytea_fullwidth(ord(c))) for c in s))
    return {fw(k): v for k, v in we.TAG_RULES.items()}


@pytest.mark.parametrize("no_norm", [False, True])
def test_tokenize_lines(model, no_norm):
    name, mb, p, o = model
    data, _ = we.line_buffer(we.line_cases())
    for wsconst in WSCONST:
        got, nl = p.tokenize_lines(data, no_norm=no_norm, wsconst=wsconst)
        want, wl = o.tokenize_lines(data, no_norm=no_norm, wsconst=wsconst)
        assert nl == wl and got.tobytes() == want, (name, no_norm, wsconst)
        if name not in TAGGED:
            continue
        got, nl = p.tokenize_lines(data, no_norm=no_norm, wsconst=wsconst, predict_tags=True)
        want, wl = o.tokenize_lines(data, no_norm=no_norm, wsconst=wsconst, predict_tags=True)
        assert nl == wl and got.tobytes() == want, (name, no_norm, wsconst, "tags")
        rules = _rules(no_norm)
        tagger = vb.PatternMatchTagger(p, rules)
        got, nl = p.tokenize_lines(data, no_norm=no_norm, wsconst=wsconst, predict_tags=True, tag_rules=tagger)
        want, wl = tr.oracle_tokenize_lines(o, data, rules, no_norm=no_norm, wsconst=wsconst)
        assert nl == wl and got.tobytes() == want, (name, no_norm, wsconst, "rules")
    if name == "tag":  # (the model's suffixes and the rules' tags are both in the output)
        assert want.count(we.TAG_SUFFIX.encode()) > 100 and want.count(b"r\\/1") > 100


def _to_dev(text: bytes, offs):
    t = torch.frombuffer(bytearray(text), dtype=torch.uint8).cuda()
    # a fresh allocation: the device offsets are the caller's (the device calls add the text's address mod 16)
    assert t.data_ptr() % 16 == 0
    return t, torch.as_tensor(np.asarray(offs, np.int64)).cuda()


@pytest.mark.parametrize("no_norm", [False, True])
def test_tokenize_device(model, no_norm):
    name, mb, p, _ = model
    text, offs, idx = we.doc_batch(we.doc_cases())
    td, od = _to_dev(text, offs)
    tags = [False, True] if name in TAGGED else [False]
    do = TokenizeDocOracle(mb, predict_tags=name in TAGGED)
    for wsconst, predict_tags in itertools.product(WSCONST, tags):
        chars, off, status = p.tokenize_device(td, od, no_norm=no_norm, wsconst=wsconst, predict_tags=predict_tags).to_host()
        b = chars.tobytes()
        got = [b[off[d]:off[d + 1]] for d in range(len(offs) - 1)]
        want, wst = do.tokenize_docs(text, offs, no_norm=no_norm, wsconst=wsconst, predict_tags=predict_tags)
        assert np.array_equal(status, wst) and not status.any()
        assert got == want, (name, no_norm, wsconst, predict_tags)


@pytest.mark.parametrize("no_norm", [False, True])
def test_token_spans(model, no_norm):
    name, mb, p, _ = model
    cases = we.span_cases() + we.grapheme_cases(docs=True) + [c for c in we.tok_cases() if c.kernel == "tok"]
    text, offs, idx = we.doc_batch(cases)
    td, od = _to_dev(text, offs)
    so = SpansOracle(mb, predict_tags=name in TAGGED)
    for wsconst in WSCONST:
        want = so.token_spans(text, offs, no_norm=no_norm, wsconst=wsconst)
        for r in (p.token_spans(text, offs, no_norm=no_norm, wsconst=wsconst),
                  p.token_spans_device(td, od, no_norm=no_norm, wsconst=wsconst).to_host()):
            assert np.array_equal(r.status, want["status"]) and not r.status.any()
            assert np.array_equal(r.n_tokens, want["n_tokens"]), (name, no_norm, wsconst)
            assert np.array_equal(r.token_ends, want["token_ends"]), (name, no_norm, wsconst)


@pytest.fixture(scope="module")
def eval_models():
    out = {}
    for name in ("all", "tag"):
        mb = _model_bytes(name)
        tags = name == "tag"
        out[name] = (vb.Predictor(vb.Model.read(mb), predict_tags=tags), OraclePredictor(mb, predict_tags=tags))
    return out


def _eval_check(p, o, data, **kw):
    want, rows = eo.evaluate_lines(o, data, **kw)
    got, lc = p.evaluate_lines(data, per_line=True, **kw)
    assert got == want, kw
    assert lc.tolist() == rows, kw
    return rows


@pytest.mark.parametrize("no_norm", [False, True])
def test_evaluate_lines(eval_models, no_norm):
    gold, _ = we.line_buffer(we.gold_cases())
    ev = we.eval_cases()
    lines = "\n".join(g for _, g, _ in ev) + "\n" + "\n".join(a for _, _, a in ev if a) + "\n"
    for name, (p, o) in eval_models.items():
        for predict_tags in ([False, True] if name == "tag" else [False]):
            _eval_check(p, o, gold, no_norm=no_norm, predict_tags=predict_tags)
            rows = _eval_check(p, o, lines.encode(), no_norm=no_norm, predict_tags=predict_tags)
            if name == "tag" and predict_tags:
                assert any(r[6] != r[4] for r in rows) and any(r[6] == r[4] for r in rows)


def test_evaluate_errors(eval_models):
    p, o = eval_models["all"]
    runs = [(c.key, we.line_buffer([c], lead=b"ab c\n")[0]) for c in we.gold_error_cases()]
    runs += [(name, b"\n".join(lines) + b"\n") for name, lines, _ in we.gold_error_multi()]
    for key, data in runs:
        with pytest.raises(eo.GoldError) as want:
            eo.evaluate_lines(o, data)
        with pytest.raises(vb.VaporettoError) as got:
            p.evaluate_lines(data)
        assert got.value.code == want.value.code and str(got.value) == want.value.msg, key
