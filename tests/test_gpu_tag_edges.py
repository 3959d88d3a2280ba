"""Device tag prediction on tokens whose ends sit on the edges of k_tags' chunk and ring arithmetic
(vpt_testlib/tag_edges.py): tokens up to 300 characters of every UTF-8 width at every start alignment, whole-sentence
tokens and one-token lines over 65 535 bytes, through every device tag path -- vpt_predict_batch_tags,
vpt_predict_batch_compact, vpt_tokenize_lines_tags and vpt_evaluate_lines -- against the CPU oracle, the host path and
the hand-derived tags of the edge model.  A tag model the device cannot serve is reported, never written untagged."""
import numpy as np
import pytest

import vaporetto_b200 as vb
from vpt_testlib import eval_oracle as eo
from vpt_testlib import tag_edges as te
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.oracle import OraclePredictor
from test_gpu_tags import _batch, _check_against_host_and_oracle, _check_compact

pytestmark = pytest.mark.gpu

VPT_UNSUPPORTED = 17


@pytest.fixture(scope="module")
def edge():
    cases = te.edge_cases()
    mb = encode_model(te.model(cases))
    p, o = vb.Predictor(vb.Model.read(mb), predict_tags=True), OraclePredictor(mb, predict_tags=True)
    pairs = [(c.sentence, c.align) for c in cases]
    pairs += [(te.LONG_KNOWN, 0), (te.LONG_KNOWN, 3), (te.LONG_UNKNOWN, 1), (te.LONG_UNKNOWN, 2)]
    return cases, p, o, pairs


def test_batch_tags(edge):
    """Per-character tags of every edge sentence: device == host path (fill_tags) == oracle == by hand, nothing unserved."""
    cases, p, o, pairs = edge
    sents, idx = te.aligned_batch(pairs)
    res = _check_against_host_and_oracle(p, o, sents)
    text, offs = _batch(sents)
    assert [int(offs[i]) % 4 for i in idx] == [a for _, a in pairs]
    _, tok, cand, unserved = p.predict_batch_tags(text, offs)
    assert unserved == 0
    known = set(te.known_tokens(cases))
    for c, i in zip(cases, idx):
        c0, c1 = int(res.char_offsets[i]), int(res.char_offsets[i + 1])
        assert cand[c0:c1].tolist() == te.expected_sentence_cands(c.tokens, known), (c.kind, c.w, c.align, c.known)
    for (line, _), i in zip(pairs[len(cases):], idx[len(cases):]):
        c1 = int(res.char_offsets[i + 1])
        want = te.expected_cands(line, None) if line == te.LONG_KNOWN else [-1, -1]
        assert cand[c1 - 1].tolist() == want and (tok[c1 - 1] >= 0) == (want[0] >= 0)


def test_compact(edge):
    """Token records of vpt_predict_batch_compact (the per-token locate + lookup kernels) == the per-character arrays."""
    _, p, _, pairs = edge
    sents, _ = te.aligned_batch(pairs)
    text, offs = _batch(sents)
    r = _check_compact(p, text, offs, tags=True)
    assert r.n_unserved == 0


def _lines(pairs):
    return te.aligned_lines(pairs, crlf_every=3)


@pytest.mark.parametrize("no_norm", [False, True])
@pytest.mark.parametrize("chunk", [None, "4096", "65536"])
def test_tokenize_lines_tags(edge, no_norm, chunk, monkeypatch):
    """--predict-tags output byte for byte against the oracle's CLI loop.  Lines start at all four alignments, every
    third ends in CRLF; 65 536-byte chunks are shorter than the 70 000-byte lines, so a nominal cut falls inside each."""
    cases, p, o, pairs = edge
    if chunk is not None:
        monkeypatch.setenv("VPT_CHUNK_BYTES", chunk)
    data = _lines(pairs)
    want, nl = o.tokenize_lines(data, no_norm=no_norm, predict_tags=True)
    got, gl = p.tokenize_lines(data, no_norm=no_norm, predict_tags=True)
    assert gl == nl
    assert got.tobytes() == want
    # the long lines by hand: the 70 000-byte known token is tagged, the longer line that starts with a known
    # 65 535-byte prefix is not
    out = want.split(b"\n")
    b, e = te.expected_cands(te.LONG_KNOWN, None)
    assert te.LONG_KNOWN.encode() + b"/" + te.TAGS[0][b].encode() + b"/" + te.TAGS[1][e].encode() in out
    assert te.LONG_UNKNOWN.encode() in out


def _perturbed(gold: bytes) -> bytes:
    """The gold corpus with the tags of the long tokens changed on every other line."""
    lines = gold.split(b"\n")
    for i in range(0, len(lines), 2):
        if len(lines[i]) > 200:
            lines[i] = lines[i].replace(b"/A/", b"/B/").replace(b"/E", b"/C")
    return b"\n".join(lines)


@pytest.mark.parametrize("no_norm", [False, True])
def test_evaluate_lines_tags(edge, no_norm):
    """vpt_evaluate_lines with predict_tags against the oracle's restatement, per line: on the oracle's own tagged
    output and on a copy where long tokens' tags are changed.  On its own output every line with a tagged token is
    perfect; a line without any tagged token (a twin's) counts no correct word, in the oracle's restatement of the
    reference as on the device."""
    _, p, o, pairs = edge
    gold, _ = o.tokenize_lines(_lines(pairs), no_norm=no_norm, predict_tags=True)
    perturbed = _perturbed(gold)
    n_cor = []
    for data in (gold, perturbed):
        want, rows = eo.evaluate_lines(o, data, no_norm=no_norm, predict_tags=True)
        got, lc = p.evaluate_lines(data, no_norm=no_norm, predict_tags=True, per_line=True)
        assert got == want
        assert lc.tolist() == rows
        assert got["fp"] == got["fn"] == 0 and got["n_sys"] == got["n_ref"]
        n_cor.append([r[6] for r in rows])
        if data is gold:
            tagged = [i for i, line in enumerate(data.split(b"\n")) if b"/" in line]
            assert len(tagged) > 100
            assert all(rows[i][4] == rows[i][5] == rows[i][6] for i in tagged)
    changed = [i for i, (a, b) in enumerate(zip(gold.split(b"\n"), perturbed.split(b"\n"))) if a != b]
    assert len(changed) > 50
    assert all(n_cor[1][i] < n_cor[0][i] for i in changed)
    assert all(n_cor[1][i] == n_cor[0][i] for i in range(len(n_cor[0])) if i not in set(changed))


def test_unusable_token_model():
    """One token whose tag slot has 65 candidates (more scores than the device tables hold): the batch path counts it
    unserved and the host path serves it as the oracle does; the lines and evaluate paths refuse the model up front."""
    cases = te.edge_cases()[:4]
    big = te.pad_token(3, 4)
    extra = dict(token=big, tags=[[str(k) for k in range(65)]], char_ngrams=[], type_ngrams=[], bias=list(range(65)))
    mb = encode_model(te.model(cases, extra_tag_models=[extra]))
    p, o = vb.Predictor(vb.Model.read(mb), predict_tags=True), OraclePredictor(mb, predict_tags=True)
    sents = [big + te.target_token(3, 5), cases[0].sentence]
    text, offs = _batch(sents)
    res, tok, cand, unserved = p.predict_batch_tags(text, offs)
    assert unserved >= 1
    assert tok[len(big) - 1] == -1
    hs = vb.Sentence.from_raw(sents[0])
    p.predict(hs)
    hs.fill_tags()
    ott, oti = o.predict_tags(sents[0])
    assert hs._tag_cand.reshape(-1, p.n_tags).tolist() == oti.tolist()
    assert oti[len(big) - 1].tolist() == [64, -1]
    assert p.predict_batch_compact(text, offs, tags=True).n_unserved >= 1
    data = "\n".join(sents).encode() + b"\n"
    with pytest.raises(vb.VaporettoError) as e:
        p.tokenize_lines(data, predict_tags=True)
    assert e.value.code == VPT_UNSUPPORTED
    gold, _ = o.tokenize_lines(data, predict_tags=True)
    with pytest.raises(vb.VaporettoError) as e:
        p.evaluate_lines(gold, predict_tags=True)
    assert e.value.code == VPT_UNSUPPORTED
    # without tags both paths still run
    assert p.tokenize_lines(data)[0].tobytes() == o.tokenize_lines(data)[0]
    assert p.evaluate_lines(gold) == eo.evaluate_lines(o, gold)[0]
