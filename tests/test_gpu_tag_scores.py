"""Tag candidate scores from the device (vpt_predict_batch_compact_tag_scores, vpt_token_spans_tag_scores) byte for byte
against the CPU oracle's raw scores (tests/native/tag_scores_oracle.cpp), their invariants, their edges, and the
Sentence path (Predictor.store_tag_scores + Token.tag_candidates)."""
import ctypes as C
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import vaporetto_b200 as vb
from golden import reference_kat as kat
from test_gpu_parity import _random_model, read
from test_tag_scores_cpu import KAT_SCORES, OVERRUN_MODEL
from vpt_testlib import synth
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.tag_scores_oracle import TagScoresOracle, first_max, tag_candidates

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _batch(sents):
    enc = [s.encode() if isinstance(s, str) else s for s in sents]
    offs = np.zeros(len(enc) + 1, np.uint64)
    np.cumsum([len(e) for e in enc], out=offs[1:])
    return np.frombuffer(b"".join(enc) + b"\0", np.uint8)[: int(offs[-1])], offs


def _own_tags(p, tid):
    L = vb.lib()
    return [[L.vpt_tag_string(p._h, tid, k, c).decode() for c in range(L.vpt_tag_n_candidates(p._h, tid, k))]
            for k in range(L.vpt_tag_n_slots(p._h, tid))]


def _invariants(p, r):
    """Record count with scores, total, layout and the arg-max of every slot against token_cands."""
    ids = r.token_ids
    lens = p._score_lens()
    assert r.score_offsets.size == ids.size + 1
    assert int(r.score_offsets[-1]) == r.tag_scores.size == int(sum(int(lens[t]) for t in ids if t >= 0))
    assert int(np.count_nonzero(np.diff(r.score_offsets.astype(np.int64)))) == int(np.count_nonzero(ids >= 0))
    for rec in np.flatnonzero(ids >= 0)[:4000]:
        tid = int(ids[rec])
        v = r.tag_scores[int(r.score_offsets[rec]):int(r.score_offsets[rec + 1])]
        off = 0
        own = _own_tags(p, tid)
        for k, cands in enumerate(own[: p.n_tags]):
            if len(cands) >= 2:
                assert int(r.token_cands[rec, k]) == first_max(v[off:off + len(cands)].tolist())
                off += len(cands)
        assert r.tag_candidates(int(rec)) == tag_candidates(own, v)


def _check_compact(p, o, text, offs):
    r = p.predict_batch_compact(text, offs, tags=True, tag_scores=True)
    plain = p.predict_batch_compact(text, offs, tags=True)
    for f in ("boundary_bits", "n_chars", "status", "n_tokens", "token_ids", "token_cands"):
        assert np.array_equal(getattr(r, f), getattr(plain, f)), f
    ids, sc = o.compact(text, offs)
    assert (r.token_ids >= 0).tolist() == (ids >= 0).tolist()
    assert r.tag_scores.tobytes() == sc.tobytes()
    _invariants(p, r)
    return r


def _check_spans(p, o, text, offs, no_norm=False, wsconst=""):
    r = p.token_spans(text, offs, no_norm=no_norm, wsconst=wsconst, tags=True, tag_scores=True)
    plain = p.token_spans(text, offs, no_norm=no_norm, wsconst=wsconst, tags=True)
    for f in ("n_tokens", "status", "token_ends", "token_ids", "token_cands"):
        assert np.array_equal(getattr(r, f), getattr(plain, f)), f
    ids, sc = o.spans(text, offs, no_norm=no_norm, wsconst=wsconst)
    assert (r.token_ids >= 0).tolist() == (ids >= 0).tolist()
    assert r.tag_scores.tobytes() == sc.tobytes()
    _invariants(p, r)
    return r


def _make(mb):
    return vb.Predictor(vb.Model.read(mb), predict_tags=True), TagScoresOracle(mb)


def test_reference_models():
    p, o = _make(encode_model(kat.PREDICTOR_TEST_MODEL))
    text, offs = _batch(["この人は地球人だ", "地球人", "", "この人", "人"])
    r = _check_compact(p, o, text, offs)
    assert r.tag_scores[: len(KAT_SCORES)].tolist() == KAT_SCORES
    assert r.tag_candidates(1) == [[("名詞", 76), ("接尾辞", 4)], [("ジン", 4), ("ヒト", 82)]]
    assert r.tag_candidates(3) == [[("名詞", 0)], [("マンホーム", 2), ("チキュー", 92)]]
    assert r.tag_candidates(0) == []
    _check_spans(p, o, text, offs, no_norm=True)
    p, o = _make(read("model.bin"))
    sents = ["まぁ社長は火星猫だ", "まぁ良いだろう", "火星", "社長は社長だ" * 30, "a\x00b", b"\xff\xfe", ""]
    text, offs = _batch(sents)
    _check_compact(p, o, text, offs)
    for no_norm in (False, True):
        for ws in ("", "D", "KH", "DRHTKOG"):
            _check_spans(p, o, text, offs, no_norm=no_norm, wsconst=ws)


@pytest.mark.parametrize("cw,tw,maxdict,tags", [(3, 3, 5, 3), (1, 5, 3, 2), (5, 4, 4, 3), (3, 3, 9, 6)])
def test_random_tag_models(cw, tw, maxdict, tags):
    rng = np.random.default_rng(99 + 1000 * cw + 100 * tw + maxdict + tags)
    for _ in range(2):
        model, alpha = _random_model(rng, cw, tw, maxdict=maxdict, tags=tags)
        p, o = _make(encode_model(model))
        sents = ["".join(rng.choice(list(alpha), size=rng.integers(1, 60))) for _ in range(300)]
        sents += ["".join(rng.choice(list(alpha), size=n)) for n in (1, 2, 31, 32, 33, 64, 65, 300)] + ["", "x\ny\r\nz"]
        text, offs = _batch(sents)
        _check_compact(p, o, text, offs)
        _check_spans(p, o, text, offs, wsconst="O")


def _synthetic():
    mb = synth.gen_model_bccwj_shaped(n_patterns=30_000, sample_sentences=50_000, tag_models=1_500)
    text, offs, _ = synth.gen_text(6_000, 40, seed=synth.TEXT_SEED + 21)
    sents = [bytes(text[int(offs[i]):int(offs[i + 1])]) for i in range(len(offs) - 1)]
    sents[5], sents[77], sents[78], sents[4999] = b"", b"a\x00b", b"\xc3", "あ".encode()
    return mb, sents


def _compact_chunked():
    mb, sents = _synthetic()
    p, o = _make(mb)
    text, offs = _batch(sents)
    r = _check_compact(p, o, text, offs)
    assert int((r.token_ids >= 0).sum()) > 1000


@pytest.mark.parametrize("chunk", [None, "700", "4096"])
def test_synthetic_model_chunk_borders(chunk):
    """A config-3-shaped tag model: compact scores at several chunk sizes (VPT_CHUNK_SENTENCES is read once per process:
    the small sizes run in a child process), with empty, NUL and invalid UTF-8 sentences."""
    if chunk is None:
        _compact_chunked()
        return
    code = ("import os,sys; sys.path.insert(0, %r); os.environ['VPT_CHUNK_SENTENCES']=%r\n"
            "import test_gpu_tag_scores as t; t._compact_chunked()\n") % (HERE, chunk)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-3000:]


@pytest.mark.parametrize("chunk_bytes", ["300", "5000"])
def test_spans_chunk_borders(chunk_bytes, monkeypatch):
    monkeypatch.setenv("VPT_CHUNK_BYTES", chunk_bytes)
    mb, sents = _synthetic()
    p, o = _make(mb)
    text, offs = _batch(sents[:2000])
    _check_spans(p, o, text, offs)
    _check_spans(p, o, text, offs, no_norm=True, wsconst="DG")


def test_model_without_tag_slots():
    model = dict(char_ngrams=[("ab", [1, -2, 3])], type_ngrams=[], dict=[], bias=0, char_window=2, type_window=0,
                 tag_models=[])
    p = vb.Predictor(vb.Model.read(encode_model(model)), predict_tags=True)
    assert p.n_tags == 0
    text, offs = _batch(["abab", "ba", ""])
    r = p.token_spans(text, offs, tags=True, tag_scores=True)
    assert r.token_ids.size > 0 and (r.token_ids == -1).all() and r.tag_scores.size == 0
    assert r.tag_candidates(0) == []


def test_token_beyond_the_device_limits():
    """A tag model of 65 scores is beyond the device path: unserved, id -1, no scores; vpt_fill_tags serves it with its
    scores on the Sentence path."""
    big = dict(token="人", tags=[["c%d" % i for i in range(65)]], char_ngrams=[("人", [(0, list(range(65)))])], type_ngrams=[],
               bias=[(-1) ** i * i for i in range(65)])
    small = dict(token="火", tags=[["x", "y"]], char_ngrams=[], type_ngrams=[], bias=[5, 9])
    model = dict(char_ngrams=[("人火", [1, -50, 2, 3])], type_ngrams=[], dict=[("人", [99, 99], "")], bias=-10, char_window=2,
                 type_window=0, tag_models=[big, small])
    mb = encode_model(model)
    p, o = _make(mb)
    text, offs = _batch(["人火人", "火"])
    r = p.predict_batch_compact(text, offs, tags=True, tag_scores=True)
    assert r.n_unserved >= 1
    toks = []
    for s in ("人火人", "火"):
        sent = vb.Sentence.from_raw(s)
        p.predict(sent)
        toks += [t.surface() for t in sent.iter_tokens()]
    assert [int(i) >= 0 for i in r.token_ids] == [t == "火" for t in toks]
    assert r.tag_scores.tolist() == [5, 9, 0, 0, 0, 0, 0, 0] * toks.count("火")
    p.store_tag_scores(True)
    sent = vb.Sentence.from_raw("人火人")
    p.predict(sent)
    sent.fill_tags()
    cands = {t.surface(): t.tag_candidates() for t in sent.iter_tokens()}
    if "人" in cands:
        assert len(cands["人"]) == 1 and len(cands["人"][0]) == 65
        v = [s for _, s in cands["人"][0]]
        assert v == [((-1) ** i * i + i) for i in range(65)]


def test_candidate_overrun_model():
    """"a" has more candidates than scores: id -1 and no scores on both paths (the oracle and vpt_fill_tags reject it)."""
    p = vb.Predictor(vb.Model.read(encode_model(OVERRUN_MODEL)), predict_tags=True)
    sents = ["a", "b", "ab", "ba", "aab", "bb"]
    text, offs = _batch(sents)
    toks = []
    for s in sents:
        sent = vb.Sentence.from_raw(s)
        p.predict(sent)
        toks += [t.surface() for t in sent.iter_tokens()]
    for r in (p.predict_batch_compact(text, offs, tags=True, tag_scores=True),
              p.token_spans(text, offs, no_norm=True, tags=True, tag_scores=True)):
        assert [int(i) >= 0 for i in r.token_ids] == [t == "b" for t in toks]
        assert r.tag_scores.tolist() == [7, 8, 0, 0, 0, 0, 0, 0] * toks.count("b")
        _invariants(p, r)
    sent = vb.Sentence.from_raw("a")
    p.predict(sent)
    with pytest.raises(vb.VaporettoError):
        sent.fill_tags()


def test_capacity_one_short_and_errors():
    mb = read("model.bin")
    p = vb.Predictor(vb.Model.read(mb), predict_tags=True)
    text, offs = _batch(["まぁ社長は火星猫だ", "火星", "社長は社長だ"])
    full = p.predict_batch_compact(text, offs, tags=True, tag_scores=True)
    need = full.tag_scores.size
    assert need > 0
    L = vb.lib()
    n = len(offs) - 1
    cap = text.size
    bits = np.zeros(cap, np.uint32)
    nch, st, ntk = np.zeros(n, np.uint32), np.zeros(n, np.uint8), np.zeros(n, np.uint32)
    ids, cands = np.zeros(cap, np.int32), np.zeros(cap * max(p.n_tags, 1), np.uint8)
    sc = np.zeros(need, np.int32)
    nb, nt, nu, ns = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_uint64()
    args = [p._h, text.ctypes.data, offs.ctypes.data, n, bits.ctypes.data, bits.size, nch.ctypes.data, st.ctypes.data,
            ntk.ctypes.data, ids.ctypes.data, cands.ctypes.data, cap, C.byref(nb), C.byref(nt), C.byref(nu)]
    assert L.vpt_predict_batch_compact_tag_scores(*args, sc.ctypes.data, need - 1, C.byref(ns)) == 2
    assert ns.value == need
    assert L.vpt_predict_batch_compact_tag_scores(*args, sc.ctypes.data, need, C.byref(ns)) == 0
    assert ns.value == need and np.array_equal(sc, full.tag_scores)
    ends = np.zeros(cap, np.uint32)
    sargs = [p._h, text.ctypes.data, offs.ctypes.data, n, 0, 0, ntk.ctypes.data, st.ctypes.data, ends.ctypes.data,
             ids.ctypes.data, cands.ctypes.data, cap, C.byref(nt)]
    spans = p.token_spans(text, offs, tags=True, tag_scores=True)
    need_s = spans.tag_scores.size
    assert L.vpt_token_spans_tag_scores(*sargs, sc.ctypes.data, need_s - 1, C.byref(ns)) == 2 and ns.value == need_s
    # scores need tags; a predictor made without tag prediction gets the existing message
    assert L.vpt_predict_batch_compact_tag_scores(*args[:9], None, None, cap, C.byref(nb), C.byref(nt), C.byref(nu),
                                                  sc.ctypes.data, need, C.byref(ns)) == 2
    p0 = vb.Predictor(vb.Model.read(mb), predict_tags=False)
    with pytest.raises(vb.VaporettoError, match="predict_tags = false"):
        p0.predict_batch_compact(text, offs, tags=True, tag_scores=True)
    with pytest.raises(vb.VaporettoError, match="predict_tags = false"):
        p0.token_spans(text, offs, tags=True, tag_scores=True)
    with pytest.raises(vb.VaporettoError):
        p.predict_batch_compact(text, offs, tag_scores=True)


def test_two_threads_on_one_predictor():
    mb, sents = _synthetic()
    p = vb.Predictor(vb.Model.read(mb), predict_tags=True)
    text, offs = _batch(sents)
    want_c = p.predict_batch_compact(text, offs, tags=True, tag_scores=True).tag_scores
    want_s = p.token_spans(text, offs, tags=True, tag_scores=True).tag_scores
    errs = []

    def work(k):
        try:
            for _ in range(3):
                if k == 0:
                    assert np.array_equal(p.predict_batch_compact(text, offs, tags=True, tag_scores=True).tag_scores, want_c)
                else:
                    assert np.array_equal(p.token_spans(text, offs, tags=True, tag_scores=True).tag_scores, want_s)
        except BaseException as e:  # (re-raised below)
            errs.append(e)
    th = [threading.Thread(target=work, args=(k,)) for k in (0, 1)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs


def test_sentence_path():
    """store_tag_scores + Token.tag_candidates against the oracle and against the compact result's tag_candidates."""
    for mb in (encode_model(kat.PREDICTOR_TEST_MODEL), read("model.bin")):
        p, o = _make(mb)
        sents = ["この人は地球人だ", "まぁ社長は火星猫だ", "火星人", "社長は社長だ"]
        text, offs = _batch(sents)
        r = p.predict_batch_compact(text, offs, tags=True, tag_scores=True)
        sent = vb.Sentence.from_raw(sents[0])
        p.predict(sent)
        sent.fill_tags()
        with pytest.raises(RuntimeError, match="store_tag_scores"):
            next(iter(sent.iter_tokens())).tag_candidates()
        p.store_tag_scores(True)
        rec = 0
        for s in sents:
            sent = vb.Sentence.from_raw(s)
            p.predict(sent)
            sent.fill_tags()
            ids, sc = o.compact(*_batch([s]))
            off = 0
            for k, tok in enumerate(sent.iter_tokens()):
                got = tok.tag_candidates()
                assert got == r.tag_candidates(rec), (s, k)
                if ids[k] >= 0:
                    n = int(p._score_lens()[int(r.token_ids[rec])])
                    assert got == tag_candidates(_own_tags(p, int(r.token_ids[rec])), sc[off:off + n])
                    off += n
                rec += 1
        p.store_tag_scores(False)
