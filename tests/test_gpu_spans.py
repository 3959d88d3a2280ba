"""vpt_token_spans on the device: vaporetto_tantivy's token_stream for a batch of documents (pre-filter, predict,
SplitLinebreaksFilter, wsconst post-filters, boundary_pos), bit-exact against the CPU oracle
(tests/vpt_testlib/spans_oracle.py) and the reference's known answers; tags, properties, chunking, errors, threads."""
import ctypes as C
import itertools
import os
import random
import threading

import numpy as np
import pytest

import vaporetto_b200 as vb
from golden import tantivy_kat as kat
from vpt_testlib import spans_oracle as so
from vpt_testlib import synth
from vpt_testlib.bincode_model import encode_model
from test_gpu_parity import _random_model, make, read
from test_spans_cpu import LINEBREAKS, batch, random_doc

pytestmark = pytest.mark.gpu

ALL_WSCONST = ["".join(c) for k in range(8) for c in itertools.combinations("DRHTKOG", k)]


def check_vs_oracle(p, o, text, off, no_norm=False, wsconst="", tags=False):
    r = p.token_spans(text, off, no_norm=no_norm, wsconst=wsconst, tags=tags)
    w = o.token_spans(text, off, no_norm=no_norm, wsconst=wsconst, tags=tags)
    ctx = (no_norm, wsconst, tags)
    assert np.array_equal(r.status, w["status"]), ctx
    assert np.array_equal(r.n_tokens, w["n_tokens"]), ctx
    assert np.array_equal(r.token_ends, w["token_ends"]), ctx
    if tags:
        assert np.array_equal(r.token_ids, w["token_ids"]), ctx
        assert np.array_equal(r.token_cands, w["token_cands"]), ctx
    return r


def check_properties(r, text, off):
    """The tokens tile every document, every end is on a character boundary, the total is the sum of the counts."""
    t = np.frombuffer(text, np.uint8) if isinstance(text, bytes) else text
    assert int(r.token_base[-1]) == r.token_ends.size == int(r.n_tokens.sum())
    for d in range(off.size - 1):
        lo, hi = int(off[d]), int(off[d + 1])
        sp = r.spans(d)
        if r.status[d] != 0:
            assert sp.shape[0] == 0
            continue
        assert sp.shape[0] >= 1 and sp[0, 0] == 0 and sp[-1, 1] == hi - lo
        assert np.all(sp[1:, 0] == sp[:-1, 1]) and np.all(sp[:, 1] > sp[:, 0])
        assert np.all((t[lo + sp[:-1, 1].astype(np.int64)] & 0xC0) != 0x80)


@pytest.mark.parametrize("text,wsconst,tokens", kat.TANTIVY_TOKEN_STREAMS)
def test_tantivy_known_answers(text, wsconst, tokens):
    p = make(read("tantivy_model.bin"))
    b, off = batch([text])
    r = p.token_spans(b, off, wsconst=wsconst)
    assert r.token_ends.tolist() == [t[2] for t in tokens]
    got = vb.Tokenizer(p, wsconst).token_stream(text)
    assert [(t.text, t.offset_from, t.offset_to, t.position, t.position_length) for t in got] == tokens
    # all six in one device call
    texts = [c[0] for c in kat.TANTIVY_TOKEN_STREAMS if c[1] == wsconst]
    many = vb.Tokenizer(p, wsconst).token_streams(texts * 3)
    assert [[(t.text, t.offset_from, t.offset_to, t.position, t.position_length) for t in d] for d in many][texts.index(text)] == tokens


@pytest.mark.parametrize("text,tokens", kat.SPLIT_LINEBREAKS)
def test_split_linebreaks_known_answers(text, tokens):
    m = dict(char_ngrams=[], type_ngrams=[], dict=[], bias=-1, char_window=1, type_window=1, tag_models=[])
    p = make(encode_model(m))
    b, off = batch([text])
    r = p.token_spans(b, off, no_norm=True)
    assert [b[f:t].decode() for f, t in r.spans(0).tolist()] == tokens


def newline_docs(rng):
    docs = ["\n", "\r", "\r\n", "\n\n\n", "\r\r\n\n", "。\n", "\r\n。", "a\r\nb", "東京\n", "\n東京", "\r\n東京\r\n",
            "。\n。\n。", "\n\r\n\r", "🤌🏿\n🇯🇵🇯\r\n👩‍👩‍👧", "ＡＢＣ\nabc123\r\n１２３", "(a-b)[c]/d.e,f!g?"]
    docs += [random_doc(rng, rng.randrange(1, 80)) for _ in range(120)]
    docs += ["".join(rng.choice(LINEBREAKS) for _ in range(rng.randrange(1, 30))) for _ in range(10)]
    return docs


@pytest.mark.parametrize("model", ["tantivy_model.bin", "model.bin"])
def test_every_wsconst_vs_oracle(model):
    """Newline-rich documents (runs, at the start and the end), emoji ZWJ and RI sequences, full-width-mapped ASCII,
    normalised or not, under every one of the 128 wsconst combinations."""
    rng = random.Random(11)
    mb = read(model)
    p, o = make(mb), so.SpansOracle(mb)
    b, off = batch(newline_docs(rng))
    for ws in ALL_WSCONST:
        for no_norm in (False, True):
            r = check_vs_oracle(p, o, b, off, no_norm=no_norm, wsconst=ws)
    check_properties(r, b, off)


@pytest.mark.parametrize("cw,tw,maxdict", [(3, 3, 3), (2, 4, 6), (5, 1, 12)])
def test_random_models_vs_oracle(cw, tw, maxdict):
    nprng = np.random.default_rng(cw * 100 + tw * 10 + maxdict)
    rng = random.Random(cw + tw + maxdict)
    for _ in range(3):
        m, alpha = _random_model(nprng, cw, tw, maxdict=maxdict)
        mb = encode_model(m)
        p, o = make(mb), so.SpansOracle(mb)
        docs = ["".join(rng.choice(list(alpha) + LINEBREAKS) for _ in range(rng.randrange(1, 200))) for _ in range(300)]
        b, off = batch(docs)
        for ws in ("", "O", "G", "OG", "DRHTKOG", rng.choice(ALL_WSCONST)):
            for no_norm in (False, True):
                check_vs_oracle(p, o, b, off, no_norm=no_norm, wsconst=ws)


def edge_docs():
    """Empty, NUL and invalid-UTF-8 documents between good ones; 1 character, 128 +- 1 bytes, 64 KiB, and about 20 MiB
    in the middle of the batch."""
    rng = random.Random(5)
    big = "".join(random_doc(rng, 40) + "\n" for _ in range(210_000)).encode()[: 20 << 20]
    big = big.decode("utf-8", "ignore").encode()
    docs = ["東", b"", "a\x00b", b"\xe3\x81", "a", b"\xff\n", "\n", "x" * 127, "x" * 128, "x" * 129,
            "あ" * 42 + "a", "\r\n" * 64, "あ" * 43, random_doc(rng, 64 * 1024 // 3)]
    docs += [random_doc(rng, rng.randrange(1, 100)) for _ in range(200)]
    docs += [big, b"", "局"] + [random_doc(rng, rng.randrange(1, 100)) for _ in range(200)] + [b"\x00", "end\r"]
    return docs


@pytest.mark.parametrize("chunk", ["4096", None])
def test_edge_documents_vs_oracle(chunk, monkeypatch):
    if chunk:
        monkeypatch.setenv("VPT_CHUNK_BYTES", chunk)
    mb = read("tantivy_model.bin")
    p, o = make(mb), so.SpansOracle(mb)
    b, off = batch(edge_docs())
    for ws, no_norm in (("", False), ("OG", False), ("D", True)):
        r = check_vs_oracle(p, o, b, off, no_norm=no_norm, wsconst=ws)
    check_properties(r, b, off)
    assert r.status.tolist()[:6] == [0, 1, 2, 3, 0, 3]


def test_config2_batch_vs_oracle():
    """200 000 documents on a config-2-shaped model (four chunks by document count)."""
    mb = synth.gen_model_bccwj_shaped(n_patterns=20000, sample_sentences=50000)
    text, offs, _ = synth.gen_text(200_000, 40)
    p, o = make(mb), so.SpansOracle(mb)
    r = check_vs_oracle(p, o, text, offs)
    assert r.n_tokens.min() >= 1


def test_no_norm_matches_compact_boundaries():
    """With no_norm and no wsconst, on documents without line breaks, the token ends are predict's boundaries."""
    mb = synth.gen_model_bccwj_shaped(n_patterns=5000, sample_sentences=20000)
    text, offs, _ = synth.gen_text(5000, 40, ragged=True)
    p = make(mb)
    r = p.token_spans(text, offs, no_norm=True)
    c = p.predict_batch_compact(text, offs)
    t = np.asarray(text, np.uint8)
    for d in range(0, offs.size - 1, 7):
        s = bytes(t[int(offs[d]):int(offs[d + 1])]).decode()
        starts = np.cumsum([0] + [len(ch.encode()) for ch in s])
        want = [int(starts[i + 1]) for i, x in enumerate(c.boundaries(d)) if x] + [int(starts[-1])]
        assert r.spans(d)[:, 1].tolist() == want


@pytest.mark.parametrize("which", ["model.bin", "synthetic"])
def test_tags_vs_oracle(which):
    rng = random.Random(3)
    if which == "model.bin":
        mb = read("model.bin")
        docs = ["まぁ社長は火星猫だ", "まぁ良いだろう\nまぁ社長は\r\n火星猫だ", "火星猫\n", "\n社長"] + newline_docs(rng)[:60]
    else:
        m, alpha = _random_model(np.random.default_rng(9), 3, 3, maxdict=4, tags=3)
        mb = encode_model(m)
        docs = ["".join(rng.choice(list(alpha) + LINEBREAKS) for _ in range(rng.randrange(1, 120))) for _ in range(400)]
    p, o = make(mb, tags=True), so.SpansOracle(mb, predict_tags=True)
    b, off = batch(docs)
    for ws in ("", "O", "G", "DRHTKOG"):
        for no_norm in (False, True):
            r = check_vs_oracle(p, o, b, off, no_norm=no_norm, wsconst=ws, tags=True)
    assert (r.token_ids >= 0).any()


def test_tags_render_like_tokenize_lines_tags():
    """For documents without line breaks, spans + tags written as tokenized text equal vpt_tokenize_lines_tags on the
    same documents joined by '\\n'."""
    p = make(read("model.bin"), tags=True)
    rng = random.Random(4)
    alpha = list("まぁ社長は火星猫だ良いろう") + list("ab1 /\\")
    docs = ["まぁ社長は火星猫だ", "まぁ良いだろう"] + ["".join(rng.choice(alpha) for _ in range(rng.randrange(1, 30)))
                                                       for _ in range(300)]
    b, off = batch(docs)
    r = p.token_spans(b, off, tags=True)
    esc = lambda s: s.replace("\\", "\\\\").replace(" ", "\\ ").replace("/", "\\/")
    lines = []
    for d, doc in enumerate(docs):
        raw = doc.encode()
        words = []
        for k, (f, t) in enumerate(r.spans(d).tolist()):
            rec = int(r.token_base[d]) + k
            w = esc(raw[f:t].decode())
            tid = int(r.token_ids[rec])
            cands = r.token_cands[rec].tolist()
            last = max([i for i, c in enumerate(cands) if c != 255], default=-1) if tid >= 0 else -1
            for i in range(last + 1):
                w += "/" + (esc(p.tag_string(tid, i, cands[i])) if cands[i] != 255 else "")
            words.append(w)
        lines.append(" ".join(words))
    want, _ = p.tokenize_lines(("\n".join(docs) + "\n").encode(), predict_tags=True)
    assert ("\n".join(lines) + "\n").encode() == want.tobytes()


def test_errors():
    p = make(read("tantivy_model.bin"))
    L = vb.lib()
    b, off = batch(["東京特許許可局", "123456円🤌🏿"])
    n = np.zeros(2, np.uint32)
    st = np.zeros(2, np.uint8)
    ends = np.zeros(64, np.uint32)
    total = C.c_uint64()
    # too small: InvalidArgument with the total reported
    rc = L.vpt_token_spans(p._h, b, off.ctypes.data, 2, 0, 0, n.ctypes.data, st.ctypes.data, ends.ctypes.data, None, None,
                           5, C.byref(total))
    assert rc == 2 and total.value == 13 and "token_capacity" in L.vpt_last_error().decode()
    # bad wsconst bits, as the lines calls reject them
    rc = L.vpt_token_spans(p._h, b, off.ctypes.data, 2, 0, 1, n.ctypes.data, st.ctypes.data, ends.ctypes.data, None, None,
                           64, C.byref(total))
    assert rc == 2 and "wsconst_types" in L.vpt_last_error().decode()
    # tags on a predictor without tags
    with pytest.raises(vb.VaporettoError) as e:
        p.token_spans(b, off, tags=True)
    assert e.value.code == 2 and "predict_tags = false" in str(e.value)
    # no documents
    rc = L.vpt_token_spans(p._h, None, off.ctypes.data, 0, 0, 0, n.ctypes.data, st.ctypes.data, None, None, None, 0,
                           C.byref(total))
    assert rc == 0 and total.value == 0
    r = p.token_spans(b"", np.zeros(1, np.uint64))
    assert r.token_ends.size == 0 and r.n_tokens.size == 0
    # a rejected document in the adapter-shaped API names the reference's message and the document
    with pytest.raises(vb.VaporettoError) as e:
        vb.Tokenizer(p).token_streams(["東京", "a\x00b"])
    assert "must not contain NULL" in str(e.value) and "document 1" in str(e.value)
    assert vb.Tokenizer(p).token_stream("") == []


def test_two_threads_one_predictor():
    mb = read("tantivy_model.bin")
    p, o = make(mb), so.SpansOracle(mb)
    rng = random.Random(8)
    jobs = []
    for k in range(2):
        b, off = batch([random_doc(rng, rng.randrange(1, 400)) for _ in range(3000)])
        jobs.append((b, off, "OG" if k else "", o.token_spans(b, off, wsconst="OG" if k else "")))
    errors = []

    def run(job):
        b, off, ws, want = job
        try:
            for _ in range(20):
                r = p.token_spans(b, off, wsconst=ws)
                assert np.array_equal(r.token_ends, want["token_ends"])
                assert np.array_equal(r.n_tokens, want["n_tokens"])
        except BaseException as e:  # re-raised below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(j,)) for j in jobs]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
