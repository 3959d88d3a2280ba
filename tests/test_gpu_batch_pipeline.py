"""The chunk pipeline of the sentence and document batch calls (vpt_predict_batch, vpt_predict_batch_compact_tag_scores,
vpt_token_spans_tag_scores): a batch cut into many more chunks than the pipeline holds gives every output byte for byte as
one chunk does; a capacity that runs out in the middle or at the end of the batch fails with the full batch's totals;
VPT_TRACE=1 prints one line per chunk.  VPT_CHUNK_SENTENCES is read once per process: the many-chunk runs are children."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import vaporetto_b200 as vb
from vpt_testlib import synth

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
MANY_CHUNKS = {"VPT_CHUNK_SENTENCES": "1024", "VPT_CHUNK_BYTES": "4096"}  # 23 sentence chunks, hundreds of span chunks
ONE_CHUNK_BYTES = str(1 << 30)  # the span chunks' byte budget of the one-chunk run
INVALID = 2  # VPT_INVALID_ARGUMENT


def _workload(d):
    """Seeded tag model and ~20 000 sentences of mixed length with empty, NUL and invalid UTF-8 ones, written to `d`."""
    mb = synth.gen_model_bccwj_shaped(n_patterns=30_000, sample_sentences=50_000, tag_models=1_500)
    text, offs, _ = synth.gen_text(20_000, 40, seed=synth.TEXT_SEED + 33, ragged=True)
    sents = [bytes(text[int(offs[i]):int(offs[i + 1])]) for i in range(len(offs) - 1)]
    for i in list(range(0, len(sents) - 3, 997)) + [127, 128, 383, 384]:
        sents[i], sents[i + 1], sents[i + 2] = b"", "a\0b".encode(), b"\xe3\x81"
    offs = np.zeros(len(sents) + 1, np.uint64)
    np.cumsum([len(s) for s in sents], out=offs[1:])
    with open(os.path.join(d, "model.bin"), "wb") as f:
        f.write(mb)
    np.savez(os.path.join(d, "batch.npz"), text=np.frombuffer(b"".join(sents), np.uint8), offs=offs)


def _load(d):
    p = vb.Predictor(vb.Model.read(open(os.path.join(d, "model.bin"), "rb").read()), predict_tags=True)
    z = np.load(os.path.join(d, "batch.npz"))
    return p, z["text"], z["offs"]


def _outputs(p, text, offs):
    """Every output array of the three calls: batch with and without scores, compact without tags, with tags, with tags
    and scores, spans with tags and scores."""
    out = {}
    for name, r in (("batch", p.predict_batch(text, offs, want_scores=True, want_states=True)),
                    ("batch_noscores", p.predict_batch(text, offs, want_scores=False))):
        for f in ("scores", "boundaries", "bound_offsets", "status", "char_states", "type_states", "char_offsets"):
            if getattr(r, f) is not None:
                out[name + "." + f] = np.asarray(getattr(r, f))
        out[name + ".totals"] = np.array([r.n_boundaries, r.n_chars], np.uint64)
    for name, kw in (("compact", {}), ("compact_tags", {"tags": True}), ("compact_scores", {"tags": True, "tag_scores": True})):
        r = p.predict_batch_compact(text, offs, **kw)
        for f in ("boundary_bits", "n_chars", "status", "n_tokens", "token_ids", "token_cands", "tag_scores"):
            if getattr(r, f, None) is not None:
                out[name + "." + f] = np.asarray(getattr(r, f))
        out[name + ".totals"] = np.array([r.n_boundaries, r.n_unserved], np.uint64)
    r = p.token_spans(text, offs, tags=True, tag_scores=True)
    for f in ("n_tokens", "status", "token_ends", "token_ids", "token_cands", "tag_scores"):
        out["spans." + f] = np.asarray(getattr(r, f))
    return out


def _fail(rc, what):
    assert rc == INVALID, (rc, what)
    msg = vb.lib().vpt_last_error().decode()
    assert msg == "InvalidArgumentError: %s: too small for the batch" % what, msg


def _overflow(p, text, offs, full):
    """Each capacity at about half of the need and one short of it, then exact, through the C ABI."""
    L, n = vb.lib(), offs.size - 1
    u64 = lambda: C.c_uint64()
    nb, nc = (int(x) for x in full["batch.totals"])

    def batch(cap, scap):
        o = dict(scores=np.zeros(max(cap, 1), np.int32), boundaries=np.zeros(max(cap, 1), np.uint8),
                 bound_offsets=np.zeros(n + 1, np.uint64), status=np.zeros(n, np.int32),
                 char_states=np.zeros(max(scap, 1), np.uint32), type_states=np.zeros(max(scap, 1), np.uint32),
                 char_offsets=np.zeros(n + 1, np.uint64))
        a, b = u64(), u64()
        rc = L.vpt_predict_batch(p._h, text.ctypes.data, offs.ctypes.data, n, *(o[k].ctypes.data for k in (
            "scores", "boundaries")), cap, o["bound_offsets"].ctypes.data, o["status"].ctypes.data,
            o["char_states"].ctypes.data, o["type_states"].ctypes.data, scap, o["char_offsets"].ctypes.data,
            C.byref(a), C.byref(b))
        return rc, (a.value, b.value), o

    for cap, scap in ((nb // 2, nc), (nb - 1, nc), (nb, nc // 2), (nb, nc - 1)):
        rc, totals, _ = batch(cap, scap)
        _fail(rc, "out_capacity/states_capacity")
        assert totals == (nb, nc), (cap, scap, totals)
    rc, totals, o = batch(nb, nc)
    assert rc == 0 and totals == (nb, nc)
    for k, v in o.items():
        assert np.array_equal(v[: full["batch." + k].size], full["batch." + k]), k

    nt = p.n_tags
    words = full["compact_scores.boundary_bits"].size
    ntok = full["compact_scores.token_ids"].size
    nsc = full["compact_scores.tag_scores"].size

    def compact(wcap, tcap, scap):
        o = dict(boundary_bits=np.zeros(max(wcap, 1), np.uint32), n_chars=np.zeros(n, np.uint32),
                 status=np.zeros(n, np.uint8), n_tokens=np.zeros(n, np.uint32), token_ids=np.zeros(max(tcap, 1), np.int32),
                 token_cands=np.zeros(max(tcap, 1) * max(nt, 1), np.uint8), tag_scores=np.zeros(max(scap, 1), np.int32))
        a, b, c, d = u64(), u64(), u64(), u64()
        rc = L.vpt_predict_batch_compact_tag_scores(
            p._h, text.ctypes.data, offs.ctypes.data, n, o["boundary_bits"].ctypes.data, wcap, o["n_chars"].ctypes.data,
            o["status"].ctypes.data, o["n_tokens"].ctypes.data, o["token_ids"].ctypes.data, o["token_cands"].ctypes.data,
            tcap, C.byref(a), C.byref(b), C.byref(c), o["tag_scores"].ctypes.data, scap, C.byref(d))
        return rc, (a.value, b.value, d.value), o

    for wcap in (words // 2, words - 1):
        rc, totals, _ = compact(wcap, ntok, nsc)
        _fail(rc, "bits_capacity_words/token_capacity")
        assert totals[0] == nb, (wcap, totals)  # (a chunk past the bits is not issued: its tokens are not counted)
    for tcap, scap, what in ((ntok // 2, nsc, "bits_capacity_words/token_capacity"),
                             (ntok - 1, nsc, "bits_capacity_words/token_capacity"),
                             (ntok, nsc // 2, "score_capacity"), (ntok, nsc - 1, "score_capacity")):
        rc, totals, _ = compact(words, tcap, scap)
        _fail(rc, what)
        assert totals == (nb, ntok, nsc), (tcap, scap, totals)
    rc, totals, o = compact(words, ntok, nsc)
    assert rc == 0 and totals == (nb, ntok, nsc)
    o["token_cands"] = o["token_cands"].reshape(-1, max(nt, 1))
    for k, v in o.items():
        assert np.array_equal(v[: len(full["compact_scores." + k])], full["compact_scores." + k]), k

    stok = full["spans.token_ends"].size
    ssc = full["spans.tag_scores"].size

    def spans(tcap, scap):
        o = dict(n_tokens=np.zeros(n, np.uint32), status=np.zeros(n, np.uint8), token_ends=np.zeros(max(tcap, 1), np.uint32),
                 token_ids=np.zeros(max(tcap, 1), np.int32), token_cands=np.zeros(max(tcap, 1) * max(nt, 1), np.uint8),
                 tag_scores=np.zeros(max(scap, 1), np.int32))
        a, b = u64(), u64()
        rc = L.vpt_token_spans_tag_scores(
            p._h, text.ctypes.data, offs.ctypes.data, n, 0, 0, o["n_tokens"].ctypes.data, o["status"].ctypes.data,
            o["token_ends"].ctypes.data, o["token_ids"].ctypes.data, o["token_cands"].ctypes.data, tcap, C.byref(a),
            o["tag_scores"].ctypes.data, scap, C.byref(b))
        return rc, (a.value, b.value), o

    for tcap, scap, what in ((stok // 2, ssc, "token_capacity"), (stok - 1, ssc, "token_capacity"),
                             (stok, ssc // 2, "score_capacity"), (stok, ssc - 1, "score_capacity")):
        rc, totals, _ = spans(tcap, scap)
        _fail(rc, what)
        assert totals == (stok, ssc), (tcap, scap, totals)
    rc, totals, o = spans(stok, ssc)
    assert rc == 0 and totals == (stok, ssc)
    o["token_cands"] = o["token_cands"].reshape(-1, max(nt, 1))[:, :nt]
    for k, v in o.items():
        assert np.array_equal(v[: len(full["spans." + k])], full["spans." + k]), k


def _child(d, mode):
    p, text, offs = _load(d)
    if mode == "trace":
        p.predict_batch(text, offs)
        p.predict_batch_compact(text, offs, tags=True, tag_scores=True)
        p.token_spans(text, offs, tags=True, tag_scores=True)
        return
    out = _outputs(p, text, offs)
    np.savez(os.path.join(d, "many.npz"), **out)
    _overflow(p, text, offs, out)


def _run_child(d, mode, env):
    code = ("import sys; sys.path[:0] = [%r, %r]\nimport test_gpu_batch_pipeline as t; t._child(%r, %r)\n"
            % (HERE, os.path.dirname(HERE), str(d), mode))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, **env))
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stderr


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    d = tmp_path_factory.mktemp("batch_pipeline")
    _workload(d)
    return d


def test_many_chunks_equal_one_chunk(work, monkeypatch):
    monkeypatch.setenv("VPT_CHUNK_BYTES", ONE_CHUNK_BYTES)
    p, text, offs = _load(work)
    one = _outputs(p, text, offs)
    assert one["compact_scores.tag_scores"].size > 0 and int((one["compact_tags.token_ids"] >= 0).sum()) > 1000
    _run_child(work, "outputs", MANY_CHUNKS)
    many = np.load(os.path.join(work, "many.npz"))
    assert sorted(many.files) == sorted(one)
    for k, v in one.items():
        assert v.dtype == many[k].dtype and v.shape == many[k].shape and v.tobytes() == many[k].tobytes(), k


def test_trace_prints_one_line_per_chunk(work):
    err = _run_child(work, "trace", dict(MANY_CHUNKS, VPT_TRACE="1"))
    seen = {}
    for label, i in re.findall(r"^\[vpt (\w+)\] chunk (\d+) \(", err, re.M):
        seen.setdefault(label, []).append(int(i))
    assert sorted(seen) == ["batch", "compact", "spans"], err[-2000:]
    for label, idx in seen.items():
        assert idx == list(range(len(idx))), label
    assert len(seen["batch"]) == len(seen["compact"]) == 23
    assert len(seen["spans"]) > 23
