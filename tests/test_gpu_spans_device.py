"""vpt_token_spans_dev / Predictor.token_spans_device: token spans of documents already in GPU memory, against
Predictor.token_spans (the host call, pinned by tests/test_gpu_spans.py against the oracle) on the same bytes, and
against the oracle directly; offset layouts, out-of-range documents, graph capture, streams and the host-side errors."""
import random

import numpy as np
import pytest
import torch

import vaporetto_b200 as vb
from vpt_testlib import spans_oracle as so
from test_gpu_parity import make, read
from test_spans_cpu import batch, random_doc

pytestmark = pytest.mark.gpu

WSCONST_SAMPLE = ["", "G", "O", "DRHTKOG", "KG", "D"]


def to_dev(text: bytes, off, dtype=torch.int64):
    return (torch.frombuffer(bytearray(text), dtype=torch.uint8).cuda(),
            torch.as_tensor(np.asarray(off, np.int64), dtype=dtype).cuda())


def assert_same(r, w, tags, ctx=None):
    assert np.array_equal(r.status, w.status), ctx
    assert np.array_equal(r.n_tokens, w.n_tokens), ctx
    assert np.array_equal(r.token_base, w.token_base), ctx
    assert np.array_equal(r.token_ends, w.token_ends), ctx
    if tags:
        assert np.array_equal(r.token_ids, w.token_ids), ctx
        assert np.array_equal(r.token_cands, w.token_cands), ctx


def check(p, text, off, tags=False, dtype=torch.int64, **kw):
    t, o = to_dev(text, off, dtype)
    d = p.token_spans_device(t, o, tags=tags, **kw)
    r = d.to_host()
    w = p.token_spans(text, np.asarray(off, np.uint64), tags=tags, **kw)
    assert_same(r, w, tags, kw)
    assert np.array_equal(d.token_offsets.cpu().numpy(), r.token_base.astype(np.int64))
    return r


def random_docs(seed, n=300):
    rng = random.Random(seed)
    docs = [random_doc(rng, rng.randrange(1, 120)) for _ in range(n)]
    docs[5:5] = [b"", "a\x00b", b"\xe3\x81", b"\xff\n", "\n", "x" * 129]
    docs[50:50] = [random_doc(rng, 12 * 1024 // 3), random_doc(rng, 32 * 1024 // 3)]  # longer than a scoring tile
    return docs


@pytest.mark.parametrize("model", ["tantivy_model.bin", "model.bin"])
def test_random_batches_vs_host_call(model):
    mb = read(model)
    p, o = make(mb), so.SpansOracle(mb)
    text, off = batch(random_docs(1))
    for ws in WSCONST_SAMPLE:
        for no_norm in (False, True):
            r = check(p, text, off, no_norm=no_norm, wsconst=ws)
    w = o.token_spans(text, off, no_norm=True, wsconst=WSCONST_SAMPLE[-1])
    assert np.array_equal(r.token_ends, w["token_ends"]) and np.array_equal(r.status, w["status"])


def test_tags_vs_host_call_and_oracle():
    mb = read("model.bin")
    p, o = make(mb, tags=True), so.SpansOracle(mb, predict_tags=True)
    text, off = batch(["まぁ社長は火星猫だ", "まぁ良いだろう\nまぁ社長は\r\n火星猫だ"] + random_docs(2, 100))
    for ws in ("", "G", "DRHTKOG"):
        for no_norm in (False, True):
            r = check(p, text, off, tags=True, no_norm=no_norm, wsconst=ws)
    w = o.token_spans(text, off, no_norm=True, wsconst="DRHTKOG", tags=True)
    assert np.array_equal(r.token_ids, w["token_ids"]) and np.array_equal(r.token_cands, w["token_cands"])
    assert (r.token_ids >= 0).any()


def test_tags_on_a_model_without_tag_slots():
    p = make(read("tantivy_model.bin"), tags=True)
    assert p.n_tags == 0
    text, off = batch(random_docs(3, 50))
    r = check(p, text, off, tags=True)
    assert r.token_ids.size > 0 and (r.token_ids == -1).all() and r.token_cands.shape == (r.token_ids.size, 0)


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
def test_layouts(dtype):
    """int32 and int64 offsets, offsets[0] > 0, text views at every alignment 0-15, a last document that ends on the last
    byte of its tensor."""
    p = make(read("tantivy_model.bin"))
    text, off = batch(random_docs(4, 80))
    want = p.token_spans(text, off)
    pad = b"\xe3\x81\x82" * 7  # bytes in front of the first document: offsets[0] > 0
    body = pad + text
    off2 = off.astype(np.int64) + len(pad)
    for a in range(16):
        store = torch.zeros(a + len(body), dtype=torch.uint8, device="cuda")
        store[a:] = torch.frombuffer(bytearray(body), dtype=torch.uint8).cuda()
        view = store[a:]  # ends on the storage's last byte
        assert view.data_ptr() % 16 == (store.data_ptr() + a) % 16
        r = p.token_spans_device(view, torch.as_tensor(off2, dtype=dtype).cuda()).to_host()
        assert_same(r, want, False, a)


def test_bad_ranges():
    """Offsets past n_bytes but inside the tensor's allocation: VPT_SENT_BAD_RANGE, 0 tokens, neighbours unchanged."""
    p = make(read("tantivy_model.bin"))
    docs = random_docs(5, 40)
    text, off = batch(docs)
    store = torch.frombuffer(bytearray(text + "社長".encode() * 20), dtype=torch.uint8).cuda()
    view = store[:len(text)]
    nb = len(text)
    bad = off.astype(np.int64).copy()
    bad[10] = nb + 9       # documents 9 and 10
    bad = np.append(bad, nb + 30)  # one more document at the end
    r = p.token_spans_device(view, torch.as_tensor(bad).cuda()).to_host()
    w = p.token_spans(text, off)
    assert r.status[[9, 10, len(docs)]].tolist() == [4, 4, 4]  # VPT_SENT_BAD_RANGE
    assert r.n_tokens[[9, 10, len(docs)]].tolist() == [0, 0, 0]
    keep = [d for d in range(len(docs)) if d not in (9, 10)]
    assert r.status[keep].tolist() == w.status[keep].tolist()
    for d in keep:
        assert r.spans(d).tolist() == w.spans(d).tolist(), d


def test_graph_capture():
    p = make(read("tantivy_model.bin"))
    rng = random.Random(6)
    docs = [random_doc(rng, 30) for _ in range(500)]
    text, off = batch(docs)
    t, o = to_dev(text, off)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        p.token_spans_device(t, o)  # warm-up outside the graph (module loads)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        d = p.token_spans_device(t, o, wsconst="G")
    text2, off2 = batch(docs[::-1])  # same sizes, new bytes and offsets
    t.copy_(torch.frombuffer(bytearray(text2), dtype=torch.uint8).cuda())
    o.copy_(torch.as_tensor(off2.astype(np.int64)).cuda())
    g.replay()
    torch.cuda.synchronize()
    r = d.to_host()
    assert_same(r, p.token_spans(text2, off2, wsconst="G"), False)


def test_two_streams():
    p = make(read("tantivy_model.bin"))
    texts = [batch(random_docs(7 + k, 200)) for k in range(2)]
    devs = [to_dev(*tb) for tb in texts]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    outs = [p.token_spans_device(t, o, stream=s) for (t, o), s in zip(devs, streams)]
    for d, (text, off) in zip(outs, texts):
        assert_same(d.to_host(), p.token_spans(text, off), False)


def _raw_call(p, t_ptr, nb, o_ptr, n, ws_ptr, ws_bytes, out, ids=None, cands=None):
    return vb.lib().vpt_token_spans_dev(p._h, t_ptr, nb, o_ptr, 8, n, 0, 0, out[0].data_ptr(), out[1].data_ptr(),
                                        out[2].data_ptr(), out[3].data_ptr(), ids, cands, ws_ptr, ws_bytes,
                                        torch.cuda.current_stream().cuda_stream)


def test_errors_on_the_host():
    p = make(read("tantivy_model.bin"))
    text, off = batch(["東京特許許可局", "社長"])
    t, o = to_dev(text, off)
    # tags without predict_tags: the host call's message
    with pytest.raises(vb.VaporettoError) as e:
        p.token_spans_device(t, o, tags=True)
    with pytest.raises(vb.VaporettoError) as e2:
        p.token_spans(text, off, tags=True)
    assert str(e.value) == str(e2.value)
    n, nb = 2, len(text)
    out = [torch.zeros(n + 1, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"),
           torch.full((n,), 77, dtype=torch.uint8, device="cuda"), torch.zeros(nb, dtype=torch.int32, device="cuda")]
    need = vb.lib().vpt_token_spans_dev_workspace_size(p._h, n, nb, 0)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    # a workspace one byte short
    assert _raw_call(p, t.data_ptr(), nb, o.data_ptr(), n, ws.data_ptr(), need - 1, out) == 2
    assert b"workspace" in vb.lib().vpt_last_error()
    # a host pointer
    host = np.frombuffer(bytearray(text), np.uint8)
    assert _raw_call(p, host.ctypes.data, nb, o.data_ptr(), n, ws.data_ptr(), need, out) == 2
    assert b"d_utf8" in vb.lib().vpt_last_error()
    # n_bytes over the limit
    assert _raw_call(p, t.data_ptr(), 1 << 32, o.data_ptr(), n, ws.data_ptr(), need, out) == 2
    assert b"limit" in vb.lib().vpt_last_error()
    torch.cuda.synchronize()
    assert out[2].tolist() == [77, 77]  # nothing ran
    with pytest.raises(vb.VaporettoError):
        p.token_spans_device(t.cpu(), o)
    if torch.cuda.device_count() > 1:
        with pytest.raises(vb.VaporettoError):
            p.token_spans_device(t.to("cuda:1"), o.to("cuda:1"))
        # the raw pointer check too
        t1 = t.to("cuda:1")
        assert _raw_call(p, t1.data_ptr(), nb, o.data_ptr(), n, ws.data_ptr(), need, out) == 2
    # n_docs == 0
    d = p.token_spans_device(t, torch.zeros(1, dtype=torch.int32, device="cuda"))
    assert d.token_offsets.tolist() == [0]
    r = d.to_host()
    assert r.n_tokens.size == 0 and r.token_ends.size == 0
