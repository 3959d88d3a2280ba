"""vpt_tokenize_dev / Predictor.tokenize_device: the tokenized text of documents already in GPU memory as a device string
column, against the per-document CPU oracle (tests/native/tokenize_doc_oracle.cpp), against Predictor.tokenize_lines on
the same documents joined by '\\n', and its statuses against token_spans_device; tags and PatternMatchTagger rules,
offset layouts, out-of-range documents, the output capacity, graph capture, streams, the host-side errors and the C++
wrapper."""
import os
import random
import subprocess

import numpy as np
import pytest
import torch

import vaporetto_b200 as vb
from vpt_testlib import tag_rules as tr
from vpt_testlib.tokenize_doc_oracle import TokenizeDocOracle
from test_gpu_parity import make, read
from test_spans_cpu import batch, random_doc
from test_gpu_spans_device import random_docs, to_dev

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
WSCONST_SAMPLE = ["", "G", "DRHTKOG", "D"]
RULE_TAGS = ["x", "名詞", "a b", "s/l", "b\\s", "ｶﾅ/ 😀", "\\/ "]


def run(p, text, off, dtype=torch.int64, **kw):
    t, o = to_dev(text, off, dtype)
    d = p.tokenize_device(t, o, **kw)
    chars, offs, status = d.to_host()
    b = chars.tobytes()
    assert bool(d.complete.item())
    return [b[offs[i]:offs[i + 1]] for i in range(offs.size - 1)], status, d


def line_docs(docs):
    """The documents the line loop writes as one line each: no '\\n', no '\\r' in front of the '\\n' it gets."""
    enc = [d if isinstance(d, bytes) else d.encode() for d in docs]
    return [i for i, d in enumerate(enc) if b"\n" not in d and not d.endswith(b"\r")]


def check_vs_lines(p, docs, got, **kw):
    keep = line_docs(docs)
    enc = [d if isinstance(d, bytes) else d.encode() for d in docs]
    out, nl = p.tokenize_lines(b"".join(enc[i] + b"\n" for i in keep), **kw)
    assert nl == len(keep)
    assert out.tobytes() == b"".join(got[i] + b"\n" for i in keep), kw
    return keep


def spans_status(p, text, off, **kw):
    t, o = to_dev(text, off)
    kw.pop("predict_tags", None), kw.pop("tag_rules", None)
    return p.token_spans_device(t, o, **kw).to_host().status


@pytest.mark.parametrize("model", ["tantivy_model.bin", "model.bin"])
def test_random_batches(model):
    mb = read(model)
    p, o = make(mb), TokenizeDocOracle(mb)
    docs = random_docs(11)
    docs[7:7] = ["\r\n社長\r", "a\nb", "\r"]
    text, off = batch(docs)
    for k, ws in enumerate(WSCONST_SAMPLE):
        for no_norm in (False, True):
            got, status, _ = run(p, text, off, no_norm=no_norm, wsconst=ws)
            assert np.array_equal(status, spans_status(p, text, off, no_norm=no_norm, wsconst=ws))
            keep = check_vs_lines(p, docs, got, no_norm=no_norm, wsconst=ws)
            assert len(keep) < len(docs)
            if k % 2 == 0:
                want, wst = o.tokenize_docs(text, off, no_norm=no_norm, wsconst=ws)
                assert np.array_equal(status, wst)
                assert got == want, (ws, no_norm)
    assert status[[5, 6, 10]].tolist() == [1, 2, 3] and got[5] == got[6] == got[10] == b""


def rules_for(o, text, off, rng, no_norm):
    """Rules for surfaces the oracle's tagged output holds, keyed as the filter sees them, tags with ' ', '/', '\\'."""
    docs, _ = o.tokenize_docs(text, off, no_norm=no_norm, predict_tags=True)
    toks = sorted({s for d in docs if d for s, _ in tr.parse_tokenized_line(d.decode())})
    rng.shuffle(toks)
    fw = lambda s: s if no_norm else "".join(chr(vb.lib().vpt_kytea_fullwidth(ord(c))) for c in s)
    return {fw(s): [rng.choice(RULE_TAGS + [None]) for _ in range(rng.randint(1, o.n_tags + 1))] for s in toks[:100]}


def test_tags_and_rules():
    mb = read("model.bin")
    assert tr.model_tags_nonempty(mb)
    p, o = make(mb, tags=True), TokenizeDocOracle(mb, predict_tags=True)
    docs = ["まぁ社長は火星猫だ", "まぁ良いだろう\nまぁ社長は\r\n火星猫だ", "火星 猫/社長\\は"] + random_docs(12, 120)
    text, off = batch(docs)
    rng = random.Random(13)
    for ws in ("", "G", "DRHTKOG"):
        for no_norm in (False, True):
            got, status, _ = run(p, text, off, no_norm=no_norm, wsconst=ws, predict_tags=True)
            assert np.array_equal(status, spans_status(p, text, off, no_norm=no_norm, wsconst=ws))
            check_vs_lines(p, docs, got, no_norm=no_norm, wsconst=ws, predict_tags=True)
            want, _ = o.tokenize_docs(text, off, no_norm=no_norm, wsconst=ws, predict_tags=True)
            assert got == want, (ws, no_norm)
            assert b"/" in got[0]
            rules = rules_for(o, text, off, rng, no_norm)
            tagger = vb.PatternMatchTagger(p, rules)
            got_r, _, _ = run(p, text, off, no_norm=no_norm, wsconst=ws, predict_tags=True, tag_rules=tagger)
            check_vs_lines(p, docs, got_r, no_norm=no_norm, wsconst=ws, predict_tags=True, tag_rules=tagger)
            want_r, _ = o.tokenize_docs(text, off, no_norm=no_norm, wsconst=ws, predict_tags=True, rules=rules)
            assert got_r == want_r, (ws, no_norm)
            assert got_r != got


def test_tags_on_a_model_without_tag_slots():
    p = make(read("tantivy_model.bin"), tags=True)
    assert p.n_tags == 0
    text, off = batch(random_docs(14, 60))
    plain, _, _ = run(p, text, off)
    tagged, _, _ = run(p, text, off, predict_tags=True)
    assert tagged == plain


def test_predict_tags_rules_errors():
    mb = read("model.bin")
    p = make(mb, tags=True)
    text, off = batch(["まぁ社長は火星猫だ"])
    t, o = to_dev(text, off)
    with pytest.raises(vb.VaporettoError, match="predict_tags"):
        p.tokenize_device(t, o, tag_rules=vb.PatternMatchTagger(p, {"猫": ["x"]}))
    with pytest.raises(vb.VaporettoError, match="another predictor"):
        p.tokenize_device(t, o, predict_tags=True, tag_rules=vb.PatternMatchTagger(make(mb, tags=True), {"猫": ["x"]}))
    with pytest.raises(vb.VaporettoError) as e:
        make(mb).tokenize_device(t, o, predict_tags=True)
    with pytest.raises(vb.VaporettoError) as e2:
        make(mb).tokenize_lines(b"x\n", predict_tags=True)
    assert str(e.value) == str(e2.value)


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
def test_layouts_and_bad_ranges(dtype):
    """int32 and int64 offsets, offsets[0] > 0, text views at every alignment 0-15 ending on the storage's last byte, and
    documents out of range: VPT_SENT_BAD_RANGE, an empty string, neighbours unchanged."""
    p = make(read("tantivy_model.bin"))
    docs = random_docs(15, 80)
    text, off = batch(docs)
    want, wst, _ = run(p, text, off)
    pad = b"\xe3\x81\x82" * 7
    body = pad + text
    off2 = off.astype(np.int64) + len(pad)
    for a in range(16):
        store = torch.zeros(a + len(body), dtype=torch.uint8, device="cuda")
        store[a:] = torch.frombuffer(bytearray(body), dtype=torch.uint8).cuda()
        d = p.tokenize_device(store[a:], torch.as_tensor(off2, dtype=dtype).cuda())
        chars, offs, status = d.to_host()
        b = chars.tobytes()
        assert [b[offs[i]:offs[i + 1]] for i in range(len(docs))] == want, a
        assert np.array_equal(status, wst)
    store = torch.frombuffer(bytearray(text + "社長".encode() * 20), dtype=torch.uint8).cuda()
    nb = len(text)
    bad = off.astype(np.int64).copy()
    bad[10] = nb + 9
    bad = np.append(bad, nb + 30)
    d = p.tokenize_device(store[:nb], torch.as_tensor(bad, dtype=dtype).cuda())
    chars, offs, status = d.to_host()
    b = chars.tobytes()
    got = [b[offs[i]:offs[i + 1]] for i in range(len(docs) + 1)]
    assert status[[9, 10, len(docs)]].tolist() == [4, 4, 4]
    assert got[9] == got[10] == got[len(docs)] == b""
    keep = [i for i in range(len(docs)) if i not in (9, 10)]
    assert [got[i] for i in keep] == [want[i] for i in keep]
    assert np.array_equal(status, spans_status(p, text, bad))


def test_capacity():
    """The bound, exactly the total, one byte short (only the last non-empty document is missing, every byte outside the
    written ranges keeps its canary), and 0 with no output buffer (offsets only, equal to the full call's)."""
    mb = read("model.bin")
    p = make(mb, tags=True)
    docs = random_docs(16, 100) + ["社長", "", b"\xff"]
    text, off = batch(docs)
    t, o = to_dev(text, off)
    full = p.tokenize_device(t, o, predict_tags=True)
    chars, offs, status = full.to_host()
    total = int(offs[-1])
    bound = vb.lib().vpt_tokenize_dev_out_bound(p._h, None, len(docs), len(text), 1)
    assert full.chars.numel() == bound >= total
    last = max(i for i in range(len(docs)) if offs[i + 1] > offs[i])
    n, ws_bytes = len(docs), vb.lib().vpt_tokenize_dev_workspace_size(p._h, None, len(docs), len(text), 1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    for cap in (bound, total, total - 1, 0):
        canary = torch.full((cap + 64,), 0xA5, dtype=torch.uint8, device="cuda")
        out_off = torch.full((n + 1,), -7, dtype=torch.int64, device="cuda")
        status_d = torch.full((n,), 99, dtype=torch.uint8, device="cuda")
        rc = vb.lib().vpt_tokenize_dev(p._h, None, t.data_ptr(), len(text), o.data_ptr(), 8, n, 0, 0, 1,
                                       out_off.data_ptr(), canary.data_ptr() if cap else None, cap, status_d.data_ptr(),
                                       ws.data_ptr(), ws_bytes, torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        torch.cuda.synchronize()
        assert np.array_equal(out_off.cpu().numpy(), offs), cap
        assert np.array_equal(status_d.cpu().numpy(), status)
        got = canary.cpu().numpy()
        expect = np.full(cap + 64, 0xA5, np.uint8)
        for i in range(n):
            if offs[i + 1] <= cap:
                expect[offs[i]:offs[i + 1]] = chars[offs[i]:offs[i + 1]]
        assert np.array_equal(got, expect), cap
        if cap == total - 1:
            assert all(offs[i + 1] <= cap for i in range(last)) and offs[last + 1] > cap
    short = p.tokenize_device(t, o, predict_tags=True, out_capacity=total - 1)
    assert not bool(short.complete.item())
    with pytest.raises(vb.VaporettoError, match="out_capacity"):
        short.to_host()
    sizing = p.tokenize_device(t, o, predict_tags=True, out_capacity=0)
    assert np.array_equal(sizing.offsets.cpu().numpy(), offs)


def test_graph_capture_and_streams():
    p = make(read("tantivy_model.bin"))
    rng = random.Random(17)
    docs = [random_doc(rng, 30) for _ in range(500)]
    text, off = batch(docs)
    t, o = to_dev(text, off)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        p.tokenize_device(t, o)  # warm-up outside the graph (module loads)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        d = p.tokenize_device(t, o, wsconst="G")
    text2, off2 = batch(docs[::-1])  # same sizes, new bytes and offsets
    t.copy_(torch.frombuffer(bytearray(text2), dtype=torch.uint8).cuda())
    o.copy_(torch.as_tensor(off2.astype(np.int64)).cuda())
    g.replay()
    torch.cuda.synchronize()
    want, _, _ = run(p, text2, off2, wsconst="G")
    assert d.strings() == [w.decode() for w in want]
    texts = [batch(random_docs(18 + k, 200)) for k in range(2)]
    devs = [to_dev(*tb) for tb in texts]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for st in streams:
        st.wait_stream(torch.cuda.current_stream())
    outs = [p.tokenize_device(tt, oo, stream=st) for (tt, oo), st in zip(devs, streams)]
    for d, (text, off) in zip(outs, texts):
        assert d.to_host()[0].tobytes() == b"".join(run(p, text, off)[0])


def test_errors_on_the_host():
    p = make(read("tantivy_model.bin"))
    text, off = batch(["東京特許許可局", "社長"])
    t, o = to_dev(text, off)
    n, nb = 2, len(text)
    L = vb.lib()
    need = L.vpt_tokenize_dev_workspace_size(p._h, None, n, nb, 0)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out_off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    chars = torch.zeros(64, dtype=torch.uint8, device="cuda")
    status = torch.full((n,), 77, dtype=torch.uint8, device="cuda")

    def call(t_ptr=t.data_ptr(), nbytes=nb, ws_bytes=need, chars_ptr=chars.data_ptr(), ob=8):
        return L.vpt_tokenize_dev(p._h, None, t_ptr, nbytes, o.data_ptr(), ob, n, 0, 0, 0, out_off.data_ptr(), chars_ptr,
                                  64, status.data_ptr(), ws.data_ptr(), ws_bytes, torch.cuda.current_stream().cuda_stream)
    assert call(ws_bytes=need - 1) == 2 and b"workspace" in L.vpt_last_error()
    host = np.frombuffer(bytearray(text), np.uint8)
    assert call(t_ptr=host.ctypes.data) == 2 and b"d_utf8" in L.vpt_last_error()
    assert call(chars_ptr=None) == 2 and b"d_out" in L.vpt_last_error()
    assert call(nbytes=1 << 32) == 2 and b"limit" in L.vpt_last_error()
    assert call(ob=2) == 2 and b"offset_bytes" in L.vpt_last_error()
    assert L.vpt_tokenize_dev(p._h, None, t.data_ptr(), nb, o.data_ptr(), 8, n, 0, 1 << 8, 0, out_off.data_ptr(),
                              chars.data_ptr(), 64, status.data_ptr(), ws.data_ptr(), need, None) == 2
    torch.cuda.synchronize()
    assert status.tolist() == [77, 77]  # nothing ran
    with pytest.raises(vb.VaporettoError):
        p.tokenize_device(t.cpu(), o)
    with pytest.raises(vb.VaporettoError):
        p.tokenize_device(t, o, out_capacity=-1)
    d = p.tokenize_device(t, torch.zeros(1, dtype=torch.int32, device="cuda"))
    assert d.offsets.tolist() == [0] and d.strings() == []


def test_cpp_wrapper(tmp_path):
    exe = str(tmp_path / "tokenize_dev_cpp")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-o", exe,
                           os.path.join(HERE, "native", "tokenize_dev_cpp.cpp"), "-I" + os.path.join(cuda, "include"),
                           "-L" + os.path.join(ROOT, "vaporetto_b200"), "-lvaporetto_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "vaporetto_b200"), "-L" + os.path.join(cuda, "lib64"),
                           "-lcudart"])
    mb_path = os.path.join(HERE, "golden", "model.bin")
    docs = ["まぁ社長は火星猫だ", "まぁ良いだろう", "火星 猫"]
    out = subprocess.run([exe, mb_path, "1"] + docs, capture_output=True)
    assert out.returncode == 0, out.stderr
    p = make(read("model.bin"), tags=True)
    want, _ = p.tokenize_lines("\n".join(docs).encode() + b"\n", predict_tags=True)
    assert out.stdout == want.tobytes()
