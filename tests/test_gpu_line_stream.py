"""The line stream (vpt_line_stream_*): the loops of vpt_tokenize_lines, vpt_tokenize_lines_tags and vpt_evaluate_lines
fed in pieces.  For every way of cutting the input into feeds, the stream's output equals the whole-buffer call's on the
concatenation, and that equals the CPU oracle's restatement of the reference CLI loops.  Also: flush, errors and
poisoning, bounded host memory, concurrent streams, free mid-stream, and the CLIs reading stdin incrementally."""
import ctypes as C
import itertools
import os
import random
import select
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

import vaporetto_b200 as vb
from vpt_testlib import eval_oracle as eo
from vpt_testlib import synth
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.oracle import OraclePredictor
from test_gpu_lines import _random_lines
from test_gpu_parity import _random_model, make, read

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
TOOLS = os.path.join(os.path.dirname(HERE), "tools")
MODEL = os.path.join(HERE, "golden", "model.bin")
DOCS = os.path.join(HERE, "golden", "docs.tok")
CHUNKS = ["64", "4096", None]  # VPT_CHUNK_BYTES (None: the default, 16 MiB)

SEMANTICS = [
    b"", b"\n", b"\n\n\n", b"\r\n", b"\r", b"a", b"a\n", b"a\r", b"a\r\n", b"a\r\r\n", b"a\rb\n", b"\r\r",
    "まぁ社長は火星猫だ".encode(),
    "まぁ社長は火星猫だ\r".encode(),                                     # a trailing '\r'
    "まぁ社長は火星猫だ\r\nまぁ社長は火星猫だ".encode(),                  # an unterminated last line
    "火星 猫/です\\ね\n\n 火星\n/\n\\\n".encode(),                        # escapes of ' ', '/', '\\'
    "まぁ\x00社長\n火星猫\n\x00\n".encode(),                               # NUL lines -> empty lines
    b"\xe3\x81\n" + "火星猫\n".encode() + b"\xff\xfe\n\xc0\x80\n\xe3",       # malformed UTF-8 lines -> empty lines
    "\U00020000\U0002a6df火星été ab12 ｶﾀｶﾅ\n".encode(),
    "ｶﾞｰﾃﾞﾝ－ハウス―A–B─C ｢x｣ ～ ､ ･ ｡\nVaporetto 1.5 (v0.6.5) - 100%\n".encode(),
    "\n".join("まぁ社長は火星猫だ"[: 1 + i % 9] for i in range(300)).encode(),
]


def long_lines():
    # a line over 64 KiB between short ones; it is longer than the 64- and 4096-byte chunks
    return ("まぁ社長は火星猫だ\n" * 3 + "火星猫だ" * 6000 + "\r\n" + "まぁ社長は\n" * 5).encode()


def stream(p, pieces, kind="tokenize", flush_after=(), **flags):
    """Runs a stream over `pieces`; returns (output, n_lines) for tokenize, the totals for evaluate."""
    parts = []
    with p.line_stream(kind, **flags) as s:
        for i, piece in enumerate(pieces):
            parts.append(s.feed(piece))
            if i in flush_after:
                parts.append(s.flush())
        r = s.finish()
    if kind == "evaluate":
        assert parts == [b""] * len(parts)
        return r
    return b"".join(parts) + r[0], r[1]


def splits(data, rng, big):
    """One feed; 1-byte feeds (small inputs); random sizes from 0 to 3x the chunk size with empty feeds mixed in."""
    yield [data]
    if len(data) <= 2048:
        yield [data[i:i + 1] for i in range(len(data))]
    for _ in range(2):
        pieces, pos = [], 0
        while pos < len(data):
            n = 0 if rng.random() < 0.15 else rng.randrange(0, 3 * big + 1)
            pieces.append(data[pos:pos + n])
            pos += n
        yield pieces


def chunk_size(chunk):
    return int(chunk) if chunk else 16 << 20


@pytest.fixture(scope="module")
def kat():
    mb = read("model.bin")
    return make(mb), OraclePredictor(mb)


@pytest.fixture(scope="module")
def kat_tags():
    mb = read("model.bin")
    return vb.Predictor(vb.Model.read(mb), predict_tags=True), OraclePredictor(mb, predict_tags=True)


def check_tokenize(p, o, data, rng, big, modes, oracle=True):
    for flags in modes:
        want, wl = p.tokenize_lines(data, **flags)
        want = want.tobytes()
        if oracle:
            assert (want, wl) == o.tokenize_lines(data, **flags), (flags, data[:100])
        for pieces in splits(data, rng, big):
            got, nl = stream(p, pieces, **flags)
            assert nl == wl and got == want, (flags, [len(x) for x in pieces][:20], data[:100])


MODES = [dict(no_norm=n, wsconst=w) for n, w in itertools.product((False, True), ("", "DRHTKO", "G"))]


@pytest.mark.parametrize("chunk", CHUNKS)
def test_equivalence_tokenize(kat, chunk, monkeypatch):
    """Line endings, escapes, NUL and malformed UTF-8, docs.tok, a line over 64 KiB, an unterminated last line, a trailing
    '\\r', empty input and input of only '\\n', under every split, with no_norm both ways and three --wsconst sets."""
    if chunk:
        monkeypatch.setenv("VPT_CHUNK_BYTES", chunk)
    p, o = kat
    rng = random.Random(11)
    for data in SEMANTICS + [open(DOCS, "rb").read(), long_lines()]:
        check_tokenize(p, o, data, rng, chunk_size(chunk), MODES)


def test_cut_inside_characters_and_crlf(kat, monkeypatch):
    """Two feeds, cut at every offset of a short line: inside each multi-byte character and between '\\r' and '\\n'."""
    p, o = kat
    data = "まぁ社長\r\n火星é\U00020000猫\r\nab\r".encode()
    want, wl = o.tokenize_lines(data)
    for chunk in ("64", None):
        if chunk:
            monkeypatch.setenv("VPT_CHUNK_BYTES", chunk)
        for k in range(len(data) + 1):
            assert stream(p, [data[:k], data[k:]]) == (want, wl), k
            assert stream(p, [data[:k], b"", data[k:]], flush_after={0}) == (want, wl), k


@pytest.mark.parametrize("chunk", CHUNKS)
def test_equivalence_random_models(chunk, monkeypatch):
    if chunk:
        monkeypatch.setenv("VPT_CHUNK_BYTES", chunk)
    rng = np.random.default_rng(23)
    prng = random.Random(23)
    for cw, tw, maxdict in [(3, 3, 3), (2, 4, 6)]:
        m, alpha = _random_model(rng, cw, tw, maxdict=maxdict)
        alphabet = list(alpha) + list(" /\\é\U00020000") + list("ab.-ｱ－―｢､")
        mb = encode_model(m)
        p, o = make(mb), OraclePredictor(mb)
        for n_lines, maxlen in ((300, 80), (5, 3000)):
            data = _random_lines(rng, n_lines, alphabet, maxlen)
            check_tokenize(p, o, data, prng, chunk_size(chunk), [dict(no_norm=False), dict(no_norm=True, wsconst="DG")])


def test_line_longer_than_default_chunk(kat):
    """A 17 MB line (longer than the default chunk) between short lines, fed in 1 MiB pieces."""
    p, _ = kat
    data = "まぁ社長は火星猫だ\n".encode() * 10 + "火星猫だ".encode() * ((17 << 20) // 12 + 1) + b"\n" + "猫\n".encode()
    assert max(len(x) for x in data.split(b"\n")) > 16 << 20
    want, wl = p.tokenize_lines(data)
    got, nl = stream(p, [data[i:i + (1 << 20)] for i in range(0, len(data), 1 << 20)])
    assert nl == wl and got == want.tobytes()


@pytest.mark.parametrize("chunk", ["4096", None])
def test_equivalence_tags(kat_tags, chunk, monkeypatch):
    """--predict-tags on the bundled model and on a synthetic tag model (1 500 tag models)."""
    if chunk:
        monkeypatch.setenv("VPT_CHUNK_BYTES", chunk)
    p, o = kat_tags
    rng = random.Random(3)
    data = ("まぁ社長は火星猫だ\r\n\nまぁ良いだろう\nVaporetto 1.5/2 a\\b\n" + "火星猫は社長だ" * 40 + "\n猫").encode()
    check_tokenize(p, o, data, rng, chunk_size(chunk),
                   [dict(no_norm=n, wsconst=w, predict_tags=True) for n, w in ((False, ""), (True, ""), (False, "G"))])
    mb = synth.gen_model_bccwj_shaped(n_patterns=30_000, sample_sentences=50_000, tag_models=1_500)
    ps, os_ = vb.Predictor(vb.Model.read(mb), predict_tags=True), OraclePredictor(mb, predict_tags=True)
    text, offs, _ = synth.gen_text(3000, 40, seed=synth.TEXT_SEED + 31)
    lines = [text[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)]
    lines[3], lines[17], lines[18] = b"", b"a\x00b", b"\xff\xfe"
    data = b"\r\n".join(lines)
    check_tokenize(ps, os_, data, rng, chunk_size(chunk), [dict(no_norm=n, predict_tags=True) for n in (False, True)])


def gold_corpus():
    """A gold corpus in the tokenized format (the oracle's tagged output of synthetic text, with merged and split tokens,
    CRLF, empty lines, a line over 64 KiB and an unterminated last line), and its predictor pair."""
    mb = synth.gen_model_bccwj_shaped(n_patterns=30_000, sample_sentences=50_000, tag_models=1_500)
    p, o = vb.Predictor(vb.Model.read(mb), predict_tags=True), OraclePredictor(mb, predict_tags=True)
    text, offs, _ = synth.gen_text(1500, 40, seed=synth.TEXT_SEED + 41)
    raw = b"\n".join(text[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)) + b"\n"
    tagged, _ = o.tokenize_lines(raw, predict_tags=True)
    rng = random.Random(5)
    gold = []
    for line in tagged.decode().split("\n")[:-1]:
        toks = line.split(" ")
        for _ in range(2):  # merge two neighbours (their tags dropped) or split one off
            i = rng.randrange(len(toks))
            if i + 1 < len(toks) and rng.random() < 0.5:
                toks[i:i + 2] = [toks[i].split("/")[0] + toks[i + 1].split("/")[0]]
        gold.append(" ".join(toks))
    long_line = " ".join(gold[:1100])
    assert len(long_line.encode()) > 65536
    parts = [g + ("\r\n" if i % 7 == 0 else "\n") + ("\n" if i % 11 == 0 else "") for i, g in enumerate(gold[1100:])]
    data = ("".join(parts[:100]) + long_line + "\n" + "".join(parts[100:])).encode().rstrip(b"\n")
    return p, o, data


@pytest.mark.parametrize("chunk", CHUNKS)
def test_equivalence_evaluate(kat_tags, chunk, monkeypatch):
    """Evaluate with no_norm x predict_tags on docs.tok and a perturbed synthetic gold corpus, every split."""
    if chunk:
        monkeypatch.setenv("VPT_CHUNK_BYTES", chunk)
    rng = random.Random(8)
    p, o = kat_tags
    pairs = [(p, o, open(DOCS, "rb").read()), gold_corpus(), (p, o, b""), (p, o, b"\n")]
    for (pp, oo, data), no_norm, predict_tags in itertools.product(pairs, (False, True), (False, True)):
        flags = dict(no_norm=no_norm, predict_tags=predict_tags)
        want = pp.evaluate_lines(data, **flags)
        assert want == eo.evaluate_lines(oo, data, **flags)[0]
        for pieces in splits(data, rng, chunk_size(chunk)):
            assert stream(pp, pieces, "evaluate", **flags) == want, flags


def test_flush(kat, monkeypatch):
    """After flush() the delivered bytes are the whole-buffer output of exactly the complete lines fed so far; a partial
    line's output comes once its '\\n' arrives, or at finish."""
    p, _ = kat
    monkeypatch.setenv("VPT_CHUNK_BYTES", "4096")
    lines = ["まぁ社長は火星猫だ", "まぁ良いだろう", "Vaporetto 1.5", "火星猫は社長だ" * 30]
    with p.line_stream() as s:
        got = b""
        fed = b""
        for i, line in enumerate(lines * 20):
            piece = (line + "\r\n").encode()
            half = len(piece) // 2
            got += s.feed(piece[:half])
            got += s.flush()
            assert got == p.tokenize_lines(fed)[0].tobytes()  # the half line is held
            got += s.feed(piece[half:])
            fed += piece
            if i % 3 == 0:
                got += s.flush()
                assert got == p.tokenize_lines(fed)[0].tobytes()
        got += s.feed("猫".encode())
        got += s.flush()
        assert got == p.tokenize_lines(fed)[0].tobytes()
        rest, n = s.finish()
    assert got + rest == p.tokenize_lines(fed + "猫".encode())[0].tobytes() and n == 81
    assert rest == "猫\n".encode()


def expect_error(fn):
    with pytest.raises(vb.VaporettoError) as e:
        fn()
    return e.value.code, str(e.value)


@pytest.mark.parametrize("bad", [b"a  b", b"a\xffb", b" a", b"\\"])
@pytest.mark.parametrize("predict_tags", [False, True])
def test_bad_gold_line_in_third_chunk(kat_tags, monkeypatch, bad, predict_tags):
    """A bad gold line (or invalid UTF-8) in the third of several chunks: the whole-buffer call's status and message,
    line number included; every later call returns the same error."""
    p, o = kat_tags
    monkeypatch.setenv("VPT_CHUNK_BYTES", "1000")
    good = open(DOCS, "rb").read().split(b"\n")[0]
    lines = [good] * 30 + [bad] + [good] * 40 + [b"a  b"] + [good] * 30
    data = b"\n".join(lines) + b"\n"
    assert len(b"\n".join(lines[:30])) > 125 + 250  # past the first two chunks (ramping up from 1000 / 8)
    want = expect_error(lambda: p.evaluate_lines(data, predict_tags=predict_tags))
    assert "(line 30)" in want[1]
    with pytest.raises(eo.GoldError) as oracle:
        eo.evaluate_lines(o, data, predict_tags=predict_tags)
    assert (oracle.value.code, oracle.value.msg) == want
    s = p.line_stream("evaluate", predict_tags=predict_tags)
    try:
        first = None
        for i in range(0, len(data), 97):
            try:
                s.feed(data[i:i + 97])
            except vb.VaporettoError as e:
                first = (e.code, str(e))
                break
        if first is None:
            first = expect_error(s.finish)
        assert first == want
        assert expect_error(lambda: s.feed(good + b"\n")) == want
        assert expect_error(s.flush) == want
        assert expect_error(s.finish) == want
    finally:
        s.close()


def raw_stream(p, sink, kind=0, no_norm=0, wsconst=0, predict_tags=0):
    h = C.c_void_p()
    rc = vb.lib().vpt_line_stream_new(p._h, kind, no_norm, wsconst, predict_tags, C.cast(sink, C.c_void_p), None, C.byref(h))
    return rc, h


def feed_raw(h, data):
    a = np.frombuffer(data, np.uint8)
    return vb.lib().vpt_line_stream_feed(h, a.ctypes.data, a.size)


def test_failing_sink(kat, monkeypatch):
    """A sink that fails on its second call: VPT_IO_ERROR "write callback failed", and no further callbacks."""
    p, _ = kat
    monkeypatch.setenv("VPT_CHUNK_BYTES", "64")
    calls = []

    @vb.STREAM_WRITE_FN
    def sink(ctx, data, n):
        calls.append(n)
        return 1 if len(calls) == 2 else 0

    rc, h = raw_stream(p, sink)
    assert rc == 0
    L = vb.lib()
    try:
        data = "まぁ社長は火星猫だ\n".encode() * 100
        rc = feed_raw(h, data)
        assert rc == 5 and L.vpt_last_error() == b"write callback failed" and len(calls) == 2
        assert feed_raw(h, data) == 5 and L.vpt_last_error() == b"write callback failed"
        assert L.vpt_line_stream_flush(h) == 5 and L.vpt_last_error() == b"write callback failed"
        assert L.vpt_line_stream_finish(h, None, None) == 5
        assert len(calls) == 2
    finally:
        L.vpt_line_stream_free(h)


def test_calls_after_finish(kat):
    p, _ = kat
    s = p.line_stream()
    s.feed(b"a\n")
    assert s.finish()[1] == 1
    for call in (lambda: s.feed(b"b\n"), s.flush, s.finish):
        code, msg = expect_error(call)
        assert code == 2 and "already finished" in msg
    s.close()
    s.close()


def test_flags_rejected_at_new(kat):
    """Invalid flags are rejected by vpt_line_stream_new with the whole-buffer calls' statuses and messages."""
    p, _ = kat
    L = vb.lib()

    @vb.STREAM_WRITE_FN
    def sink(ctx, data, n):
        return 0

    def whole(fn, *args):
        rc = fn(*args)
        return rc, L.vpt_last_error()

    for kind in (0, 1):
        # a wsconst bit that is not a character type
        want = whole(L.vpt_tokenize_lines, p._h, b"a", 1, 0, 1, None, 0, None, None)
        rc, h = raw_stream(p, sink, kind=kind, wsconst=1)
        assert (rc, L.vpt_last_error()) == want and want[0] == 2 and not h.value
        # tags on a predictor created without tags
        want = whole(L.vpt_evaluate_lines, p._h, b"a", 1, 0, 0, 1, C.byref(vb._EvalCounts()), None, 0)
        rc, h = raw_stream(p, sink, kind=kind, predict_tags=1)
        assert (rc, L.vpt_last_error()) == want and want[0] == 2 and not h.value
    # a tag model beyond the device limits (a tag slot with 65 candidates)
    m = dict(char_ngrams=[], type_ngrams=[], dict=[], bias=1, char_window=1, type_window=1,
             tag_models=[dict(token="猫", tags=[[str(k) for k in range(65)]], char_ngrams=[], type_ngrams=[],
                              bias=list(range(65)))])
    pt = vb.Predictor(vb.Model.read(encode_model(m)), predict_tags=True)
    want = expect_error(lambda: pt.tokenize_lines(b"a\n", predict_tags=True))
    assert want[0] == 17
    assert expect_error(lambda: pt.line_stream(predict_tags=True)) == want
    assert expect_error(lambda: pt.line_stream("evaluate", predict_tags=True)) == want
    # a tokenize stream needs a sink; an evaluate stream does not
    h = C.c_void_p()
    assert L.vpt_line_stream_new(p._h, 0, 0, 0, 0, None, None, C.byref(h)) == 2
    assert L.vpt_line_stream_new(p._h, 1, 0, 0, 0, None, None, C.byref(h)) == 0
    L.vpt_line_stream_free(h)
    assert L.vpt_line_stream_new(p._h, 2, 0, 0, 0, C.cast(sink, C.c_void_p), None, C.byref(h)) == 2


def vm_hwm() -> int:
    """The process's peak resident memory in bytes: VmHWM, or getrusage's ru_maxrss where /proc does not report it."""
    for line in open("/proc/self/status"):
        if line.startswith("VmHWM:"):
            return int(line.split()[1]) * 1024
    import resource
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024


def test_bounded_memory():
    """2 GiB of config-2-shaped lines, one ~16 MiB block fed 128 times into a sink that only counts: the peak resident
    memory grows by less than 256 MiB between 256 MiB fed and 2 GiB fed, and the output is 128 times the block's."""
    mb = synth.gen_model_bccwj_shaped(n_patterns=30_000, sample_sentences=50_000)
    p = vb.Predictor(vb.Model.read(mb))
    text, offs, _ = synth.gen_text(150_000, 40, seed=synth.TEXT_SEED + 51)
    lines =[text[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)]
    block = b"\n".join(lines) + b"\n"
    block = block[: block.rindex(b"\n", 0, 16 << 20) + 1]
    one = len(p.tokenize_lines(block)[0])
    del text, offs, lines
    total = [0]

    @vb.STREAM_WRITE_FN
    def sink(ctx, data, n):
        total[0] += n
        return 0

    rc, h = raw_stream(p, sink)
    assert rc == 0
    L = vb.lib()
    try:
        a = np.frombuffer(block, np.uint8)
        for i in range(128):
            assert L.vpt_line_stream_feed(h, a.ctypes.data, a.size) == 0
            if i == 15:
                hwm0 = vm_hwm()
        n = C.c_uint64()
        assert L.vpt_line_stream_finish(h, C.byref(n), None) == 0
        hwm1 = vm_hwm()
    finally:
        L.vpt_line_stream_free(h)
    assert n.value == 128 * block.count(b"\n")
    assert total[0] == 128 * one
    assert hwm1 - hwm0 < 256 << 20, (hwm0, hwm1)


def test_two_streams_two_threads(kat, monkeypatch):
    """Two streams on one predictor, driven from two threads at once, both give the whole-buffer output."""
    p, o = kat
    monkeypatch.setenv("VPT_CHUNK_BYTES", "4096")
    datas = [("まぁ社長は火星猫だ\n" * 3000).encode(), ("Vaporetto 1.5\r\n火星猫は社長だ\n" * 2500).encode()]
    wants = [p.tokenize_lines(datas[0])[0].tobytes(), p.tokenize_lines(datas[1], no_norm=True)[0].tobytes()]
    results = [None, None]
    errors = []

    def run(k):
        try:
            rng = random.Random(k)
            d = datas[k]
            pieces, pos = [], 0
            while pos < len(d):
                n = rng.randrange(0, 3000)
                pieces.append(d[pos:pos + n])
                pos += n
            for _ in range(3):
                results[k] = stream(p, pieces, no_norm=bool(k))
                time.sleep(0)
        except BaseException as e:  # reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=run, args=(k,)) for k in (0, 1)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    assert results[0] == (wants[0], 3000) and results[1] == (wants[1], 5000)


def test_free_mid_stream(kat, monkeypatch):
    """free with chunks in flight calls nothing back, and the predictor still gives correct whole-buffer output."""
    p, o = kat
    monkeypatch.setenv("VPT_CHUNK_BYTES", "4096")
    calls = [0]

    @vb.STREAM_WRITE_FN
    def sink(ctx, data, n):
        calls[0] += 1
        return 0

    rc, h = raw_stream(p, sink)
    assert rc == 0
    data = ("まぁ社長は火星猫だ\n" * 2000).encode()
    assert feed_raw(h, data + "まぁ社長".encode()) == 0
    before = calls[0]
    assert before > 0  # back-pressure delivered the oldest chunks
    vb.lib().vpt_line_stream_free(h)
    assert calls[0] == before
    with p.line_stream() as s:  # closed mid-stream through the Python object as well
        s.feed(data)
    got, nl = p.tokenize_lines(data)
    assert (got.tobytes(), nl) == o.tokenize_lines(data)


def read_until(f, n, timeout):
    """Reads exactly n bytes from pipe f (fails after `timeout` seconds)."""
    buf = b""
    end = time.monotonic() + timeout
    while len(buf) < n:
        left = end - time.monotonic()
        assert left > 0, f"timed out with {len(buf)} of {n} bytes: {buf!r}"
        r, _, _ = select.select([f], [], [], left)
        if r:
            chunk = os.read(f.fileno(), n - len(buf))
            assert chunk, f"end of output after {len(buf)} of {n} bytes"
            buf += chunk
    return buf


def test_predict_cli_incremental(kat):
    """The predict CLI hands back each complete line while stdin stays open, then the rest at the end."""
    p, o = kat
    first = "まぁ社長は火星猫だ\nまぁ良いだろう\n".encode()
    third = "Vaporetto 1.5 火星猫\r\n".encode()
    want_first = o.tokenize_lines(first)[0]
    want_all = o.tokenize_lines(first + third)[0]
    proc = subprocess.Popen([sys.executable, os.path.join(TOOLS, "predict_cli.py"), "--model", MODEL],
                            stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    try:
        proc.stdin.write(first + third[:7])
        proc.stdin.flush()
        assert read_until(proc.stdout, len(want_first), 60) == want_first
        proc.stdin.write(third[7:])
        proc.stdin.close()
        rest = proc.stdout.read()
        assert proc.wait(60) == 0
        assert want_first + rest == want_all
    finally:
        if proc.poll() is None:
            proc.kill()
            proc.wait()


def test_evaluate_cli_in_pieces(kat_tags):
    """The evaluate CLI fed in pieces prints what the whole-buffer evaluate gives."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("evaluate_cli", os.path.join(TOOLS, "evaluate_cli.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    p, _ = kat_tags
    docs = open(DOCS, "rb").read()
    data = docs * 50 + "まぁ/名詞 社長/名詞 は 火星 猫 だ\r\n".encode() * 30
    for args, flags in (([], {}), (["--predict-tags", "--metric", "word"], dict(predict_tags=True))):
        want = cli.report(p.evaluate_lines(data, **flags), "word" if "word" in args else "char")
        proc = subprocess.Popen([sys.executable, os.path.join(TOOLS, "evaluate_cli.py"), "--model", MODEL, *args],
                                stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
        try:
            for i in range(0, len(data), 333):
                proc.stdin.write(data[i:i + 333])
                proc.stdin.flush()
            proc.stdin.close()
            out = proc.stdout.read()
            assert proc.wait(60) == 0
            assert out.decode() == want
        finally:
            if proc.poll() is None:
                proc.kill()
                proc.wait()
