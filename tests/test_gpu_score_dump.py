"""The predict CLI's --scores / --tag-scores on the device (vpt_line_stream_new_scores, Predictor.line_stream(scores=,
tag_scores=), tools/predict_cli.py) byte for byte against the dump oracle (tests/native/dump_oracle.cpp), through the
line stream: each dump alone and both, --no-norm and the default, --wsconst D and G, with and without tag rules, on the
reference fixtures, random and synthetic models, rejected and edge lines, chunk sizes from 64 B up and every split of a
short input."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import vaporetto_b200 as vb
from golden import reference_kat as kat
from test_gpu_line_stream import vm_hwm
from test_gpu_lines import _random_lines
from test_gpu_parity import _random_model, read
from test_tag_scores_cpu import OVERRUN_MODEL
from vpt_testlib import synth
from vpt_testlib import tag_rules as tr
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.dump_oracle import DumpOracle
from vpt_testlib.oracle import OraclePredictor

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = [(True, False), (False, True), (True, True)]  # (scores, tag_scores)
EDGE = "まぁ社長は火星猫だ\r\n\n\0x\n人\n\xff\n" "a\r\n" + "社長" * 3000 + "\nこの人は地球人だ\nＡＢＣ１２３ abc 123\n"


def stream_out(p, data: bytes, pieces=None, flush_at=None, **kw) -> bytes:
    """The stream's whole output for `data` fed in `pieces` (sizes; default: all at once), flushing after piece
    `flush_at`."""
    out = []
    with p.line_stream(**kw) as st:
        lo = 0
        for k, n in enumerate(pieces or [len(data)]):
            out.append(st.feed(data[lo:lo + n]))
            lo += n
            if flush_at == k:
                out.append(st.flush())
        out.append(st.feed(data[lo:]))
        out.append(st.finish()[0])
    return b"".join(out)


def check(p, d, data, predict_tags, wsconsts=("",), modes=MODES, rules=None, o=None, **kw):
    for no_norm in (False, True):
        for ws in wsconsts:
            for scores, tag_scores in modes:
                if tag_scores and not predict_tags:
                    continue
                got = stream_out(p, data, no_norm=no_norm, wsconst=ws, predict_tags=predict_tags, scores=scores,
                                 tag_scores=tag_scores, tag_rules=None if rules is None else rules[0], **kw)
                lines = None
                if rules is not None:
                    lines = tr.oracle_tokenize_lines(o, data, rules[1], no_norm=no_norm, wsconst=ws)[0]
                want = d.dump_lines(data, no_norm=no_norm, wsconst=ws, scores=scores, tag_scores=tag_scores, token_lines=lines)
                assert got == want, (no_norm, ws, scores, tag_scores)


def test_bundled_and_reference_models():
    mb = read("model.bin")
    check(vb.Predictor(vb.Model.read(mb)), DumpOracle(mb), EDGE.encode("utf-8", "surrogateescape").replace(b"\xc3\xbf", b"\xff"),
          False, wsconsts=("", "D", "G"))
    for model in (kat.PREDICTOR_TEST_MODEL,):
        mb = encode_model(model)
        data = ("この人は地球人だ\n人\n\n人は\n" + EDGE).encode().replace(b"\xc3\xbf", b"\xff")
        check(vb.Predictor(vb.Model.read(mb), predict_tags=True), DumpOracle(mb, predict_tags=True), data, True,
              wsconsts=("", "D", "G"))


@pytest.mark.parametrize("cw,tw,maxdict,tags", [(3, 3, 5, 3), (1, 5, 3, 2), (2, 2, 2, 0), (4, 4, 6, 4)])
def test_random_models(cw, tw, maxdict, tags):
    rng = np.random.default_rng(7000 + 100 * cw + 10 * tw + tags)
    model, alpha = _random_model(rng, cw, tw, maxdict=maxdict, tags=tags)
    mb = encode_model(model)
    data = _random_lines(rng, 400, alpha + "ＡＢａｂ１２ !?", 30)
    check(vb.Predictor(vb.Model.read(mb), predict_tags=tags > 0), DumpOracle(mb, predict_tags=tags > 0), data, tags > 0,
          wsconsts=("", "D", "G"))


def test_wrapping_scores():
    """Weights whose sums pass INT32_MAX and INT32_MIN: the printed scores wrap as the reference's i32 adds do."""
    big = 2 ** 31 - 1
    model = dict(char_ngrams=[("ab", [big, big, big]), ("b", [big, -big, big, 1])], type_ngrams=[(b"\x02", [big, 1])],
                 dict=[("ab", [-big, -big, -big], "")], bias=-2 ** 31, char_window=2, type_window=1, tag_models=[])
    mb = encode_model(model)
    p, d = vb.Predictor(vb.Model.read(mb)), DumpOracle(mb)
    data = b"ab\nbab\naabb\nabab ab\nb\n"
    check(p, d, data, False, modes=[(True, False)])
    out = stream_out(p, data, no_norm=True, scores=True).decode()
    assert any(int(x.split(" ")[-1]) < -2 ** 30 for x in out.split("\n") if ":" in x)


def test_long_tags_and_rules():
    tags = ["x" * 300, "名詞/固有 名詞\\", "y"]
    model = dict(char_ngrams=[("ab", [3, -4, 5, 1]), ("人", [1, 2])], type_ngrams=[], dict=[("地球", [3, -3, 3], "")],
                 bias=1, char_window=2, type_window=0,
                 tag_models=[dict(token="人", tags=[tags, ["a"], ["p", "q"]], char_ngrams=[("人", [(0, [5, -5, 7, 1, 2])])],
                                  type_ngrams=[], bias=[1, 2, 3, 4, 5]),
                             dict(token="地球", tags=[["b", "c"]], char_ngrams=[], type_ngrams=[], bias=[7, 8])])
    mb = encode_model(model)
    p, d, o = vb.Predictor(vb.Model.read(mb), predict_tags=True), DumpOracle(mb, predict_tags=True), OraclePredictor(mb, predict_tags=True)
    data = "人\n地球人ab\n\nab人地球\n人人人\n".encode()
    check(p, d, data, True)
    rules = {"ａｂ": ["R1", "R2", "R3"], "ab": ["S"], "人": [None, None, "Z"], "地球": [None, "T"]}
    check(p, d, data, True, rules=(vb.PatternMatchTagger(p, rules), rules), o=o)


def test_tags_holding_newlines():
    """A tag string may hold a '\n' (only ' ', '\\' and '/' are escaped), in the model or in a rule: the token lines are
    placed by their computed sizes, not found by their '\n's, so the lines after such a tag stay where they belong."""
    model = dict(kat.PREDICTOR_TEST_MODEL)
    model["tag_models"] = [dict(kat.PREDICTOR_TEST_MODEL["tag_models"][0], tags=[["名\n詞", "接尾辞"], ["ジ\nン", "\n"]])] + \
        list(kat.PREDICTOR_TEST_MODEL["tag_models"][1:])
    mb = encode_model(model)
    data = "この人は地球人だ\n人\n\n人は\nこの\n".encode() * 50
    check(vb.Predictor(vb.Model.read(mb), predict_tags=True), DumpOracle(mb, predict_tags=True), data, True)
    # a rule's tag: "こ" has no tag model, the rule fills its first slot (worked out by hand; scores as in
    # test_score_dump_cpu.test_no_norm_glue_and_deviation_1)
    p = vb.Predictor(vb.Model.read(encode_model(kat.PREDICTOR_TEST_MODEL)), predict_tags=True)
    rules = vb.PatternMatchTagger(p, {"こ": ["x\ny"]})
    one = ("こ/x\ny の0:この 5\n\n\n" "こ\nの\n\n", "人/接尾辞/ヒト\n\n" "人\t名詞:40,接尾辞:41\tジン:42,ヒト:43\n\n")
    for no_norm in (True, False):
        got = stream_out(p, "この\n人\n".encode() * 30, no_norm=no_norm, predict_tags=True, tag_rules=rules, scores=True,
                         tag_scores=True).decode()
        want = one if no_norm else ("こ/x\ny の\n0:この 5\n\n" "こ\nの\n\n", one[1])
        assert got == "".join(want) * 30


def test_chunk_of_many_lines():
    """One chunk of 300 000 short lines: the size scan carries its prefix over more than 1024 blocks of 256 lines."""
    mb = read("model.bin")
    rng = np.random.default_rng(5)
    alpha = list("まぁ社長は火星猫だＡ1 ")
    data = "".join("".join(rng.choice(alpha, size=int(rng.integers(1, 5)))) + "\n" for _ in range(300_000)).encode()
    p, d = vb.Predictor(vb.Model.read(mb), predict_tags=True), DumpOracle(mb, predict_tags=True)
    os.environ["VPT_CHUNK_BYTES"] = str(256 << 20)
    try:
        for no_norm in (False, True):
            got = stream_out(p, data, no_norm=no_norm, predict_tags=True, scores=True, tag_scores=True)
            assert got == d.dump_lines(data, no_norm=no_norm, scores=True, tag_scores=True)
    finally:
        del os.environ["VPT_CHUNK_BYTES"]


def test_overrun_tokens_print_bare():
    """Deviation 3: "a" lists 10 candidates against a vector of 8 scores; it prints its surface alone, "b" its pairs."""
    p = vb.Predictor(vb.Model.read(encode_model(OVERRUN_MODEL)), predict_tags=True)
    out = stream_out(p, b"a\nb\nab\n", no_norm=True, predict_tags=True, tag_scores=True).decode()
    blocks = out.split("\n")
    assert "a" in blocks and not any(b.startswith("a\t") for b in blocks)
    assert any(b.startswith("b\tx:") for b in blocks)


@pytest.mark.parametrize("chunk", ["64", "1000", "65536", "1048576"])
def test_chunk_sizes_and_splits(chunk, monkeypatch):
    monkeypatch.setenv("VPT_CHUNK_BYTES", chunk)
    mb = encode_model(kat.PREDICTOR_TEST_MODEL)
    p, d = vb.Predictor(vb.Model.read(mb), predict_tags=True), DumpOracle(mb, predict_tags=True)
    rng = np.random.default_rng(int(chunk))
    data = _random_lines(rng, 300, "この人は地球人だＡａ1 ", 40)
    kw = dict(predict_tags=True, scores=True, tag_scores=True)
    for no_norm in (False, True):
        want = d.dump_lines(data, no_norm=no_norm, scores=True, tag_scores=True)
        assert stream_out(p, data, no_norm=no_norm, **kw) == want
        assert stream_out(p, data, pieces=[len(data) // 3] * 2, flush_at=0, no_norm=no_norm, **kw) == want
    short = "この人\n\n人\nは地球人だ\n".encode()
    want = d.dump_lines(short, scores=True, tag_scores=True)
    for k in range(len(short) + 1):
        assert stream_out(p, short, pieces=[k], flush_at=0, **kw) == want


def test_flag_errors():
    mb = encode_model(kat.PREDICTOR_TEST_MODEL)
    L = vb.lib()
    no_tags = vb.Predictor(vb.Model.read(mb))
    with pytest.raises(vb.VaporettoError, match="needs predict_tags"):
        no_tags.line_stream(tag_scores=True)
    model = dict(kat.PREDICTOR_TEST_MODEL, tag_models=[])
    slotless = vb.Predictor(vb.Model.read(encode_model(model)), predict_tags=True)
    with pytest.raises(vb.VaporettoError, match="tag slots"):
        slotless.line_stream(predict_tags=True, tag_scores=True)
    p = vb.Predictor(vb.Model.read(mb), predict_tags=True)
    h = C.c_void_p()
    sink = vb.STREAM_WRITE_FN(lambda ctx, data, n: 0)
    assert L.vpt_line_stream_new_scores(p._h, None, 0, 0, 1, 4, C.cast(sink, C.c_void_p), None, C.byref(h)) == 2
    assert L.vpt_line_stream_new_scores(p._h, None, 0, 1, 1, 1, C.cast(sink, C.c_void_p), None, C.byref(h)) == 2
    assert L.vpt_line_stream_new_scores(p._h, None, 0, 0, 1, 1, None, None, C.byref(h)) == 2
    with pytest.raises(vb.VaporettoError):
        p.line_stream(kind="evaluate", scores=True)
    # dumps == 0 is the stream without dumps
    data = "この人は地球人だ\n".encode()
    assert stream_out(p, data, predict_tags=True) == bytes(p.tokenize_lines(data, predict_tags=True)[0])


def test_bounded_memory():
    """About 1 M config-2-shaped lines with both dumps, one ~16 MiB block fed 16 times into a sink that only counts:
    the peak resident memory grows by less than 256 MiB between 2 and 8 blocks, and the output is 8 times the block's."""
    mb = synth.gen_model_bccwj_shaped(n_patterns=30_000, sample_sentences=50_000)
    p = vb.Predictor(vb.Model.read(mb))
    text, offs, _ = synth.gen_text(150_000, 40, seed=synth.TEXT_SEED + 52)
    block = b"\n".join(text[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)) + b"\n"
    block = block[: block.rindex(b"\n", 0, 16 << 20) + 1]
    one = len(stream_out(p, block, scores=True))
    total = [0]

    @vb.STREAM_WRITE_FN
    def sink(ctx, data, n):
        total[0] += n
        return 0

    L = vb.lib()
    h = C.c_void_p()
    assert L.vpt_line_stream_new_scores(p._h, None, 0, 0, 0, 1, C.cast(sink, C.c_void_p), None, C.byref(h)) == 0
    try:
        a = np.frombuffer(block, np.uint8)
        for i in range(8):
            assert L.vpt_line_stream_feed(h, a.ctypes.data, a.size) == 0
            if i == 1:
                hwm0 = vm_hwm()
        n = C.c_uint64()
        assert L.vpt_line_stream_finish(h, C.byref(n), None) == 0
        hwm1 = vm_hwm()
    finally:
        L.vpt_line_stream_free(h)
    assert total[0] == 8 * one
    assert hwm1 - hwm0 < 256 << 20


def test_cli_end_to_end():
    cli = os.path.join(ROOT, "tools", "predict_cli.py")
    model = os.path.join(ROOT, "tests", "golden", "model.bin")
    mb = read("model.bin")
    d = DumpOracle(mb)
    text = "まぁ社長は火星猫だ\r\n\nまぁ良いだろう\nVaporetto 1.5\n".encode()
    for args, kw in ((["--scores"], dict(scores=True)), (["--scores", "--no-norm", "--wsconst", "D"], dict(scores=True, no_norm=True, wsconst="D"))):
        out = subprocess.run([sys.executable, cli, "--model", model] + args, input=text, capture_output=True)
        assert out.returncode == 0, out.stderr.decode()
        assert out.stdout == d.dump_lines(text, **kw)
    out = subprocess.run([sys.executable, cli, "--model", model, "--tag-scores"], input=text, capture_output=True)
    assert out.returncode != 0 and b"--tag-scores needs --predict-tags" in out.stderr
