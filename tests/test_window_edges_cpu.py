"""The window-edge cases of vpt_testlib.window_edges, checked without a GPU: every case lands on the edge it names in the
layout the device sees, every case is live (with the CPU oracles alone, its answer changes when the feature at the edge
is removed), and every (kernel, edge, b0) the edge suite must reach has a case."""
import ast
import itertools
import re

import pytest

from vpt_testlib import eval_oracle as eo
from vpt_testlib import window_edges as we
from vpt_testlib.oracle import OraclePredictor, char_types
from vpt_testlib.spans_oracle import SpansOracle
from vpt_testlib.tokenize_doc_oracle import TokenizeDocOracle


@pytest.fixture(scope="module")
def ora():
    return {"all": OraclePredictor(we.model_all()), "tag": OraclePredictor(we.model_tag(), predict_tags=True)}


def _bounds(ora, line: bytes, **kw):
    out, n = ora.tokenize_lines(line + b"\n", **kw)
    assert n == 1
    return eo.parse_tokenized(out[:-1].decode())[1]


def _swap(b: bytes, at: int, to: bytes = b"q") -> bytes:
    return b[:at] + to + b[at + 1:]


def test_cases_land_on_their_edges():
    cases = we.all_cases()
    for c in cases:
        # the feature's bytes are in the payload where the case says, and that byte lands on the named coordinate
        assert c.payload[c.at - c.k:c.at - c.k + len(c.feature)] == c.feature and c.b0 + c.at == c.coord, c.key
        m = re.search(r"@(\d+)(?:\|(\d+))?", c.edge)
        if m:
            assert c.coord == int(m.group(2) or m.group(1)), c.key
        if c.edge.startswith("esc"):
            assert c.feature == ast.literal_eval(c.edge[3:c.edge.index("@")]).encode(), c.key
        loc = we.locate(c.coord)
        if c.edge.endswith(("@127", "@128")) or "127|128" in c.edge:
            assert loc["window"] == (c.coord >= 128) and loc["lane"] == (31 if c.coord == 127 else 0), c.key
    # the layouts put every case at its b0 (line_buffer and doc_batch check it and raise otherwise)
    we.line_buffer(we.line_cases())
    we.line_buffer(we.gold_cases())
    text, offs, idx = we.doc_batch(we.doc_cases() + we.span_cases())
    for c, d in zip(we.doc_cases() + we.span_cases(), idx):
        assert offs[d] % 4 == c.b0 and text[offs[d]:offs[d + 1]] == c.payload
    # the named edges
    for c in cases:
        if c.edge.startswith("b1="):
            b1 = int(c.edge[3:].split("/")[0])
            assert c.b1 == b1 and we.streaming(b1) == (b1 > 128)
        if c.edge.startswith("char"):
            w, x = int(c.edge[4]), int(c.edge.split("@")[1])
            assert x < 128 <= x + w - 1 and len(c.payload[c.at:].decode("utf-8", "ignore")[0].encode()) == w
        if c.kernel == "wsconst":
            cls = c.info["cls"]
            chars = c.payload.decode()
            k = c.info["first"]
            ty = char_types(chars)
            assert ty[k] == ty[k + 1] == "DRHTKO".index(cls) + 1
            a, b = (c.b0 + len(chars[:i].encode()) for i in (k, k + 1))  # the coordinates of characters k and k + 1
            assert we.locate(a)["window"] == 0 and we.locate(b)["window"] == (0 if c.edge == "cont-only" else 1)
            if c.edge == "cont-only":
                assert b == 127 and c.b1 == 131
        if c.kernel == "grapheme":
            k = c.info["boundary"]
            chars = c.payload.decode()
            first = c.b0 + len(chars[:k + 1].encode())
            assert first == 128 or (c.edge.startswith("ri-even") and first == 132)
    # line paths: the test buffers are one chunk of the line pipeline
    assert we.line_chunk_count(2 << 20) == 1 and we.line_chunk_count((2 << 20) + 1) == 2


def test_a_case_off_its_edge_raises(monkeypatch):
    """A filler one byte too long, a feature string edited, or a batch that the span pipeline would cut: each raises."""
    with pytest.raises(ValueError):
        we._case("tok", "esc' '@128", 1, we.fill(128 - 1 + 1, we.TOK_ALPHA), " ", "tail", 128)
    with pytest.raises(ValueError):
        we.Case("tok", "esc' '@128", 1, b"a" * 127 + b"q" + b"tail", 127, 128, b" ")
    we.doc_batch(we.span_cases())
    monkeypatch.setenv("VPT_CHUNK_SENTENCES", "1024")
    monkeypatch.setenv("VPT_CHUNK_BYTES", "64")
    assert len(we.span_chunks([0, 10, 20])) == 2 and we.chunk_sentences() == 1024
    with pytest.raises(ValueError):
        we.doc_batch(we.span_cases())
    we.doc_batch(we.tok_cases())  # (no bound_offsets alignment needed: any chunking keeps offsets mod 16)


def test_tok_cases_are_live(ora):
    for c in we.tok_cases():
        if c.kernel == "tok":
            line = c.payload
            # the feature (an escape, a multi-byte character, the last byte) replaced by one plain byte
            feat = line[:c.at - c.k] + b"q" + line[c.at - c.k + len(c.feature):]
            got = ora["all"].tokenize_lines(line + c.end)[0]
            assert got != ora["all"].tokenize_lines(feat + c.end)[0], c.key
            # an inserted byte on either side of the window edge: dropping `extra` shifts what follows
            assert len(got) > len(line) + 1
        else:
            got = ora["tag"].tokenize_lines(c.payload + c.end, predict_tags=True)[0]
            head = c.payload[:c.at + 1].decode()
            # the tokens up to the feature, each written with its suffix, then the ' ' in front of byte 128
            want = " ".join([we.TERM + we.TAG_SUFFIX] * head.count(we.TERM))
            assert got.decode().startswith(want + " "), c.key
            assert got != ora["tag"].tokenize_lines(_swap(c.payload, c.at) + c.end, predict_tags=True)[0]


@pytest.mark.parametrize("no_norm", [False, True])
def test_wsconst_cases_are_live(ora, no_norm):
    for c in we.wsconst_cases():
        k = c.info["first"]
        plain = _bounds(ora["all"], c.payload, no_norm=no_norm)
        filt = _bounds(ora["all"], c.payload, no_norm=no_norm, wsconst=c.info["cls"])
        assert plain[k] == 1 and filt[k] == 0, c.key
        assert [i for i in range(len(plain)) if plain[i] != filt[i]].count(k) == 1


def test_grapheme_cases_are_live(ora):
    docs = TokenizeDocOracle(we.model_all())
    for c in we.grapheme_cases(docs=True):
        k = c.info["boundary"]
        if c.edge.startswith("crlf"):
            text, offs, idx = we.doc_batch([c])
            out = [docs.tokenize_docs(text, offs, wsconst=ws)[0][idx[0]] for ws in ("", "G")]
            plain, filt = (eo.parse_tokenized(o.decode().replace("\r", "R").replace("\n", "N"))[1] for o in out)
        else:
            plain = _bounds(ora["all"], c.payload)
            filt = _bounds(ora["all"], c.payload, wsconst="G")
        assert plain[k] == 1 and filt[k] == 0, c.key


def test_span_cases_are_live():
    so = {"none": SpansOracle(we.model_none()), "tag": SpansOracle(we.model_tag())}
    for c in we.span_cases():
        text, offs, idx = we.doc_batch([c])
        d = idx[0]
        if c.edge.startswith("lb"):
            ends = so["none"].token_spans(text, offs)
            first = int(sum(ends["n_tokens"][:d]))
            e = ends["token_ends"][first:first + ends["n_tokens"][d]].tolist()
            assert c.at in e and c.at + 1 in e, c.key  # a boundary on both sides of the line break
        else:
            ends = so["tag"].token_spans(text, offs)
            first = int(sum(ends["n_tokens"][:d]))
            e = ends["token_ends"][first:first + ends["n_tokens"][d]].tolist()
            if c.edge.startswith("tok"):
                assert c.at in e, c.key  # a token starts on the edge coordinate
            else:
                nb = c.info["nb"]
                assert ends["n_tokens"][d] == c.payload.count(b"#") + 1 and e[-2] == nb, c.key
        o = so["none"] if c.edge.startswith("lb") else so["tag"]
        feat = c.at - 1 if c.edge.startswith("tok") else c.at  # (tok: the '#' that ends the token before the edge)
        assert c.edge.startswith("lb") or c.payload[feat:feat + 1] == we.TERM.encode()
        t2 = _swap(text, offs[d] + feat)
        assert o.token_spans(t2, offs)["token_ends"].tolist() != o.token_spans(text, offs)["token_ends"].tolist(), c.key


def test_gold_cases_are_live():
    for c in we.gold_cases():
        line = c.payload.decode()
        want = eo.parse_tokenized(line)
        try:
            other = eo.parse_tokenized(_swap(c.payload, c.at).decode() if c.payload[c.at] < 0x80
                                       else c.payload[:c.at].decode() + "q" + c.payload[c.at:].decode()[1:])
        except eo.GoldError:
            other = None
        assert other != want, c.key
        if c.edge.startswith("bs"):
            L = c.info["L"]
            assert c.payload[c.at - L + 1:c.at + 1] == b"\\" * L and c.payload[c.at - L:c.at - L + 1] != b"\\"
        if c.edge.startswith("tagpos"):
            assert c.payload[c.at:c.at + 1] == b"/" and c.payload[c.at - 1:c.at] == we.TERM.encode()


def test_gold_error_cases_are_live(ora):
    msgs = {"DoubleWs": "consecutive whitespaces", "Slash": "a slash must follow", "NUL": "must not contain NULL",
            "EndWs": "must not end with a whitespace", "utf8": "valid UTF-8"}
    for c in we.gold_error_cases():
        data, offs = we.line_buffer([c], lead=b"ab c\n")
        with pytest.raises(eo.GoldError) as e:
            eo.evaluate_lines(ora["all"], data)
        kind = c.info["kind"]
        assert msgs["utf8" if kind.startswith("utf8") else kind] in e.value.msg and e.value.line == data.count(b"\n") - 1
        # the same buffer with the feature byte (UTF-8: the bad sequence) replaced by a plain one has no error
        at = offs[0] + c.at
        if kind.startswith("utf8"):
            at, n = offs[0] + c.at - c.k, len(c.feature)
            eo.evaluate_lines(ora["all"], data[:at] + b"q" + data[at + n:])
        else:
            eo.evaluate_lines(ora["all"], _swap(data, at))
    for name, lines, where in we.gold_error_multi():
        with pytest.raises(eo.GoldError) as e:
            eo.evaluate_lines(ora["all"], b"\n".join(lines) + b"\n")
        assert e.value.line == where, name


def test_eval_cases_are_live(ora):
    for name, gold, alt in we.eval_cases():
        nb = len(eo.parse_tokenized(gold)[0]) - 1
        assert nb == int(name.split("/")[0][3:])
        if alt is None:
            continue
        tags = "tags" in name
        _, a = eo.evaluate_lines(ora["tag"], gold.encode() + b"\n", predict_tags=tags)
        _, b = eo.evaluate_lines(ora["tag"], alt.encode() + b"\n", predict_tags=tags)
        assert a[0][6] != b[0][6], name  # n_cor


# ---- coverage: the spec's (kernel, edge, b0) list, written out apart from the builders --------------------------------

def required():
    req = set()
    for b0 in range(4):
        for x, e in itertools.product((3, 4, 63, 64, 126, 127, 128, 129, 255, 256), " /\\"):
            req.add(("tok", f"esc{e!r}@{x}", b0))
        for w in (2, 3, 4):
            for j in range(1, w):
                req.add(("tok", f"char{w}@{128 - j}", b0))
        for b1 in (127, 128, 129, 255, 256, 257):
            req |= {("tok", f"b1={b1}", b0), ("tok", f"b1={b1}/crlf", b0)}
        req |= {("tags", "suffix@127", b0), ("tags", "suffix@128", b0)}
        for cls in "DRHTKO":
            req.add(("wsconst", f"pair{cls}@127|128", b0))
        req.add(("wsconst", "cont-only", b0))
        for g in ("extend", "zwj", "hangul", "gb9c", "ri-odd", "ri-even", "prepend0600", "prepend110bd", "crlf"):
            req.add(("grapheme", f"{g}@127|128", b0))
        for x in (126, 127, 128, 129):
            req |= {("spans", f"lb'\\n'@{x}", b0), ("spans", f"lb'\\r'@{x}", b0)}
        req |= {("spans", "tok@127", b0), ("spans", "tok@128", b0)}
        for nb in (127, 128, 129):
            req.add(("spans", f"run{nb}", b0))  # (b0 here: bound_offsets % 4)
        for L in range(1, 10):
            for x in list(range(124, 133)) + [x for x in range(9) if x - L + 1 >= b0]:
                for e in (" ", "/", "\\", "k"):
                    req.add(("gold", f"bs{L}@{x}/{e!r}", b0))
        req |= {("gold", "field@120..135", b0), ("gold", "fields@124..133", b0), ("gold", "tagpos@128", b0)}
        for w in (2, 3, 4):
            for j in range(1, w):
                req.add(("gold", f"char{w}@{128 - j}", b0))
        for x in (127, 128):
            for k in ("DoubleWs", "Slash", "NUL", "EndWs"):
                req.add(("gold_err", f"{k}@{x}", b0))
        for k in ("missing", "surrogate", "overlong3", "overlong2"):
            req.add(("gold_err", f"utf8-{k}@127", b0))
        req.add(("gold_err", "utf8-stray@128", b0))
    return req


def test_every_required_edge_has_a_case():
    have = {c.key for c in we.all_cases()}
    missing = sorted(required() - have)
    assert not missing, missing[:20]
    names = [n for n, _, _ in we.eval_cases()]
    for nb in (31, 32, 33, 63, 64, 65):
        assert f"nb={nb}" in names and f"nb={nb}/dis31-to-end" in names
        if nb >= 33:
            for k in ("dis31-shared32", "shared31-dis32", "tags-right", "tags-wrong"):
                assert f"nb={nb}/{k}" in names
    assert {n for n, _, _ in we.gold_error_multi()} == {"window2-then-3", "window3-before-line-start"}
