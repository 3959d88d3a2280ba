"""Every scoring-kernel variant with the full-width pre-filter on (no_norm=False, the default of every tokenizing entry
point), on models whose patterns are filter images and text that spells them through their sources
(vpt_testlib/norm_variants.py; test_norm_variants_cpu.py checks that the filter changes what each model matches).
Bit-exact against the CPU oracles: token spans, tokenized text with tags, i32 boundary scores through the line stream,
known tag tokens at the byte-length limit of the token table, and the wsconst post-filters on filtered types."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import vaporetto_b200 as vb
from vpt_testlib import norm_variants as nv
from vpt_testlib import tile_edges as te
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.dump_oracle import DumpOracle
from vpt_testlib.oracle import OraclePredictor
from vpt_testlib.spans_oracle import SpansOracle
from vpt_testlib.tokenize_doc_oracle import TokenizeDocOracle
from test_gpu_score_dump import stream_out

pytestmark = pytest.mark.gpu

RECIPES = nv.recipes()
SCORE_KERNELS = nv.SCORE_KERNELS


def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def device_predictor(budget, args, tags, monkeypatch):
    if budget:
        monkeypatch.setenv("VPT_SEED_BUDGET", budget)   # 16-bit seeds: the seed table stays in global memory
    else:
        monkeypatch.delenv("VPT_SEED_BUDGET", raising=False)
    mb, words = nv.norm_model(*args)
    return mb, words, vb.Predictor(vb.Model.read(mb), predict_tags=tags)


def host_batch(sents):
    enc = [s.encode() for s in sents]
    offs = np.zeros(len(enc) + 1, np.uint64)
    np.cumsum([len(e) for e in enc], out=offs[1:])
    return b"".join(enc), offs


def to_dev(sents):
    text, offs = host_batch(sents)
    return (text, offs, torch.frombuffer(bytearray(text), dtype=torch.uint8).cuda(),
            torch.from_numpy(offs.astype(np.int64)).cuda())


def oracle_parts(fn, sents, parts=8):
    """fn(text, offsets) over `parts` slices of the documents, on as many threads (the oracle calls release the GIL;
    every result of the document oracles is per document)."""
    cut = np.linspace(0, len(sents), parts + 1).astype(int)
    with ThreadPoolExecutor(parts) as ex:
        return list(ex.map(lambda k: fn(*host_batch(sents[cut[k]:cut[k + 1]])), range(parts)))


def check_docs(p, mb, sents, states):
    """One launch over the documents: token spans (plain) or tokenized text with tags (states), filter on."""
    _, _, d_text, d_offs = to_dev(sents)
    if not states:
        r = p.token_spans_device(d_text, d_offs, no_norm=False).to_host()
        o = SpansOracle(mb)
        w = oracle_parts(lambda t, off: o.token_spans(t, off, no_norm=False), sents)
        assert np.array_equal(r.status, np.concatenate([x["status"] for x in w]))
        assert np.array_equal(r.n_tokens, np.concatenate([x["n_tokens"] for x in w]))
        assert np.array_equal(r.token_ends, np.concatenate([x["token_ends"] for x in w]))
        return
    d = p.tokenize_device(d_text, d_offs, no_norm=False, predict_tags=True)
    chars, out_offs, status = d.to_host()
    assert bool(d.complete.item())
    b = chars.tobytes()
    got = [b[out_offs[i]:out_offs[i + 1]] for i in range(len(sents))]
    o = TokenizeDocOracle(mb, predict_tags=True)
    w = oracle_parts(lambda t, off: o.tokenize_docs(t, off, no_norm=False, predict_tags=True), sents)
    assert np.array_equal(status, np.concatenate([x[1] for x in w]))
    want = [doc for x in w for doc in x[0]]
    bad = [i for i in range(len(sents)) if got[i] != want[i]]
    assert not bad, (len(bad), sents[bad[0]], got[bad[0]], want[bad[0]])
    assert any(b"/" in g for g in got)   # tags were written


def check_scores(p, mb, sents, states):
    """The sentences as lines (every fifth ending in '\\r\\n') through the scores line stream, filter on: every i32
    boundary score against the dump oracle; the filter changes the output."""
    data = b"".join(s.encode() + (b"\r\n" if i % 5 == 4 else b"\n") for i, s in enumerate(sents))
    got = stream_out(p, data, no_norm=False, predict_tags=states, scores=True)
    want = DumpOracle(mb, predict_tags=states).dump_lines(data, no_norm=False, scores=True)
    assert got == want
    assert got != stream_out(p, data, no_norm=True, predict_tags=states, scores=True)


@pytest.mark.parametrize("name,budget,args,tags,states,key", RECIPES, ids=[r[0] for r in RECIPES])
def test_norm_variant_at_tile_edges(name, budget, args, tags, states, key, monkeypatch):
    mb, words, p = device_predictor(budget, args, tags, monkeypatch)
    # the device paths ask for pattern-id states exactly when they predict tags
    plan = p.kernel_plan(states)
    assert te.plan_key(plan) == key, plan
    rng = np.random.default_rng(sum(map(ord, name)))
    spelled = [nv.source_spellings(w, rng) for w in words]   # a long pattern is hit only through the filter
    # one launch of at least three rounds of groups over all sub-blocks of the device, edge groups in every round
    subs = plan["sub_blocks"] * n_sm()
    b = te.build(plan, nv.TEXT_ALPHABET, spelled, n_groups=3 * subs + 8, seed=sum(map(ord, name)), tail=63)
    assert (len(b.sents) + te.GROUP - 1) // te.GROUP >= 3 * subs
    check_docs(p, mb, b.sents, states)
    check_scores(p, mb, b.sents[:1200] + b.sents[-63:], states)


@pytest.mark.parametrize("name,args,tags,states,key", SCORE_KERNELS, ids=[r[0] for r in SCORE_KERNELS])
def test_norm_one_warp_kernels(name, args, tags, states, key, monkeypatch):
    mb, words, p = device_predictor(None, args, tags, monkeypatch)
    assert te.plan_key(p.kernel_plan(states)) == key
    sents = nv.text_for(words, 4000, np.random.default_rng(sum(map(ord, name))))
    check_docs(p, mb, sents, states)
    check_scores(p, mb, sents[:1200], states)


# ---- known tag tokens at the byte-length limit of the token table --------------------------------------------------

def test_tag_tokens_at_the_image_byte_limit():
    """A token is looked up by the bytes of its image, and the table holds none longer than its longest known token
    (max_token_bytes): ASCII sources whose image is exactly that long are found, one byte more is not, although the raw
    tokens are a third as long; a known token written in images matches its sources only under the filter."""
    term = "~"                                   # a fixed point: ends every token (char window 1, bias -1)
    longest = "ＡＢＣＤＥ" + "#" * 2 + term        # 18 bytes: max_token_bytes
    short = "ｘ−ｙ" + term                        # matches "x-y~" only through the filter ('-' -> U+2212)
    known = [longest, short, "ａ" + term, "ー" + term]
    model = dict(char_ngrams=[(term, [0, 2])], type_ngrams=[], dict=[], bias=-1, char_window=1, type_window=1,
                 tag_models=[dict(token=t, tags=[["P", "Q", "R"]], char_ngrams=[], type_ngrams=[],
                                  bias=[int(k == i % 3) for k in range(3)]) for i, t in enumerate(known)])
    mb = encode_model(model)
    p, o = vb.Predictor(vb.Model.read(mb), predict_tags=True), OraclePredictor(mb, predict_tags=True)
    at_limit = "ABCDE##" + term                  # 8 bytes raw, image 18
    over = [at_limit[:-1] + "#" + term, "ABCDE" + "é" + "#" + term, "ABCDEF" + term]   # images of 19 bytes
    assert len(nv.normalize(at_limit).encode()) == len(longest.encode()) == 18
    assert all(len(nv.normalize(t).encode()) == 19 and len(t.encode()) < 10 for t in over)
    toks = [at_limit, longest, "x-y" + term, short, "a" + term] + [d + term for d in nv.DASHES] + over
    rng = np.random.default_rng(1)
    lines = ["".join(rng.permutation(toks).tolist()) for _ in range(300)] + toks
    data = "".join(s + ("\r\n" if i % 7 == 3 else "\n") for i, s in enumerate(lines)).encode()
    out = {}
    for no_norm in (False, True):
        got, nl = p.tokenize_lines(data, no_norm=no_norm, predict_tags=True)
        want, wl = o.tokenize_lines(data, no_norm=no_norm, predict_tags=True)
        assert nl == wl == len(lines) and got.tobytes() == want, no_norm
        out[no_norm] = got.tobytes().decode().split("\n")[-len(toks) - 1:-1]   # the lines of one token each
    assert [("/" in x) for x in out[False]] == [True] * (5 + len(nv.DASHES)) + [False] * len(over), out[False]
    assert [("/" in x) for x in out[True]] == [False, True, False, True] + [False] * (1 + len(nv.DASHES) + len(over))


# ---- the wsconst post-filters on filtered character types ---------------------------------------------------------

# (the wsconst letters are KyTea's: T is katakana, K kanji)
WSCONST_CASES = [
    ("T", ["アイ" + d + "ウエ" + d + "オ" for d in nv.DASHES] + ["カ" + "".join(nv.DASHES) + "キ"]),
    ("D", ["12３4５6", "年12月3日", "0-9,1.5"]),
    ("R", ["abＣdE", "xY人Zz", "a.b-c"]),
    ("DG", ["1́2́３", "ab́c12", "é1é2"]),
]


@pytest.mark.parametrize("wsconst,cases", WSCONST_CASES, ids=[c[0] for c in WSCONST_CASES])
def test_wsconst_on_filtered_types(wsconst, cases):
    mb, _ = nv.norm_model(3, 3, (1, 2, 3), (), 0)
    p, o, so_ = vb.Predictor(vb.Model.read(mb)), OraclePredictor(mb), SpansOracle(mb)
    rng = np.random.default_rng(len(wsconst))
    alpha = list(nv.TEXT_ALPHABET)
    docs = cases + ["".join(rng.choice(alpha, size=5).tolist()) + c + "".join(rng.choice(alpha, size=3).tolist())
                    for c in cases for _ in range(40)]
    data = "".join(d + "\n" for d in docs).encode()
    text, offs, _, _ = to_dev(docs)
    outs = {}
    for no_norm in (False, True):
        got, nl = p.tokenize_lines(data, no_norm=no_norm, wsconst=wsconst)
        want, wl = o.tokenize_lines(data, no_norm=no_norm, wsconst=wsconst)
        assert nl == wl == len(docs) and got.tobytes() == want, no_norm
        outs[no_norm] = got.tobytes()
        r = p.token_spans(text, offs.astype(np.uint64), no_norm=no_norm, wsconst=wsconst)
        w = so_.token_spans(text, offs.astype(np.uint64), no_norm=no_norm, wsconst=wsconst)
        assert np.array_equal(r.n_tokens, w["n_tokens"]) and np.array_equal(r.token_ends, w["token_ends"]), no_norm
    assert outs[False] != outs[True]
    if wsconst == "T":   # under the filter every dash is Katakana: each case is one token
        assert outs[False].decode().split("\n")[:len(cases)] == cases


def test_every_norm_variant_reached(monkeypatch):
    """The norm recipes reach, on the device, every tile variant the dispatch can launch except the unreachable ones
    (tile_edges.UNREACHABLE), and both one-warp-per-sentence kernels."""
    reached = set()
    for name, budget, args, tags, states, key in RECIPES:
        reached.add(te.plan_key(device_predictor(budget, args, tags, monkeypatch)[2].kernel_plan(states)))
    tiles = set(reached)
    for name, args, tags, states, key in SCORE_KERNELS:
        reached.add(te.plan_key(device_predictor(None, args, tags, monkeypatch)[2].kernel_plan(states)))
    want = (te.all_plan_keys() - set(te.UNREACHABLE)) | {k[-1] for k in SCORE_KERNELS}
    assert reached == want, sorted(want ^ reached)
    assert {k[0] for k in reached - tiles} == {"k_score_general", "k_score_fast"}
    print(f"\nnorm variants reached: {len(tiles)} tile variants of {len(te.all_plan_keys())} (unreachable: "
          f"{len(te.UNREACHABLE)}, {sorted(set(te.UNREACHABLE.values()))}) and {sorted({k[0] for k in reached - tiles})}")
    for k in sorted(reached):
        print("  ", dict(zip(te.PLAN_KEYS, k)))
