"""The CPU oracle of vpt_predict_tags_batch_dev (vpt_testlib/tags_given_oracle.py): the reference's predict_tags on
boundaries the caller gives.  On the predicted boundaries it is OraclePredictor.predict_tags; on given ones it agrees
with the library's host path (vpt_fill_tags on the same boundaries and pattern-id states), with the reference's known
answer (predictor.rs:863-903) and with the hand-derived tags of the tag_edges model."""
import numpy as np
import pytest

import vaporetto_b200 as vb
from golden import reference_kat as kat
from test_gpu_parity import _random_model, read
from vpt_testlib import tag_edges as te
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.oracle import OraclePredictor
from vpt_testlib.tags_given_oracle import TagsGivenOracle, bound_offsets, char_offsets


def batch(sents):
    enc = [s.encode() if isinstance(s, str) else s for s in sents]
    offs = np.zeros(len(enc) + 1, np.uint64)
    np.cumsum([len(e) for e in enc], out=offs[1:])
    return np.frombuffer(b"".join(enc), np.uint8), offs


def token_bounds(tokens):
    """0 / 1 per pair of adjacent characters: a boundary after every token but the last."""
    out = []
    for t in tokens:
        out += [0] * (len(t) - 1) + [1]
    return out[:-1]


def host_tags(p, text: str, bounds, char_states, type_states):
    """The library's host path: a Sentence with the given boundaries and pattern-id states, then fill_tags
    (vpt_fill_tags).  -> (tag_token [chars], tag_cand [chars, n_tags])."""
    s = vb.Sentence.from_raw(text)
    s.boundaries_mut()[:] = np.asarray(bounds, np.uint8)
    s._char_states = np.ascontiguousarray(char_states, np.uint32)
    s._type_states = np.ascontiguousarray(type_states, np.uint32)
    s._predictor = p
    s.fill_tags()
    return s._tag_token, s._tag_cand.reshape(-1, max(p.n_tags, 1))[:, : p.n_tags]


def given(g, sents, bounds_per_sentence):
    """The oracle harness on one boundary list per sentence (None: the predicted ones) -> per sentence (tok, cand)."""
    text, offs = batch(sents)
    coff = char_offsets(text, offs)
    boff = bound_offsets(coff)
    bd = None
    if bounds_per_sentence is not None:
        bd = np.zeros(max(int(boff[-1]), 1), np.uint8)
        for i, b in enumerate(bounds_per_sentence):
            bd[boff[i]:boff[i + 1]] = b
    tok, cand = g.tags(text, offs, boff, bd, coff)
    return [(tok[coff[i]:coff[i + 1]], cand[coff[i]:coff[i + 1]]) for i in range(len(sents))]


def check_sentences(mb, sents, bounds_per_sentence=None):
    """Harness == OraclePredictor.predict_tags on the predicted boundaries (bounds_per_sentence None), and == the host
    path on whatever boundaries it got: ids through the host path (the oracle may number repeated tokens otherwise),
    known-ness and candidates through both."""
    g, o = TagsGivenOracle(mb), OraclePredictor(mb, predict_tags=True)
    hp = vb.Predictor(vb.Model.read(mb), predict_tags=True, device=-1)  # host-only handle: vpt_fill_tags
    res = given(g, sents, bounds_per_sentence)
    for i, s in enumerate(sents):
        tok, cand = res[i]
        _, bd, cs, ts = o.predict(s, states=True)
        b = bd if bounds_per_sentence is None else bounds_per_sentence[i]
        if bounds_per_sentence is None:
            ott, oti = o.predict_tags(s)
            assert tok.tolist() == ott.tolist() and cand.tolist() == oti.tolist(), (i, s)
        htt, htc = host_tags(hp, s, b, cs, ts)
        assert (tok >= 0).tolist() == (htt >= 0).tolist(), (i, s)
        assert cand.tolist() == htc.tolist(), (i, s)
    return res


def test_predicted_boundaries_equal_predict_tags():
    mb = encode_model(kat.PREDICTOR_TEST_MODEL)
    check_sentences(mb, ["この人は地球人だ", "地球人", "この人", "人"])
    check_sentences(read("model.bin"),["まぁ社長は火星猫だ", "まぁ良いだろう", "火星", "社長は社長だ" * 30])


@pytest.mark.parametrize("cw,tw", [(3, 3), (1, 5), (2, 2)])
def test_random_tag_models(cw, tw):
    """Predicted, all-1, all-0 and random boundaries on the random tag models of test_gpu_tags, and sentences tiled
    from the models' own tokens with the tiling as boundaries."""
    rng = np.random.default_rng(9000 + 10 * cw + tw)
    model, alpha = _random_model(rng, cw, tw, maxdict=5, tags=4)
    mb = encode_model(model)
    sents = ["".join(rng.choice(list(alpha), size=int(rng.integers(1, 60)))) for _ in range(60)]
    check_sentences(mb, sents)
    n = [len(s) for s in sents]
    check_sentences(mb, sents, [[1] * (k - 1) for k in n])
    check_sentences(mb, sents, [[0] * (k - 1) for k in n])
    check_sentences(mb, sents, [rng.integers(0, 2, size=k - 1).tolist() for k in n])
    toks = [t["token"] for t in model["tag_models"]]
    tiles = [[toks[int(j)] for j in rng.integers(len(toks), size=int(rng.integers(1, 12)))] for _ in range(40)]
    res = check_sentences(mb, ["".join(t) for t in tiles], [token_bounds(t) for t in tiles])
    # every token of a tiling is known: its last character carries a token id
    for t, (tok, _) in zip(tiles, res):
        ends = np.cumsum([len(x) for x in t]) - 1
        assert (tok[ends] >= 0).all()


def test_reference_known_answer():
    """predictor.rs:863-903: the tags of 「この人は地球人だ」 on its boundaries given explicitly, read through the host
    predictor's tag strings; and the same sentence cut into characters."""
    case = kat.PREDICT_BOUNDARIES
    mb = encode_model(case["model"])
    g = TagsGivenOracle(mb)
    hp = vb.Predictor(vb.Model.read(mb), predict_tags=True, device=-1)
    text = case["text"]
    (tok, cand), = given(g, [text], [case["boundaries"]])
    _, _, cs, ts = OraclePredictor(mb, predict_tags=True).predict(text, states=True)
    htt, htc = host_tags(hp, text, case["boundaries"], cs, ts)
    assert cand.tolist() == htc.tolist() and (tok >= 0).tolist() == (htt >= 0).tolist()
    tags = [None if htt[i] < 0 or cand[i, k] < 0 else hp.tag_string(int(htt[i]), k, int(cand[i, k]))
            for i in range(len(text)) for k in range(g.n_tags)]
    assert tags == case["tags"]
    check_sentences(mb, [text], [[1] * (len(text) - 1)])


def test_tag_edges_tokens_as_boundaries():
    """Every tag_edges case with its own token list as the boundaries, on a copy of the edge model whose scoring
    predicts a boundary everywhere (bias +1): the harness gives the hand-derived candidates
    (tag_edges.expected_sentence_cands) and the host path's."""
    cases = te.edge_cases()
    mb = encode_model(dict(te.model(cases), bias=1))
    known = set(te.known_tokens(cases))
    o = OraclePredictor(mb, predict_tags=True)
    assert o.predict(cases[0].sentence)[1].tolist() == [1] * (len(cases[0].sentence) - 1)
    res = check_sentences(mb, [c.sentence for c in cases], [token_bounds(c.tokens) for c in cases])
    for c, (tok, cand) in zip(cases, res):
        want = te.expected_sentence_cands(c.tokens, known)
        assert cand.tolist() == want, (c.kind, c.w, c.align, c.known)
        assert (tok >= 0).tolist() == [w[0] >= 0 for w in want]


def test_rejected_sentences_get_minus_one():
    """Empty, NUL and invalid UTF-8 sentences: -1 over the characters the caller counts for them."""
    mb = encode_model(kat.PREDICTOR_TEST_MODEL)
    g = TagsGivenOracle(mb)
    sents = [b"", "a\0b".encode(), b"\xe3\x81", "この人は地球人だ".encode()]
    text, offs = batch(sents)
    coff = np.array([0, 0, 3, 4, 12], np.uint64)   # (a caller may count characters of a rejected sentence)
    boff = np.array([0, 0, 2, 3, 10], np.uint64)
    bd = np.ones(10, np.uint8)
    tok, cand = g.tags(text, offs, boff, bd, coff)
    assert (tok[:4] == -1).all() and (cand[:4] == -1).all()
    assert (tok[4:] >= 0).any()
