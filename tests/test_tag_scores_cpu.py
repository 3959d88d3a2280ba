"""Tag candidate scores on the CPU: the oracle's score path pinned by known answers worked out by hand, the kernels' own
score code (tags_token.hpp, host build) against the oracle over the product's tag tables, and the restatement of
Token::tag_candidates."""
import os

import numpy as np
import pytest

from golden import reference_kat as kat
from vpt_testlib import oracle
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.oracle import OraclePredictor
from vpt_testlib.tag_scores_oracle import TagScoresOracle, emul_lib, first_max, tag_candidates

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")


def _batch(sents):
    enc = [s.encode() if isinstance(s, str) else s for s in sents]
    offs = np.zeros(len(enc) + 1, np.uint64)
    np.cumsum([len(e) for e in enc], out=offs[1:])
    return np.frombuffer(b"".join(enc) or b"\0", np.uint8)[: int(offs[-1])], offs


# "この人は地球人だ" on the reference's tag test model (predictor.rs:863-903), tokens この|人|は|地球|人|だ.  By hand:
#  人 (char 2): bias [40, 41, 42, 43] + type n-gram HKH at rel 1 (の人は) [36, -37, -38, 39]       = [76, 4, 4, 82]
#  地球 (char 5): bias [46, 47] + char n-gram は地球人 at rel 1 (ends at char 6) [-44, 45]         = [2, 92]
#  人 (char 6): bias [40, 41, 42, 43] + char n-gram は地球人 at rel 0 [-32, 33, 34, -35]           = [8, 74, 76, 8]
# (the other tokens have no tag model; no other pattern on the chains carries tag weights).  A bias of up to eight
# weights is a fixed eight-wide vector (WeightVector::from with fix-weight-length, predictor.rs:118-135), so each score
# vector is eight long, zero-padded.
KAT_IDS_KNOWN = [False, True, False, True, True, False]
Z4 = [0, 0, 0, 0]
KAT_SCORES = [76, 4, 4, 82] + Z4 + [2, 92] + Z4 + [0, 0] + [8, 74, 76, 8] + Z4
KAT_TAGS = {"人": [["名詞", "接尾辞"], ["ジン", "ヒト"]], "地球": [["名詞"], ["マンホーム", "チキュー"]]}


def test_known_answers_of_the_reference_test_model():
    o = TagScoresOracle(encode_model(kat.PREDICTOR_TEST_MODEL))
    text, offs = _batch(["この人は地球人だ"])
    ids, sc = o.compact(text, offs)
    assert (ids >= 0).tolist() == KAT_IDS_KNOWN
    assert sc.tolist() == KAT_SCORES
    # their first strict maxima are the reference's expected tags (PREDICT_BOUNDARIES["tags"], per char, n_tags = 2)
    want = kat.PREDICT_BOUNDARIES["tags"]
    vecs = {2: ("人", KAT_SCORES[0:8]), 5: ("地球", KAT_SCORES[8:16]), 6: ("人", KAT_SCORES[16:24])}
    for ch, (tok, v) in vecs.items():
        got, off = [], 0
        for cands in KAT_TAGS[tok]:
            if len(cands) == 1:
                got.append(cands[0])
            else:
                got.append(cands[first_max(v[off:off + len(cands)])])
                off += len(cands)
        assert got == want[2 * ch:2 * ch + 2], (ch, tok)
    # and Token::tag_candidates of them
    assert tag_candidates(KAT_TAGS["人"], KAT_SCORES[0:8]) == [[("名詞", 76), ("接尾辞", 4)], [("ジン", 4), ("ヒト", 82)]]
    assert tag_candidates(KAT_TAGS["地球"], KAT_SCORES[8:16]) == [[("名詞", 0)], [("マンホーム", 2), ("チキュー", 92)]]
    # the spans chain on the same text (no line breaks, nothing to post-filter) gives the same records
    ids2, sc2 = o.spans(text, offs, no_norm=True)
    assert (ids2 >= 0).tolist() == KAT_IDS_KNOWN and sc2.tolist() == KAT_SCORES


def test_tag_candidates_restatement():
    # one-candidate slots give score 0 and consume no score; empty slots give []; scores are read in slot order
    assert tag_candidates([], []) == []
    assert tag_candidates([[]], []) == [[]]
    assert tag_candidates([["a"]], []) == [[("a", 0)]]
    assert tag_candidates([["a", "b"], [], ["c"], ["d", "e", "f"]], [5, -6, 7, 8, 9]) == \
        [[("a", 5), ("b", -6)], [], [("c", 0)], [("d", 7), ("e", 8), ("f", 9)]]
    assert tag_candidates([["a"], ["b", "c"]], [1, 2, 99]) == [[("a", 0)], [("b", 1), ("c", 2)]]
    assert first_max([3, 7, 7, 1]) == 1 and first_max([-2**31, -2**31]) == 0


def _fullwidth(text):
    return "".join(chr(oracle.lib().ora_kytea_fullwidth(ord(c))) for c in text)


def _emul(L, mb, text, norm=False):
    """Records of one sentence by the kernels' score code: boundaries from the oracle, states from the host emulation of
    the scoring kernels, tokens looked up by the image of their original bytes when norm."""
    seen = _fullwidth(text) if norm else text
    _, bd = OraclePredictor(mb).predict(seen)
    sb = seen.encode()
    cs = np.zeros(len(sb) + 1, np.uint32)
    ts = np.zeros(len(sb) + 1, np.uint32)
    sc0 = np.zeros(len(sb) + 1, np.int32)
    info = np.zeros(4, np.int32)
    n = L.emul_predict(mb, len(mb), 1, sb, len(sb), sc0.ctypes.data, cs.ctypes.data, ts.ctypes.data, info.ctypes.data)
    assert n > 0, L.emul_last_error()
    b = text.encode()
    bd = np.ascontiguousarray(np.asarray(bd, np.uint8))
    ids = np.zeros(n, np.int32)
    cap = 64 * n
    out = np.zeros(cap, np.int32)
    uns = np.zeros(1, np.int32)
    import ctypes as C
    tot = C.c_uint64()
    r = L.emul_tag_scores(mb, len(mb), b, len(b), bd.ctypes.data, cs.ctypes.data, ts.ctypes.data, int(norm), ids.ctypes.data,
                          out.ctypes.data, uns.ctypes.data, cap, C.byref(tot))
    assert r >= 0, r
    return ids[:r], out[: tot.value], int(uns[0])


def _check(mb, texts, norm=False):
    L = emul_lib()
    o = TagScoresOracle(mb)
    for text in texts:
        ids, sc, uns = _emul(L, mb, text, norm=norm)
        t, offs = _batch([text])
        oids, osc = o.spans(t, offs, no_norm=not norm) if norm else o.compact(t, offs)
        assert uns == 0
        assert (ids >= 0).tolist() == (oids >= 0).tolist(), text
        assert sc.tolist() == osc.tolist(), text


def test_kernel_score_code_on_reference_models():
    _check(encode_model(kat.PREDICTOR_TEST_MODEL), ["この人は地球人だ", "地球人", "この人", "人"])
    with open(os.path.join(GOLDEN, "model.bin"), "rb") as f:
        _check(f.read(), ["まぁ社長は火星猫だ", "まぁ良いだろう", "火星", "社長は社長だ" * 5])


@pytest.mark.parametrize("cw,tw,maxdict,tags", [(3, 3, 5, 3), (1, 5, 3, 2), (2, 2, 2, 4), (5, 4, 4, 3), (4, 5, 9, 6)])
def test_kernel_score_code_on_random_models(cw, tw, maxdict, tags):
    """Random tag models with windows up to 5 (suffix chains through n-grams and dictionary words): the vectors the
    kernels store equal the oracle's raw scores."""
    from test_gpu_parity import _random_model
    rng = np.random.default_rng(4242 + 1000 * cw + 100 * tw + maxdict + tags)
    for _ in range(3):
        model, alpha = _random_model(rng, cw, tw, maxdict=maxdict, tags=tags)
        mb = encode_model(model)
        _check(mb, ["".join(rng.choice(list(alpha), size=rng.integers(1, 40))) for _ in range(40)])


def test_kernel_score_code_with_the_fullwidth_prefilter():
    """norm = 1: tokens are looked up by their full-width image; the scores are those of the pre-filtered sentence."""
    rng = np.random.default_rng(5)
    alpha = list("あいう人aB1x!?-")
    fw = _fullwidth
    tms = []
    for t in range(6):
        tok = fw("".join(rng.choice(alpha, size=rng.integers(1, 3))))
        cn = [(fw("".join(rng.choice(alpha, size=rng.integers(1, 3)))),
               [(int(rng.integers(0, 4)), rng.integers(-99, 99, size=3).tolist())]) for _ in range(4)]
        tms.append(dict(token=tok, tags=[["x", "y"], ["p"], ["q", "r"]], char_ngrams=cn, type_ngrams=[], bias=[1, 2, 3, 4]))
    cng = {fw("".join(rng.choice(alpha, size=rng.integers(1, 4)))): rng.integers(-500, 500, size=4).tolist() for _ in range(30)}
    model = dict(char_ngrams=list(cng.items()), type_ngrams=[(bytes([2]), [5, -5, 7, 1, 0, 2])], dict=[], bias=-3,
                 char_window=3, type_window=3, tag_models=tms)
    texts = ["".join(rng.choice(alpha, size=rng.integers(1, 25))) for _ in range(60)]
    _check(encode_model(model), texts, norm=True)


OVERRUN_MODEL = dict(
    char_ngrams=[("ab", [3, -4, 5, 1])], type_ngrams=[], dict=[], bias=1, char_window=2, type_window=0,
    # "a": 5 + 5 candidates, but a bias of 3 (an eight-wide vector): more candidates than scores
    tag_models=[dict(token="a", tags=[list("vwxyz"), list("pqrst")], char_ngrams=[], type_ngrams=[], bias=[1, 2, 3]),
                dict(token="b", tags=[["x", "y"]], char_ngrams=[], type_ngrams=[], bias=[7, 8])])


def test_overrun_model_has_no_scores():
    """A token whose slots have more candidates than its score vector has scores: the kernels answer -1 for it and count
    no scores (vpt_fill_tags reports InvalidModel); the well-formed token beside it keeps its vector."""
    model = OVERRUN_MODEL
    mb = encode_model(model)
    L = emul_lib()
    for text in ("a", "b", "ab", "ba", "aab"):
        ids, sc, uns = _emul(L, mb, text)
        bd = OraclePredictor(mb).predict(text)[1].tolist()
        toks, cur = [], text[0]
        for c, b in zip(text[1:], bd):
            if b == 1:
                toks.append(cur)
                cur = c
            else:
                cur += c
        toks.append(cur)
        assert [int(i) >= 0 for i in ids] == [t == "b" for t in toks], (text, toks)
        assert sc.tolist() == [7, 8, 0, 0, 0, 0, 0, 0] * toks.count("b")
        assert uns == toks.count("a")
