"""The restated chunk and ring arithmetic of k_tags (vpt_testlib/tag_edges.py), the edge cases it builds, and the
oracle's tags for the edge model's long tokens -- everything the GPU edge tests (test_gpu_tag_edges.py) rely on."""
import random

import pytest

from vpt_testlib import tag_edges as te
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.oracle import OraclePredictor


@pytest.fixture(scope="module")
def cases():
    return te.edge_cases()


def test_shortest_stale_tokens():
    """The shortest token whose first ring slot is overwritten before its end is handled, per character width, for a
    sentence starting 4-byte aligned; for 1-byte characters it moves by one per byte of misalignment."""
    assert [te.shortest_stale(w, 0) for w in (1, 2, 3, 4)] == [(98, 127), (162, 63), (183, 42), (194, 31)]
    assert [te.shortest_stale(1, a)[0] for a in range(4)] == [98, 99, 100, 101]
    # 400 x 'a' with the token [50, 249]: its end is handled in the step at 224, when slot 50 holds character 306
    nd = te.uniform_nd(1, 400, 0)
    assert nd[249 // te.STEP] == 384
    assert max(c for c in range(nd[7]) if c % te.RING == 50) == 306
    assert te.outcome(1, 400, 0, 50, 249, fixed=False) == "stale"
    assert te.outcome(1, 400, 0, 50, 249, fixed=True) == "ok"


def test_edge_cases_reach_their_edges(cases):
    kinds = {}
    for c in cases:
        kinds.setdefault(c.kind, set()).add((c.w, c.align))
        s, e = c.span()
        L = e - s + 1
        tok = c.tokens[c.target]
        assert len(tok) == L and tok.endswith(te.term(c.w))
        assert all(len(ch.encode("utf-8")) == c.w for ch in c.sentence)
        assert all(t.endswith(te.term(c.w)) for t in c.tokens)
        assert te.outcome(c.w, len(c.sentence), c.align, s, e, fixed=True) == "ok"
        if c.kind == "stale":
            assert c.old == "stale"
        if c.kind in ("len217", "whole300", "steps8"):
            assert c.old == "unserved" and L > te.NEAR
        if c.kind == "len216":
            assert L == te.NEAR and c.old != "unserved"
    every = {(w, a) for w in (1, 2, 3, 4) for a in range(4)}
    for k in ("stale", "stale-1", "len216", "len217", "lane0", "lane31", "steps1", "steps2", "steps8", "whole2",
              "whole40", "whole100", "whole300"):
        assert kinds[k] == every, k
    reachable = {(2, 1), (2, 3), (3, 0), (3, 1), (3, 2), (3, 3), (4, 1), (4, 2), (4, 3)}
    assert kinds["window-first"] == kinds["window-last"] == reachable


def test_twins_differ_in_one_character(cases):
    known = set(te.known_tokens(cases))
    by_kind = {}
    for c in cases:
        by_kind.setdefault((c.kind, c.w, c.align), []).append(c)
    for pair in by_kind.values():
        k = [c for c in pair if c.known]
        u = [c for c in pair if not c.known]
        for a, b in zip(k, u):
            ta, tb = a.tokens[a.target], b.tokens[b.target]
            assert ta in known and tb not in known
            assert len(ta) == len(tb) and sum(x != y for x, y in zip(ta, tb)) == 1
            assert a.span() == b.span()


def test_fixed_carry_is_always_live():
    """Random sentences of mixed widths and random token ends at every alignment: the carried first byte is always
    read from a live slot (locate() asserts it), while the first k_tags reads stale slots in some of them."""
    rng = random.Random(5)
    stale = 0
    for _ in range(300):
        n = rng.randint(1, 900)
        widths = [rng.choice((1, 1, 2, 3, 4)) for _ in range(n)]
        lead = [0]
        for w in widths[:-1]:
            lead.append(lead[-1] + w)
        nbytes = lead[-1] + widths[-1]
        p_end = rng.choice((0.002, 0.01, 0.1, 0.5))
        ends = [i for i in range(n - 1) if rng.random() < p_end] + [n - 1]
        for align in range(4):
            nd = te.step_nd(lead, nbytes, align)
            s = 0
            for e in ends:
                assert te.locate(nd, n, s, e, fixed=True)[0] == "ok"
                stale += te.locate(nd, n, s, e, fixed=False)[0] == "stale"
                s = e + 1
    assert stale > 0


def test_oracle_tags_the_long_tokens_by_hand(cases):
    """The edge model's boundaries are exactly the token ends, and the oracle's predict_tags gives the hand-derived
    candidates (tag_edges.expected_cands) on every case -- lengths up to 300 characters -- and on the 70 000-byte lines."""
    mb = encode_model(te.model(cases))
    o = OraclePredictor(mb, predict_tags=True)
    assert o.n_tags == 2
    known = set(te.known_tokens(cases))
    for c in cases:
        _, bounds = o.predict(c.sentence)
        want_b = []
        for t in c.tokens:
            want_b += [0] * (len(t) - 1) + [1]
        assert bounds.tolist() == want_b[:-1], (c.kind, c.w, c.align)
        tt, ti = o.predict_tags(c.sentence)
        want = te.expected_sentence_cands(c.tokens, known)
        assert ti.tolist() == want, (c.kind, c.w, c.align, c.known)
        assert [x >= 0 for x in tt.tolist()] == [w[0] >= 0 for w in want]
    # (the prefix has no terminator: only its bias counts)
    for line, want in ((te.LONG_KNOWN, te.expected_cands(te.LONG_KNOWN, None)), (te.LONG_UNKNOWN, [-1, -1]),
                       (te.LONG_PREFIX, [1, len(te.LONG_PREFIX) % 3])):
        tt, ti = o.predict_tags(line)
        assert (tt[:-1] < 0).all() and (tt[-1] >= 0) == (want[0] >= 0)
        assert ti[-1].tolist() == want
