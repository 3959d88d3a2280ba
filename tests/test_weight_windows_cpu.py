"""CPU checks of the weight-window cases (vpt_testlib/weight_windows.py): the restated builder and plan against the
library's plan on host-only predictors, every case on the edge it names, and, with the oracle, that the gap cases are
live and that the weight-value cases really wrap and really score 0."""
import itertools

import numpy as np
import pytest

import vaporetto_b200 as vb
from vpt_testlib import weight_windows as ww
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.oracle import OraclePredictor

CASES = ww.all_cases()


def host_plan(mb, tags, states=False):
    return ww.library_plan(vb.Predictor(vb.Model.read(mb), predict_tags=tags, device=-1).kernel_plan(states))


def _sweep_model(r0, width, tw, tng, tags=False, seed=0):
    hi = r0 + width - 1
    rows = ((r0, hi),) if width <= 6 else ((r0, r0 + 5), (hi - 5, hi))
    return ww.build_model(cw=ww.window_for(r0, hi), rows=rows, tw=tw, tng_lens=tng if tw else (), tags=2 if tags else 0,
                          n_per_len=4, seed=seed)


@pytest.mark.parametrize("width", [5, 6, 7])
def test_plan_sweep_r0_width_type_window(width):
    """r0 -26..20, row widths 5..7, type windows 0..4: the restated plan is the library's."""
    seen = set()
    for r0, tw in itertools.product(range(-26, 21), range(5)):
        md = _sweep_model(r0, width, tw, tuple(range(1, min(2 * tw, 4) + 1)), seed=(r0 + 30) * 7 + tw)
        f = ww.restate(md)
        assert f["smin"] == r0 and f["smax"] - f["smin"] == width
        want = ww.plan(f)
        assert host_plan(encode_model(md), False) == want, (r0, width, tw)
        seen.add(want["kernel"])
    assert seen == ({"k_tile_fast"} if width == 7 else {"k_fused", "k_tile_fast", "k_score_fast"})


@pytest.mark.parametrize("tags", [False, True])
def test_plan_sweep_type_ngram_lengths(tags):
    """Type windows 0..4 with type n-grams of one length 1..6 (split tables, the type automaton, tag light tables)."""
    for r0, tw, L in itertools.product((-5, -4, -3, 0, 1, -7), range(5), range(1, 7)):
        md = _sweep_model(r0, 6, tw, (L,), tags=tags, seed=100 + L)
        want = ww.plan(ww.restate(md, tags))
        assert host_plan(encode_model(md), tags, states=tags) == want, (r0, tw, L, tags)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_case_on_its_edge(case):
    """Every case lands on the edge it names (Case.model raises otherwise), and the library plans it as restated."""
    mb = case.model()
    full = vb.Predictor(vb.Model.read(mb), predict_tags=case.tags, device=-1).kernel_plan(case.states)
    assert ww.library_plan(full) == case.plan()
    # the first groups of the device test's batch are checked on their edges (ww.check_group_edges raises)
    text, offs, sents = ww.batch(case, case.facts(), full, n_groups=4, seed=len(case.name))
    assert len(offs) - 1 == len(sents) and int(offs[-1]) == len(text)


def test_cases_reach_the_matrix():
    plans = [c.plan() for c in CASES]
    for kern, what, want in ww.MATRIX:
        assert any(all(p[k] == v for k, v in want.items()) for p in plans), f"no case reaches {kern} {what}"
    # and the window ends of every kernel
    r0s = {(c.plan()["kernel"], c.facts()["r0"]) for c in CASES if c.facts()["fast"]}
    for want in [("k_fused", r) for r in range(-5, 1)] + [("k_tile_fast", r) for r in (-8, -7, -6, 1, 2)] + \
            [("k_score_fast", r) for r in (-24, 18, -9, 3)]:
        assert want in r0s, want


GAP_CASES = [(c, side) for c in CASES for side in c.gap_sides]


@pytest.mark.parametrize("case,side", GAP_CASES, ids=[f"{c.name}-{s}" for c, s in GAP_CASES])
def test_gap_is_live(case, side):
    """With the gap one slot short, the row of a sentence's edge character would reach its neighbour's edge
    boundary: scoring the two as one sentence, with gap - 1 pattern-free characters between them, the edge boundary
    changes when the edge character is a pattern character."""
    mb = case.model()
    pl = case.plan()
    assert pl["kernel"] in ("k_fused", "k_tile_fast") and not pl["general"]
    f = case.facts()
    assert (side == "left" and pl["gap"] == -f["r0"] - 1) or (side == "right" and pl["gap"] == f["r0"] + 5)
    o = OraclePredictor(mb, predict_tags=case.tags)
    with_pat, without, j = ww.gap_probe(f, pl, side, seed=len(case.name))
    a, b = o.predict(with_pat)[0], o.predict(without)[0]
    assert len(a) == len(b) and a[j] != b[j]
    # a full gap keeps them apart: one more pattern-free character and the edge boundary no longer changes
    mid = ww.SAME_TYPE_FILL * (pl["gap"] - 1)
    k = with_pat.index(mid) if mid else None
    assert k is not None
    wide, wide_without = (with_pat[:k] + ww.SAME_TYPE_FILL + with_pat[k:], without[:k] + ww.SAME_TYPE_FILL + without[k:])
    j2 = j if side == "left" else j + 1
    a, b = o.predict(wide)[0], o.predict(wide_without)[0]
    assert a[j2] == b[j2]


VALUE_CASES = [c for c in CASES if c.values]


@pytest.mark.parametrize("case", VALUE_CASES, ids=[c.name for c in VALUE_CASES])
def test_values_wrap_and_score_exactly(case):
    mb = case.model()
    f = case.facts()
    o = OraclePredictor(mb, predict_tags=True)
    # boundaries that score exactly 0, 1, INT32_MIN, INT32_MAX: 人's row over the bias; 0 is not a boundary
    s = ww.value_sentence()
    c = s.index("人")
    sc, bd = o.predict(s)[:2]
    for k, v in enumerate(ww.EXACT):
        assert sc[c + f["r0"] + k] == v
        assert bd[c + f["r0"] + k] == (1 if v > 0 else 0)
    # the merged row of 星火 wraps in the builder
    raw = f["raw"]["星火"][1]
    assert any(v > ww.I32_MAX for v in raw)
    # device sums that wrap: a run of 火, whose row is BIG in every entry, plus the bias
    sc = o.predict(ww.WRAP_RUN)[0]
    unwrapped = ww.VALUE_BIAS + (f["smax"] - f["smin"]) * ww.BIG
    assert unwrapped > ww.I32_MAX and sc[len(sc) // 2] == ww.wrap32(unwrapped)
    # 猫社's merged row trims to empty: it adds nothing, and its pattern id is still the state after 社
    assert f["rows"]["猫社"][1] == []
    pats = sorted(f["rows"], key=lambda p: p.encode())
    s = "山猫社山山山山山山山山山山山山山山山山山山山山山山"
    sc, _, cs, _ = o.predict(s, states=True)
    assert cs[2] == pats.index("猫社")
    assert np.array_equal(sc, o.predict(s.replace("社", "山"))[0])


def test_row_merge_restatement():
    """The restated merge on hand-made rows: union of equal strings, suffix sums, wrapping, trim."""
    md = dict(char_window=2, type_window=0, bias=0, type_ngrams=[], tag_models=[],
              char_ngrams=[("a", [0, 5, 0, 0]), ("ba", [0, ww.I32_MAX, 0]), ("cb", [0, 0, 0])],
              dict=[("a", [1, 0], ""), ("xyzw", [7, 0, 0, 0, 0], "")])
    rows, raw = ww.merged_rows(md, False)
    assert rows["a"] == (-1, [6])              # the n-gram row at -2 plus the word row at -1, trimmed
    assert rows["ba"] == (-1, [ww.wrap32(ww.I32_MAX + 6)]) and raw["ba"][1][1] == ww.I32_MAX + 6
    assert rows["cb"] is not None and rows["cb"][1] == []
    assert rows["xyzw"] == (-4, [7])
    f = ww.restate(md)
    assert (f["smin"], f["smax"], f["rel_min"], f["rel_max"], f["r0"]) == (-1, 0, -4, 0, -1)
    assert f["has_overflow"] and f["fast"]
