"""CPU checks of the full-width filter models and text (vpt_testlib/norm_variants.py): the filter tables against the
fixture and the library, the kernel variant every model plans (host-only predictors), and -- by the oracle alone -- that
the filter really changes what every model matches, so that the GPU comparisons in test_gpu_norm_variants.py are not
comparisons of text the filter leaves alone."""
import json
import os

import numpy as np
import pytest

import vaporetto_b200 as vb
from vpt_testlib import norm_variants as nv
from vpt_testlib import tile_edges as te
from vpt_testlib.oracle import OraclePredictor

RECIPES = nv.recipes()
ALL_MODELS = [(name, budget, args, tags, states, key) for name, budget, args, tags, states, key in RECIPES] + \
             [(name, None, args, tags, states, key) for name, args, tags, states, key in nv.SCORE_KERNELS]


def test_tables_match_the_fixture_and_the_library(golden_dir):
    fixture = {int(k): v for k, v in json.load(open(os.path.join(golden_dir, "kytea_fullwidth_map.json"))).items()}
    assert sorted(map(ord, nv.SOURCES)) == sorted(fixture)
    assert sum(ord(c) < 0x80 for c in nv.SOURCES) == 86 and sum(ord(c) >= 0x80 for c in nv.SOURCES) == 10
    assert set(nv.IMAGES) == {chr(v) for v in fixture.values()}
    assert nv.FIXED == " #$;\\^`|~"
    assert nv.DASHES == "–―─－"
    fw = vb.lib().vpt_kytea_fullwidth
    for c in nv.SOURCES:
        assert fw(ord(c)) == fixture[ord(c)] == ord(nv.FILTER[c]) != ord(c), c
    for c in nv.IMAGES + nv.FIXED + "あアー人éß𠀋𩸽":
        assert fw(ord(c)) == ord(c), c
        assert c not in nv.SPELLINGS or c in nv.IMAGES
    rng = np.random.default_rng(0)
    word = nv.PATTERN_ALPHABET * 3
    seen = set()
    for _ in range(50):
        s = nv.source_spellings(word, rng)
        assert nv.normalize(s) == word and len(s) == len(word)
        assert all(s[i] in nv.SPELLINGS[c] for i, c in enumerate(word) if c in nv.SPELLINGS)
        seen |= {s[i] for i, c in enumerate(word) if c == "ー"}
    assert seen == set(nv.DASHES)


def host_predictor(mb, tags, budget, monkeypatch):
    if budget:
        monkeypatch.setenv("VPT_SEED_BUDGET", budget)
    else:
        monkeypatch.delenv("VPT_SEED_BUDGET", raising=False)
    return vb.Predictor(vb.Model.read(mb), predict_tags=tags, device=-1)


def test_models_keep_the_shape_of_the_tile_recipes():
    """Every norm model has the windows and the template switches of its tile_edges recipe; the recipes themselves are
    untouched (test_kernel_plan.py checks them)."""
    assert [r[1:] for r in RECIPES] == [r[1:] for r in te.variant_recipes()]
    assert {r[-1] for r in RECIPES} == te.all_plan_keys() - set(te.UNREACHABLE)


@pytest.mark.parametrize("name,budget,args,tags,states,key", ALL_MODELS, ids=[r[0] for r in ALL_MODELS])
def test_plan_and_the_filter_changes_what_matches(name, budget, args, tags, states, key, monkeypatch):
    mb, words = nv.norm_model(*args)
    p = host_predictor(mb, tags, budget, monkeypatch)
    plan = p.kernel_plan(states)
    assert te.plan_key(plan) == key, plan
    rng = np.random.default_rng(5)
    spelled = [nv.source_spellings(w, rng) for w in words]
    assert all(s != w and nv.normalize(s) == w for s, w in zip(spelled, words))
    if plan["group"]:
        sents = te.build(plan, nv.TEXT_ALPHABET, spelled, n_groups=0, seed=1, tail=1).sents
    else:
        sents = nv.text_for(words, 3000, rng)
    o = OraclePredictor(mb, predict_tags=tags)
    # boundary scores: the filter changes them on most sentences
    differ = sum(not np.array_equal(o.predict(nv.normalize(s))[0], o.predict(s)[0]) for s in sents)
    assert differ >= 0.75 * len(sents), (differ, len(sents))
    # char pattern-id states (a tag predictor emits them: a model without tag models gets one more, whose few short
    # char n-grams do not change which long patterns exist): patterns hit only under the filter, long ones included
    so = o if tags else OraclePredictor(nv.norm_model(*args[:4], 1, *args[5:])[0], predict_tags=True)
    pats = [x[0].decode() for x in so.dump_patterns(0)]
    hit = {}
    for norm in (True, False):
        hit[norm] = set()
        for s in sents:
            cs = so.predict(nv.normalize(s) if norm else s, states=True)[2]
            hit[norm] |= {pats[i] for i in cs.tolist() if i != 0xFFFFFFFF}
    only = hit[True] - hit[False]
    assert len(only) >= 15, sorted(only)
    if words:
        assert {w for w in only if len(w) >= 4}, "no long pattern is hit only under the filter"
        if args[3]:
            assert {w for w in only if len(w) in args[3]}, "no dictionary word is hit only under the filter"
    if tags:
        # known tokens (images) found only under the filter
        found = {True: 0, False: 0}
        only_norm = 0
        for s in sents[:1000]:
            tn = o.predict_tags(nv.normalize(s))[0]
            tr = o.predict_tags(s)[0]
            found[True] += int(np.count_nonzero(tn >= 0))
            found[False] += int(np.count_nonzero(tr >= 0))
            only_norm += sum(1 for i in range(len(s)) if tn[i] >= 0 and tr[i] < 0 and s[i] in nv.SOURCES)
        assert only_norm >= 100 and found[True] >= 2 * found[False], (found, only_norm)
