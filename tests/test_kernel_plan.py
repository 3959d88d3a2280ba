"""CPU checks of the kernel plan (vpt_predictor_kernel_plan on host-only predictors): which kernel variant and tile
geometry each model shape gets, and that the tile-edge batches reach the edges of every such plan."""
import pytest

import vaporetto_b200 as vb
from vpt_testlib import synth
from vpt_testlib import tile_edges as te

RECIPES = te.variant_recipes()

# k_fused buffers per (seeds in shared memory, states, overflow rows): text bytes, slots, sub-blocks per CTA
FUSED_GEOMETRY = {
    (1, 0, 0): (10240, 3840, 4), (1, 1, 0): (9216, 3328, 4), (1, 0, 1): (10240, 3840, 3), (1, 1, 1): (9216, 3264, 3),
    (0, 0, 0): (10240, 3840, 4), (0, 1, 0): (9216, 3328, 4), (0, 0, 1): (9216, 3584, 4), (0, 1, 1): (9216, 2944, 4),
}


def host_plan(mb, tags, states, budget, monkeypatch):
    if budget:
        monkeypatch.setenv("VPT_SEED_BUDGET", budget)
    else:
        monkeypatch.delenv("VPT_SEED_BUDGET", raising=False)
    return vb.Predictor(vb.Model.read(mb), predict_tags=tags, device=-1).kernel_plan(states)


@pytest.mark.parametrize("name,budget,args,tags,states,key", RECIPES, ids=[r[0] for r in RECIPES])
def test_plan_and_edges(name, budget, args, tags, states, key, monkeypatch):
    mb, words = te.variant_model(*args)
    plan = host_plan(mb, tags, states, budget, monkeypatch)
    assert te.plan_key(plan) == key
    assert plan["group"] == 64
    if plan["kernel"] == "k_fused":
        geo = FUSED_GEOMETRY[(plan["seeds_smem"], plan["states"], int(plan["deep"] == 2))]
        assert (plan["text_cap"], plan["slot_cap"], plan["sub_blocks"]) == geo
        assert plan["gap"] == (2 if plan["common_shape"] else 3) and plan["lag"] == (3 if plan["common_shape"] else 2)
    else:
        assert (plan["text_cap"], plan["slot_cap"], plan["sub_blocks"], plan["lag"]) == (12288, 3072, 4, 0)
    # every edge group lands on its side of the restated fit tests (te.EdgeBatch.add raises otherwise)
    b = te.build(plan, te.ALPHABET, words, n_groups=0, seed=1, tail=1)
    names = [e for e, _ in b.edges]
    assert sum(e.startswith("slots S = limit") for e in names) == 3
    assert sum(e.startswith("text span") for e in names) == (6 if plan["kernel"] == "k_fused" else 0)
    assert sum(e.startswith("sentence of one range") for e in names) == 4
    assert any(e.startswith("long words") for e in names) == (len([w for w in words if 4 <= len(w) <= 12]) > 0)


def test_variant_list_matches_the_library():
    """te.all_plan_keys() is the set of kernel instantiations the built library contains (their mangled names are in
    its host code, where the launches register them): a variant added to the dispatch shows up here."""
    import re
    data = open(vb._SO, "rb").read()
    fused = {("k_fused", int(s), int(c), int(d), int(st), 0, 0, 0, 0)
             for s, c, d, st in re.findall(rb"k_fusedILb([01])ELb([01])ELi([0-9]+)ELb([01])EE", data)}
    tile = {("k_tile_fast", int(s), 0, 0, 0, int(r0 == b"n3"), int(g), int(sp), int(o))
            for s, r0, g, sp, o in re.findall(rb"k_tile_fastILb([01])ELi(n?[0-9]+)ELb([01])ELb([01])ELb([01])EE", data)}
    assert len(fused) == 24 and len(tile) == 20
    assert fused | tile == te.all_plan_keys()


def test_recipes_reach_every_reachable_variant():
    keys = {r[-1] for r in RECIPES}
    assert keys == te.all_plan_keys() - set(te.UNREACHABLE)
    assert len(keys) == 24 + 12


def test_plan_of_other_shapes(monkeypatch):
    # windows > 3 need the type automaton: general tables; shallow ones through k_tile_fast, deep ones one warp per sentence
    mb = synth.gen_model_bccwj_shaped(n_patterns=2000, sample_sentences=2000, window=4)
    pl = host_plan(mb, False, False, None, monkeypatch)
    assert pl["kernel"] == "k_tile_fast" and pl["general"] == 1
    mb = synth.gen_model_bccwj_shaped(n_patterns=2000, sample_sentences=2000, window=4, dict_words=300)
    pl = host_plan(mb, False, False, None, monkeypatch)
    assert pl["kernel"] == "k_score_general" and pl["text_cap"] == 0 and pl["group"] == 0
    # the bench model shape: k_fused, common shape, seeds in shared memory
    mb = synth.gen_model_bccwj_shaped(n_patterns=2000, sample_sentences=2000)
    pl = host_plan(mb, False, False, None, monkeypatch)
    assert te.plan_key(pl) == ("k_fused", 1, 1, 0, 0, 0, 0, 0, 0)


def test_fit_restatement():
    """The restated fit tests at their edges (the numbers of fused_kernel.cuh and kernels.cu)."""
    fused = dict(kernel="k_fused", text_cap=10240, slot_cap=3840, gap=2)
    tile = dict(kernel="k_tile_fast", text_cap=12288, slot_cap=3072, gap=2)
    for lo in (0, 1, 15):
        assert te.text_fits(fused, 16 * 5 + lo, 16 * 5 + 10240 - 16)
        assert not te.text_fits(fused, 16 * 5 + lo, 16 * 5 + 10240 - 15)
    assert te.slots_fit(fused, 3840) and not te.slots_fit(fused, 3841)
    assert te.slots_fit(tile, 3064) and not te.slots_fit(tile, 3065)
    assert te.classify(fused, [0, 10], [10]) == ("fast",)
    assert te.classify(tile, [0, 10], [10]) == ("ranges", [(0, 1, False)])
    assert te.classify(fused, [0, 3840, 3850], [3840 - 4, 10]) == ("ranges", [(0, 1, False), (1, 2, False)])
    assert te.classify(fused, [0, 3837, 3847], [3837, 10]) == ("ranges", [(0, 1, True), (1, 2, False)])
