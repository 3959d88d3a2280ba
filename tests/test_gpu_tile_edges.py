"""Every variant of the tile kernels (k_fused, k_tile_fast) against the CPU oracle on batches whose groups sit exactly on
the edges of that variant's tile buffers (vpt_testlib/tile_edges.py builds them and checks each edge against its
restatement of the kernels' fit tests).  Bit-exact: scores, boundaries, offsets, status and pattern-id states.
The file takes 68 s on an H100 SXM, model builds and oracle included."""
import numpy as np
import pytest

import vaporetto_b200 as vb
from vpt_testlib import tile_edges as te
from vpt_testlib.oracle import OraclePredictor

pytestmark = pytest.mark.gpu

RECIPES = te.variant_recipes()


def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def predict_dev(p, text, offs, states):
    """The whole batch in ONE scoring launch (vpt_predict_batch_dev; the host-buffer entry point cuts a batch into
    chunks, each its own launch)."""
    import ctypes as C
    import torch
    dev = torch.device("cuda:0")
    n = len(offs) - 1
    cap = max(len(text), 1)
    d_text = torch.zeros(len(text) + 64, dtype=torch.uint8, device=dev)   # (offsets start at 0: their alignment holds)
    d_text[: len(text)] = torch.from_numpy(text.copy()).to(dev)
    d_off = torch.from_numpy(offs.astype(np.int64)).to(dev)
    ws = torch.empty(vb.lib().vpt_workspace_size(n), dtype=torch.uint8, device=dev)
    d_scores = torch.empty(cap, dtype=torch.int32, device=dev)
    d_bounds = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_boff = torch.empty(n + 1, dtype=torch.int64, device=dev)
    d_status = torch.empty(n, dtype=torch.int32, device=dev)
    d_coff = torch.empty(n + 1, dtype=torch.int64, device=dev)
    d_cs = torch.empty(cap, dtype=torch.int32, device=dev) if states else None
    d_ts = torch.empty(cap, dtype=torch.int32, device=dev) if states else None
    ptr = lambda t: None if t is None else t.data_ptr()
    rc = vb.lib().vpt_predict_batch_dev(p._h, d_text.data_ptr(), d_off.data_ptr(), n, ws.data_ptr(), ws.numel(),
                                        d_scores.data_ptr(), d_bounds.data_ptr(), d_boff.data_ptr(), d_status.data_ptr(),
                                        ptr(d_cs), ptr(d_ts), d_coff.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, vb.lib().vpt_last_error()
    torch.cuda.synchronize()
    boff = d_boff.cpu().numpy().astype(np.uint64)
    coff = d_coff.cpu().numpy().astype(np.uint64)
    nb, nc = int(boff[-1]), int(coff[-1])
    out = dict(scores=d_scores[:nb].cpu().numpy(), boundaries=d_bounds[:nb].cpu().numpy(), bound_offsets=boff,
               status=d_status.cpu().numpy(), char_offsets=coff)
    if states:
        out["char_states"] = d_cs[:nc].cpu().numpy().view(np.uint32)
        out["type_states"] = d_ts[:nc].cpu().numpy().view(np.uint32)
    return out


def check(p, o, text, offs, states):
    r = predict_dev(p, text, offs, states)
    sc, bd, boff, st = o.predict_batch(text, offs, nthreads=8)
    assert r["bound_offsets"].tolist() == boff.tolist()
    assert r["status"].tolist() == st.tolist()
    assert np.array_equal(r["scores"], sc)
    assert np.array_equal(r["boundaries"], bd)
    if states:
        cs, ts, coff = o.predict_batch_states(text, offs, nthreads=8)
        assert r["char_offsets"].tolist() == coff.tolist()
        assert np.array_equal(r["char_states"], cs)
        assert np.array_equal(r["type_states"], ts)


def device_predictor(budget, args, tags, monkeypatch):
    if budget:
        monkeypatch.setenv("VPT_SEED_BUDGET", budget)   # 16-bit seeds: the seed table stays in global memory
    else:
        monkeypatch.delenv("VPT_SEED_BUDGET", raising=False)
    mb, words = te.variant_model(*args)
    return mb, words, vb.Predictor(vb.Model.read(mb), predict_tags=tags)


@pytest.mark.parametrize("name,budget,args,tags,states,key", RECIPES, ids=[r[0] for r in RECIPES])
def test_variant_at_tile_edges(name, budget, args, tags, states, key, monkeypatch):
    mb, words, p = device_predictor(budget, args, tags, monkeypatch)
    o = OraclePredictor(mb, predict_tags=tags)
    plan = p.kernel_plan(states)
    assert te.plan_key(plan) == key, plan
    # one launch of at least three rounds of groups over all sub-blocks of the device (grid = min(SMs, groups /
    # sub-blocks) CTAs of plan["sub_blocks"] sub-blocks), with edge and slow-path groups spread over every round: a
    # sub-block takes group after group, and groups follow slow-path and overflow groups on the same sub-block
    subs = plan["sub_blocks"] * n_sm()
    b = te.build(plan, te.ALPHABET, words, n_groups=3 * subs + 8, seed=sum(map(ord, name)), tail=63)
    text, offs = b.arrays()
    n_groups_launch = (len(offs) - 1 + te.GROUP - 1) // te.GROUP
    assert n_groups_launch >= 3 * subs and (len(offs) - 1) % te.GROUP == 63
    check(p, o, text, offs, states)
    # a last group of one sentence
    b1 = te.EdgeBatch(plan, te.ALPHABET, seed=7)
    b1.filler(3)
    b1.add([b1.chars(30)], "partial last group of 1")
    text, offs = b1.arrays()
    assert (len(offs) - 1) % te.GROUP == 1
    check(p, o, text, offs, states)


def test_every_variant_reached(monkeypatch):
    """The recipes above reach, on the device, every variant the dispatch can launch (te.all_plan_keys, which
    test_kernel_plan.py checks against the kernel instantiations of the library) except the ones no valid model
    reaches (te.UNREACHABLE, with the reason)."""
    reached = set()
    for name, budget, args, tags, states, key in RECIPES:
        reached.add(te.plan_key(device_predictor(budget, args, tags, monkeypatch)[2].kernel_plan(states)))
    want = te.all_plan_keys() - set(te.UNREACHABLE)
    assert reached == want, sorted(want ^ reached)
    print(f"\ntile edge variants reached: {len(reached)} of {len(te.all_plan_keys())}; unreachable: {len(te.UNREACHABLE)} "
          f"({sorted(set(te.UNREACHABLE.values()))})")
    for k in sorted(reached):
        print("  ", dict(zip(te.PLAN_KEYS, k)))


# ---- the single-sentence path of vpt_predict at its byte limit (2 048 bytes) ------------------------------------

@pytest.mark.parametrize("nbytes", [2047, 2048, 2049])
def test_single_sentence_at_its_byte_limit(nbytes):
    mb, _ = te.variant_model(3, 3, (1, 2, 3, 4), (), tags=2)
    p, o = vb.Predictor(vb.Model.read(mb), predict_tags=True), OraclePredictor(mb, predict_tags=True)
    assert p.kernel_plan(True)["kernel"] == "k_fused"
    b = te.EdgeBatch(p.kernel_plan(True), te.ALPHABET, seed=nbytes)
    for text in (b.compose(nbytes // 3, nbytes), b.compose(nbytes, nbytes), b.compose((nbytes + 3) // 4, nbytes)):
        assert len(text.encode()) == nbytes
        s = vb.Sentence.from_raw(text)
        p.predict(s)
        sc, bd, cs, ts = o.predict(text, states=True)
        assert s.boundary_scores().tolist() == sc.tolist()
        assert s.boundaries().tolist() == bd.tolist()
        assert s._char_states.tolist() == cs.tolist()
        assert s._type_states.tolist() == ts.tolist()
