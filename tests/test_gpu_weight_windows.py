"""Every scoring kernel at the edges of the weight windows its plan accepts (vpt_testlib/weight_windows.py builds the
models and checks each one against its restatement of the builder and the plan), against the CPU oracle, bit for bit:
predict_batch (scores, boundaries, offsets, status, pattern-id states of the tag predictors), predict_batch_compact
(the boundary bits) and predict on one sentence.  Each batch holds a round of edge groups for every sub-block of the
device, whose sentences put rows against their neighbours at exactly the separator gap and across every 32-slot
chunk edge, and a last partial group.
The file takes 73 s on an H100 80GB HBM3 (SXM, 700 W power limit), CUDA start-up, model builds and oracle included."""
import numpy as np
import pytest

import vaporetto_b200 as vb
from vpt_testlib import weight_windows as ww
from vpt_testlib.oracle import OraclePredictor

pytestmark = pytest.mark.gpu

CASES = ww.all_cases()


def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_device_matches_oracle(case):
    mb = case.model()
    p = vb.Predictor(vb.Model.read(mb), predict_tags=case.tags)
    full = p.kernel_plan(case.states)
    assert ww.library_plan(full) == case.plan(), full
    o = OraclePredictor(mb, predict_tags=case.tags)
    f = case.facts()
    tiled = full["kernel"] in ("k_fused", "k_tile_fast")
    n_groups = full["sub_blocks"] * n_sm() + 8 if tiled else 64
    text, offs, sents = ww.batch(case, f, full, n_groups, seed=len(case.name))

    # predict_batch
    r = p.predict_batch(text, offs, want_states=case.states)
    sc, bd, boff, st = o.predict_batch(text, offs, nthreads=8)
    assert r.bound_offsets.tolist() == boff.tolist()
    assert r.status.tolist() == st.tolist()
    assert np.array_equal(r.scores, sc)
    assert np.array_equal(r.boundaries, bd)
    if case.states:
        cs, ts, coff = o.predict_batch_states(text, offs, nthreads=8)
        assert r.char_offsets.tolist() == coff.tolist()
        assert np.array_equal(r.char_states, cs)
        assert np.array_equal(r.type_states, ts)

    # predict_batch_compact: the boundary bits, unpacked here
    c = p.predict_batch_compact(text, offs)
    assert c.n_boundaries == len(bd)
    bits = np.unpackbits(c.boundary_bits.view(np.uint8), bitorder="little")[: len(bd)]
    assert np.array_equal(bits, bd)

    # predict: one sentence through the single-sentence path
    one = ww.value_sentence() if case.values else max((s for s in sents[:64] if len(s.encode()) <= 2048), key=len)
    s = vb.Sentence.from_raw(one)
    p.predict(s)
    if case.tags:
        osc, obd, ocs, ots = o.predict(one, states=True)
        assert s._char_states.tolist() == ocs.tolist()
        assert s._type_states.tolist() == ots.tolist()
    else:
        osc, obd = o.predict(one)
    assert s.boundary_scores().tolist() == osc.tolist()
    assert s.boundaries().tolist() == obd.tolist()
