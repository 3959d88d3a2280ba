"""The device-buffer tag call vpt_predict_tags_batch_dev and the profiled scoring call vpt_predict_batch_dev_profiled.

vpt_predict_tags_batch_dev is the call through which a caller's own 0 / 1 boundaries reach k_tags.  Every test scores a
batch with vpt_predict_batch_dev (pattern-id states on), then predicts tags on boundary patterns the test sets: the
predicted ones, all 1, all 0, random ones and tilings of the tag models' own tokens, against the CPU oracle on the same
boundaries (vpt_testlib/tags_given_oracle.py; token ids against the host path, vpt_fill_tags).  Every output buffer is
filled with a sentinel first: the call writes exactly the batch's characters, and -1 wherever no token ends.  Then the
call's contract: offsets that do not start at 0, sub-batches passed by pointer offset, nullable states, the unserved
counter, the caller's stream and the rejections.

vpt_predict_batch_dev_profiled launches the stages one at a time between events: it must write what
vpt_predict_batch_dev writes, for every kind of scoring kernel."""
import ctypes as C
import math

import numpy as np
import pytest

import vaporetto_b200 as vb
from test_gpu_batch_pipeline import _workload
from test_gpu_parity import _random_model
from test_tags_given_cpu import host_tags, token_bounds
from vpt_testlib import norm_variants as nv
from vpt_testlib import synth
from vpt_testlib import tag_edges as te
from vpt_testlib import tile_edges as tle
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.oracle import OraclePredictor
from vpt_testlib.tags_given_oracle import TagsGivenOracle

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED = 2, 17
SENTINEL = -7
GUARD = 64   # entries past the batch's characters that must keep the sentinel


def _torch():
    import torch
    return torch


def _stream_ptr(stream=None):
    torch = _torch()
    return C.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)


def _err():
    return vb.lib().vpt_last_error().decode()


def _batch(sents):
    enc = [s.encode() if isinstance(s, str) else s for s in sents]
    offs = np.zeros(len(enc) + 1, np.uint64)
    np.cumsum([len(e) for e in enc], out=offs[1:])
    return np.frombuffer(b"".join(enc), np.uint8), offs


class DevBatch:
    """A batch in device memory, with bench.py's buffers and dtypes (int64 offsets, int32 states), scored once by
    vpt_predict_batch_dev.  `lead`: bytes of other text in front of the batch, so its offsets start at `lead` while the
    text pointer stays 16-byte aligned."""

    def __init__(self, p, text, offs, lead=0, stream=None):
        torch = _torch()
        dev = torch.device("cuda:0")
        self.p, self.text, self.offs, self.n = p, text, offs, len(offs) - 1
        nbytes = int(offs[-1])
        self.d_text = torch.full((lead + nbytes + 64,), 0x5A, dtype=torch.uint8, device=dev)
        self.d_text[lead:lead + nbytes] = torch.from_numpy(text.copy()).to(dev)
        self.d_off = torch.from_numpy(offs.astype(np.int64) + lead).to(dev)
        n, cap = self.n, max(nbytes, 1)
        self.ws = torch.empty(vb.lib().vpt_workspace_size(n), dtype=torch.uint8, device=dev)
        self.d_scores = torch.empty(cap, dtype=torch.int32, device=dev)
        self.d_bounds = torch.empty(cap, dtype=torch.uint8, device=dev)
        self.d_boff = torch.empty(n + 1, dtype=torch.int64, device=dev)
        self.d_status = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        self.d_cs = torch.empty(cap, dtype=torch.int32, device=dev)
        self.d_ts = torch.empty(cap, dtype=torch.int32, device=dev)
        self.d_coff = torch.empty(n + 1, dtype=torch.int64, device=dev)
        rc = vb.lib().vpt_predict_batch_dev(p._h, self.d_text.data_ptr(), self.d_off.data_ptr(), n, self.ws.data_ptr(),
                                            self.ws.numel(), self.d_scores.data_ptr(), self.d_bounds.data_ptr(),
                                            self.d_boff.data_ptr(), self.d_status.data_ptr(), self.d_cs.data_ptr(),
                                            self.d_ts.data_ptr(), self.d_coff.data_ptr(), _stream_ptr(stream))
        assert rc == 0, _err()
        if stream is None:
            self.fetch()

    def fetch(self):
        _torch().cuda.synchronize()
        self.boff = self.d_boff.cpu().numpy().astype(np.uint64)
        self.coff = self.d_coff.cpu().numpy().astype(np.uint64)
        self.nb, self.nc = int(self.boff[-1]), int(self.coff[-1])
        self.status = self.d_status[: self.n].cpu().numpy()
        self.bounds = self.d_bounds[: self.nb].cpu().numpy()
        self.cs = self.d_cs[: self.nc].cpu().numpy().view(np.uint32)
        self.ts = self.d_ts[: self.nc].cpu().numpy().view(np.uint32)

    def outputs(self, n_tags):
        """tag_token [n_bound + n + GUARD] and tag_cand [(n_bound + n + GUARD) * n_tags] int32, filled with the
        sentinel (bench.py sizes them n_bound + n)."""
        torch = _torch()
        rows = self.nb + self.n + GUARD
        return (torch.full((rows,), SENTINEL, dtype=torch.int32, device="cuda:0"),
                torch.full((rows * max(n_tags, 1),), SENTINEL, dtype=torch.int32, device="cuda:0"))

    def tags(self, bounds=None, char_states=True, type_states=True, unserved=True, stream=None, n_sent=None,
             text_shift=0, predictor=None):
        """vpt_predict_tags_batch_dev on `bounds` (uint8 [n_bound]; None: the predicted boundaries) -> (rc, tag_token,
        tag_cand [rows, n_tags], unserved count) as host arrays of the whole output buffers."""
        torch = _torch()
        p = predictor or self.p
        nt = max(self.p.n_tags, 1)
        d_b = self.d_bounds
        if bounds is not None:
            d_b = torch.from_numpy(np.concatenate((bounds.astype(np.uint8), np.zeros(16, np.uint8)))).to("cuda:0")
        tok, cand = self.outputs(nt)
        d_uns = torch.zeros(1, dtype=torch.int32, device="cuda:0") if unserved else None
        rc = vb.lib().vpt_predict_tags_batch_dev(
            p._h, self.d_text.data_ptr() + text_shift, self.d_off.data_ptr(), self.n if n_sent is None else n_sent,
            self.d_status.data_ptr(), d_b.data_ptr(), self.d_boff.data_ptr(), self.d_coff.data_ptr(),
            self.d_cs.data_ptr() if char_states else None, self.d_ts.data_ptr() if type_states else None,
            tok.data_ptr(), cand.data_ptr(), d_uns.data_ptr() if unserved else None, _stream_ptr(stream))
        (stream or torch.cuda.current_stream()).synchronize()
        return (rc, tok.cpu().numpy(), cand.cpu().numpy().reshape(-1, nt)[:, : self.p.n_tags],
                int(d_uns.item()) if unserved else None)

    def ends(self, bounds):
        """Per character: a token ends there (a boundary after it, or the sentence's last character of a scored
        sentence)."""
        e = np.zeros(self.nc, bool)
        for i in range(self.n):
            c0, c1, b0 = int(self.coff[i]), int(self.coff[i + 1]), int(self.boff[i])
            if self.status[i] != 0 or c1 == c0:
                continue
            e[c0:c1 - 1] = bounds[b0:b0 + c1 - c0 - 1] == 1
            e[c1 - 1] = True
        return e


def check_tags(b, g, bounds, tok, cand, host_ids=None, unserved_at=()):
    """The call's outputs on `bounds` against the oracle on the same boundaries: known-ness and candidates for every
    character, token ids against the host path for the sentences `host_ids` (default all), the sentinel past the
    batch's characters, -1 wherever no token ends.  `unserved_at`: characters the device leaves to the host path
    (-1).  Returns the oracle's arrays."""
    nc = b.nc
    otok, ocand = g.tags(b.text, b.offs, b.boff, bounds, b.coff)
    if len(unserved_at):
        otok, ocand = otok.copy(), ocand.copy()
        otok[list(unserved_at)] = -1
        ocand[list(unserved_at)] = -1
    assert (tok[nc:] == SENTINEL).all() and (cand[nc:] == SENTINEL).all()
    tok, cand = tok[:nc], cand[:nc]
    bad = np.flatnonzero(((tok >= 0) != (otok >= 0)) | (cand != ocand).any(axis=1))
    assert bad.size == 0, ("differs from the oracle at characters", bad[:20].tolist(), tok[bad[:5]].tolist(),
                           otok[bad[:5]].tolist())
    ends = b.ends(bounds)
    assert (tok[~ends] == -1).all() and (cand[~ends] == -1).all()
    for i in (range(b.n) if host_ids is None else host_ids):
        c0, c1, b0 = int(b.coff[i]), int(b.coff[i + 1]), int(b.boff[i])
        if b.status[i] != 0:
            continue
        s = bytes(b.text[int(b.offs[i]):int(b.offs[i + 1])]).decode()
        htt, htc = host_tags(b.p, s, bounds[b0:b0 + c1 - c0 - 1], b.cs[c0:c1], b.ts[c0:c1])
        if len(unserved_at):
            keep = np.array([c0 + k not in unserved_at for k in range(c1 - c0)])
            htt, htc = np.where(keep, htt, -1), np.where(keep[:, None], htc, -1)
        assert tok[c0:c1].tolist() == htt.tolist() and cand[c0:c1].tolist() == htc.tolist(), (i, s)
    return otok, ocand


def differs(tok, cand, otok, ocand):
    nc = otok.size
    return bool((((tok[:nc] >= 0) != (otok >= 0)) | (cand[:nc] != ocand).any(axis=1)).any())


def random_patterns(b, rng):
    return {"predicted": b.bounds.copy(), "all1": np.ones(b.nb, np.uint8), "all0": np.zeros(b.nb, np.uint8),
            "bernoulli0.5": (rng.random(b.nb) < 0.5).astype(np.uint8),
            "bernoulli0.05": (rng.random(b.nb) < 0.05).astype(np.uint8)}


def run_patterns(b, g, patterns, host_ids=None):
    """Every pattern through the device and the oracle; the oracle on the PREDICTED boundaries must disagree with the
    device on every pattern but the predicted one (the call reads the caller's boundaries).  -> {name: (tok, cand)}"""
    ptok, pcand = g.tags(b.text, b.offs, b.boff, None, b.coff)
    out = {}
    for name, bd in patterns.items():
        rc, tok, cand, uns = b.tags(bd)
        assert rc == 0 and uns == 0, (name, rc, _err())
        check_tags(b, g, bd, tok, cand, host_ids)
        if name == "predicted":
            assert not differs(tok, cand, ptok, pcand)
        elif not np.array_equal(bd, b.bounds):
            assert differs(tok, cand, ptok, pcand), name
        out[name] = (tok, cand)
    return out


def set_pattern(b, per_sentence, default):
    """A boundary array that gives sentence i the list per_sentence[i] (None: `default`'s slice)."""
    bd = default.copy()
    for i, v in enumerate(per_sentence):
        if v is not None:
            b0, b1 = int(b.boff[i]), int(b.boff[i + 1])
            assert len(v) == b1 - b0, i
            bd[b0:b1] = v
    return bd


# ---- boundary patterns ------------------------------------------------------------------------------------------

LENGTHS = (1, 31, 32, 33, 64, 65, 100, 160, 257, 300, 517)


@pytest.mark.parametrize("cw,tw,maxdict,tags", [(3, 3, 5, 3), (1, 5, 3, 2), (2, 2, 2, 4)])
def test_random_tag_models(cw, tw, maxdict, tags):
    """The random tag models of test_gpu_tags: ragged text and sentences of LENGTHS characters under every pattern, and
    sentences tiled from the models' own tokens with the tiling as boundaries."""
    rng = np.random.default_rng(4242 + 1000 * cw + 100 * tw + maxdict + tags)
    model, alpha = _random_model(rng, cw, tw, maxdict=maxdict, tags=tags)
    mb = encode_model(model)
    p, g = vb.Predictor(vb.Model.read(mb), predict_tags=True), TagsGivenOracle(mb)
    sents = ["".join(rng.choice(list(alpha), size=int(rng.integers(1, 120)))) for _ in range(300)]
    sents += ["".join(rng.choice(list(alpha), size=n)) for n in LENGTHS]
    toks = [t["token"] for t in model["tag_models"]]
    tilings = [[toks[int(j)] for j in rng.integers(len(toks), size=int(rng.integers(1, 150)))] for _ in range(100)]
    first_tiling = len(sents)
    sents += ["".join(t) for t in tilings]
    text, offs = _batch(sents)
    b = DevBatch(p, text, offs)
    pats = random_patterns(b, rng)
    pats["tiling"] = set_pattern(b, [None] * first_tiling + [token_bounds(t) for t in tilings], pats["bernoulli0.5"])
    out = run_patterns(b, g, pats)
    tok, _ = out["tiling"]
    for k, t in enumerate(tilings):   # every token of a tiling is known
        c0 = int(b.coff[first_tiling + k])
        assert (tok[c0 + np.cumsum([len(x) for x in t]) - 1] >= 0).all()


def test_tag_edges_model():
    """The tag_edges cases with their own token lists as the boundaries, and whole-sentence tokens of LENGTHS
    characters of every UTF-8 width at every start alignment with all boundaries 0, on a copy of the edge model that
    predicts a boundary after every character (bias +1): the model no longer decides the segmentation.  Checked
    against the oracle and by hand (tag_edges.expected_sentence_cands / expected_cands)."""
    cases = te.edge_cases()
    known = set(te.known_tokens(cases))
    wholes = [(te.target_token(w, L) if L > 1 else te.term(w), te.twin_token(w, L) if L > 1 else te.pad(w), w)
              for w in (1, 2, 3, 4) for L in LENGTHS]
    extra = [te.tag_model(t) for t, _, _ in wholes if len(t) > 1 and t not in known]
    known |= {t for t, _, _ in wholes if len(t) > 1}
    mb = encode_model(dict(te.model(cases, extra_tag_models=extra), bias=1))
    p, g = vb.Predictor(vb.Model.read(mb), predict_tags=True), TagsGivenOracle(mb)
    pairs = [(c.sentence, c.align) for c in cases]
    pairs += [(s, a) for t, u, w in wholes for s in (t, u) for a in range(4)]
    sents, idx = te.aligned_batch(pairs)
    text, offs = _batch(sents)
    assert [int(offs[i]) % 4 for i in idx] == [a for _, a in pairs]
    b = DevBatch(p, text, offs)
    assert (b.bounds == 1).all()
    toks = [None] * len(sents)
    for c, i in zip(cases, idx):
        toks[i] = c.tokens
    tiling = set_pattern(b, [None if t is None else token_bounds(t) for t in toks], np.zeros(b.nb, np.uint8))
    out = run_patterns(b, g, {"predicted": b.bounds.copy(), "tiling": tiling, "all0": np.zeros(b.nb, np.uint8)})
    for name in ("tiling", "all0"):
        tok, cand = out[name]
        if name == "tiling":
            for c, i in zip(cases, idx):
                c0, c1 = int(b.coff[i]), int(b.coff[i + 1])
                assert cand[c0:c1].tolist() == te.expected_sentence_cands(c.tokens, known), (c.kind, c.w, c.align)
        for (s, _), i in zip(pairs[len(cases):], idx[len(cases):]):
            c0, c1 = int(b.coff[i]), int(b.coff[i + 1])
            want = te.expected_cands(s, None) if s in known else [-1, -1]
            assert cand[c1 - 1].tolist() == want and (tok[c1 - 1] >= 0) == (s in known), (name, len(s))
            assert (tok[c0:c1 - 1] == -1).all()


@pytest.fixture(scope="module")
def bench_shape(tmp_path_factory):
    """bench.py's config-3 shape: test_gpu_batch_pipeline's workload (1 500 tag models, 20 000 ragged sentences with
    empty, NUL and invalid UTF-8 ones)."""
    d = tmp_path_factory.mktemp("tags_device")
    _workload(d)
    mb = open(d / "model.bin", "rb").read()
    z = np.load(d / "batch.npz")
    p = vb.Predictor(vb.Model.read(mb), predict_tags=True)
    b = DevBatch(p, z["text"], z["offs"])
    assert (b.status != 0).sum() > 20
    return b, TagsGivenOracle(mb)


def test_bench_shape(bench_shape):
    """Every pattern on the bench shape; the predicted one also array for array as predict_batch_tags gives it, and
    twice with identical bytes."""
    b, g = bench_shape
    rng = np.random.default_rng(31)
    out = run_patterns(b, g, random_patterns(b, rng), host_ids=range(0, b.n, 10))
    tok, cand = out["predicted"]
    assert int((tok[: b.nc] >= 0).sum()) > 1000
    res, htok, hcand, hun = b.p.predict_batch_tags(b.text, b.offs)
    assert hun == 0 and res.char_offsets.tolist() == b.coff.tolist() and res.boundaries.tolist() == b.bounds.tolist()
    assert np.array_equal(htok, tok[: b.nc]) and np.array_equal(hcand, cand[: b.nc])
    rc, tok2, cand2, _ = b.tags()
    assert rc == 0 and tok2.tobytes() == tok.tobytes() and cand2.tobytes() == cand.tobytes()


def test_one_moved_boundary_is_seen(bench_shape):
    """Sensitivity of the comparison itself: the oracle given the predicted boundaries with one boundary removed
    disagrees with the device exactly on the two tokens that boundary separates."""
    b, g = bench_shape
    rc, tok, cand, _ = b.tags()
    assert rc == 0
    # a boundary after a known token whose sentence has a token end after it
    for i in range(b.n):
        c0, c1, b0 = int(b.coff[i]), int(b.coff[i + 1]), int(b.boff[i])
        ks = [k for k in range(c1 - c0 - 1) if b.bounds[b0 + k] == 1 and tok[c0 + k] >= 0]
        if b.status[i] == 0 and ks:
            k = ks[0]
            break
    moved = b.bounds.copy()
    moved[b0 + k] = 0
    nxt = next(j for j in range(k + 1, c1 - c0) if j == c1 - c0 - 1 or b.bounds[b0 + j] == 1)
    otok, ocand = g.tags(b.text, b.offs, b.boff, moved, b.coff)
    bad = np.flatnonzero(((tok[: b.nc] >= 0) != (otok >= 0)) | (cand[: b.nc] != ocand).any(axis=1))
    assert c0 + k in bad and set(bad.tolist()) <= {c0 + k, c0 + nxt}, (bad.tolist(), c0 + k, c0 + nxt)


# ---- the call's contract ----------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def small():
    rng = np.random.default_rng(5)
    model, alpha = _random_model(rng, 3, 3, maxdict=5, tags=4)
    mb = encode_model(model)
    sents = ["".join(rng.choice(list(alpha), size=int(rng.integers(1, 90)))) for _ in range(300)]
    sents[7], sents[100], sents[101] = "", "a\0b", "人"
    text, offs = _batch(sents)
    p = vb.Predictor(vb.Model.read(mb), predict_tags=True)
    return mb, p, TagsGivenOracle(mb), text, offs, DevBatch(p, text, offs)


def test_offsets_not_from_zero(small):
    """A slice of a larger device text: d_byte_offsets[0] = 37 with the text pointer 16-byte aligned."""
    mb, p, g, text, offs, b = small
    b37 = DevBatch(p, text, offs, lead=37)
    assert b37.boff.tolist() == b.boff.tolist() and b37.coff.tolist() == b.coff.tolist()
    bd = (np.random.default_rng(1).random(b.nb) < 0.3).astype(np.uint8)
    rc, tok, cand, _ = b37.tags(bd)
    assert rc == 0, _err()
    check_tags(b37, g, bd, tok, cand)
    rc0, tok0, cand0, _ = b.tags(bd)
    assert rc0 == 0 and tok.tobytes() == tok0.tobytes() and cand.tobytes() == cand0.tobytes()


@pytest.mark.parametrize("k,m", [(37, 101), (0, 1), (299, 1), (8, 8)])
def test_sub_batch_by_pointer_offset(small, k, m):
    """Sentences [k, k + m) through pointers into the full batch's arrays, into the full-size outputs: exactly the
    characters [coff[k], coff[k + m]) are written, equal to the full call's."""
    torch = _torch()
    mb, p, g, text, offs, b = small
    rc, ftok, fcand, _ = b.tags()
    assert rc == 0
    nt = p.n_tags
    tok, cand = b.outputs(nt)
    uns = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    rc = vb.lib().vpt_predict_tags_batch_dev(
        p._h, b.d_text.data_ptr(), b.d_off.data_ptr() + 8 * k, m, b.d_status.data_ptr() + 4 * k, b.d_bounds.data_ptr(),
        b.d_boff.data_ptr() + 8 * k, b.d_coff.data_ptr() + 8 * k, b.d_cs.data_ptr(), b.d_ts.data_ptr(), tok.data_ptr(),
        cand.data_ptr(), uns.data_ptr(), _stream_ptr())
    assert rc == 0, _err()
    torch.cuda.synchronize()
    tok, cand = tok.cpu().numpy(), cand.cpu().numpy().reshape(-1, nt)
    c0, c1 = int(b.coff[k]), int(b.coff[k + m])
    assert np.array_equal(tok[c0:c1], ftok[c0:c1]) and np.array_equal(cand[c0:c1], fcand[c0:c1])
    assert (tok[:c0] == SENTINEL).all() and (tok[c1:] == SENTINEL).all()
    assert (cand[:c0] == SENTINEL).all() and (cand[c1:] == SENTINEL).all()


@pytest.mark.parametrize("without", ["char", "type"])
def test_scorer_without_tag_weights(without):
    """A model without a char (type) scorer, so that scorer has no tag weights: its state pointer may be NULL; the
    other one is required."""
    rng = np.random.default_rng(17 if without == "char" else 18)
    model, alpha = _random_model(rng, 3, 3, maxdict=5, tags=4)
    if without == "char":
        model.update(char_ngrams=[], dict=[])
    else:
        model.update(type_ngrams=[])
    for t in model["tag_models"]:
        t["char_ngrams" if without == "char" else "type_ngrams"] = []
    mb = encode_model(model)
    p, g = vb.Predictor(vb.Model.read(mb), predict_tags=True), TagsGivenOracle(mb)
    sents = ["".join(rng.choice(list(alpha), size=int(rng.integers(1, 90)))) for _ in range(200)]
    b = DevBatch(p, *_batch(sents))
    bd = (rng.random(b.nb) < 0.4).astype(np.uint8)
    rc, tok, cand, _ = b.tags(bd, char_states=without != "char", type_states=without != "type")
    assert rc == 0, _err()
    check_tags(b, g, bd, tok, cand)
    assert (tok[: b.nc] >= 0).sum() > 20
    rc, tok, cand, _ = b.tags(bd, char_states=without == "char", type_states=without == "type")
    assert rc == INVALID and _err() == "InvalidArgumentError: states: required for tag prediction"
    assert (tok == SENTINEL).all() and (cand == SENTINEL).all()


def test_unserved_tokens():
    """A token whose own tag model has 65 scores (beyond the device tables): every token end of it is counted in
    d_unserved and left -1; the other tokens are tagged as the oracle tags them.  d_unserved may be NULL."""
    big = dict(token="人", tags=[["c%d" % i for i in range(65)]], char_ngrams=[("人", [(0, list(range(65)))])],
               type_ngrams=[], bias=[(-1) ** i * i for i in range(65)])
    small_ = dict(token="火", tags=[["x", "y"]], char_ngrams=[("人火", [(0, [3, -4])])], type_ngrams=[], bias=[5, 4])
    model = dict(char_ngrams=[("人火", [1, -50, 2, 3])], type_ngrams=[], dict=[("人", [99, 99], "")], bias=-10,
                 char_window=2, type_window=0, tag_models=[big, small_])
    mb = encode_model(model)
    p, g = vb.Predictor(vb.Model.read(mb), predict_tags=True), TagsGivenOracle(mb)
    sents = ["人火人", "火", "火人火火", "人"]
    b = DevBatch(p, *_batch(sents))
    ones = np.ones(b.nb, np.uint8)
    at = [i for i, c in enumerate("".join(sents)) if c == "人"]
    rc, tok, cand, uns = b.tags(ones)
    assert rc == 0 and uns == len(at) == 4, (rc, uns)
    check_tags(b, g, ones, tok, cand, unserved_at=at)
    assert (tok[: b.nc] >= 0).sum() == b.nc - len(at)
    rc, tok2, cand2, _ = b.tags(ones, unserved=False)
    assert rc == 0 and tok2.tobytes() == tok.tobytes() and cand2.tobytes() == cand.tobytes()


def test_model_beyond_the_device_limits():
    """Nine tag slots: the whole model is beyond the device path, VPT_UNSUPPORTED, nothing written."""
    tm = dict(token="人", tags=[["a", "b"]] * 9, char_ngrams=[], type_ngrams=[], bias=list(range(18)))
    model = dict(char_ngrams=[("人", [1, -2])], type_ngrams=[], dict=[], bias=-1, char_window=1, type_window=0,
                 tag_models=[tm])
    p = vb.Predictor(vb.Model.read(encode_model(model)), predict_tags=True)
    b = DevBatch(p, *_batch(["人人", "火人"]))
    rc, tok, cand, uns = b.tags()
    assert rc == UNSUPPORTED, rc
    assert "exceeds the limits of the device path" in _err()
    assert (tok == SENTINEL).all() and (cand == SENTINEL).all() and uns == 0


def test_rejections(small):
    """Each refusal returns VPT_INVALID_ARGUMENT with its message and writes nothing; a batch of no sentences returns 0
    and writes nothing."""
    torch = _torch()
    mb, p, g, text, offs, b = small
    nt = p.n_tags

    def untouched(res):
        rc, tok, cand, uns = res
        assert (tok == SENTINEL).all() and (cand == SENTINEL).all() and uns == 0
        return rc

    msg = "InvalidArgumentError: this predictor is created with predict_tags = false"
    for q in (vb.Predictor(vb.Model.read(mb), predict_tags=False), vb.Predictor.from_blob(p.export_blob())):
        assert untouched(b.tags(predictor=q)) == INVALID and _err() == msg
    # a text pointer that is 4-byte but not 16-byte aligned (the allocation has 64 bytes of padding)
    assert untouched(b.tags(text_shift=4)) == INVALID
    assert _err() == "InvalidArgumentError: d_utf8: must be 16-byte aligned"
    assert untouched(b.tags(n_sent=0)) == 0
    # each device buffer NULL in turn
    L = vb.lib()
    for which in range(8):
        tok, cand = b.outputs(nt)
        uns = torch.zeros(1, dtype=torch.int32, device="cuda:0")
        args = [b.d_text.data_ptr(), b.d_off.data_ptr(), b.n, b.d_status.data_ptr(), b.d_bounds.data_ptr(),
                b.d_boff.data_ptr(), b.d_coff.data_ptr(), b.d_cs.data_ptr(), b.d_ts.data_ptr(), tok.data_ptr(),
                cand.data_ptr(), uns.data_ptr()]
        args[[0, 1, 3, 4, 5, 6, 9, 10][which]] = None
        rc = L.vpt_predict_tags_batch_dev(p._h, *args, _stream_ptr())
        torch.cuda.synchronize()
        assert rc == INVALID and _err() == "InvalidArgumentError: device buffers: must not be NULL", which
        assert untouched((rc, tok.cpu().numpy(), cand.cpu().numpy(), int(uns.item()))) == INVALID
    rc = L.vpt_predict_tags_batch_dev(None, b.d_text.data_ptr(), b.d_off.data_ptr(), b.n, b.d_status.data_ptr(),
                                      b.d_bounds.data_ptr(), b.d_boff.data_ptr(), b.d_coff.data_ptr(), b.d_cs.data_ptr(),
                                      b.d_ts.data_ptr(), None, None, None, _stream_ptr())
    assert rc == INVALID and _err() == "InvalidArgumentError: predictor: must not be NULL"


def test_caller_stream(small):
    """Both calls on a side stream with nothing between them: correct once that stream is synchronised."""
    torch = _torch()
    mb, p, g, text, offs, b = small
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        bs = DevBatch(p, text, offs, stream=side)
        out = b.outputs(p.n_tags)   # (sized from the same batch scored on the default stream)
        rc = vb.lib().vpt_predict_tags_batch_dev(
            p._h, bs.d_text.data_ptr(), bs.d_off.data_ptr(), bs.n, bs.d_status.data_ptr(), bs.d_bounds.data_ptr(),
            bs.d_boff.data_ptr(), bs.d_coff.data_ptr(), bs.d_cs.data_ptr(), bs.d_ts.data_ptr(), out[0].data_ptr(),
            out[1].data_ptr(), None, _stream_ptr(side))
        assert rc == 0, _err()
    side.synchronize()
    tok, cand = out[0].cpu().numpy(), out[1].cpu().numpy().reshape(-1, p.n_tags)
    bs.fetch()
    assert bs.bounds.tolist() == b.bounds.tolist() and bs.coff.tolist() == b.coff.tolist()
    check_tags(bs, g, bs.bounds, tok, cand)


# ---- vpt_predict_batch_dev_profiled -----------------------------------------------------------------------------

def _recipe(name):
    return next(r for r in tle.variant_recipes() if r[0] == name)


def _profiled_models():
    """(id, model bytes, predict_tags, states, kernel, text alphabet, long words): one model per kind of scoring kernel,
    with and without states where the kernel serves both, and the config-2 model shape."""
    out = []
    for name in ("fused-smem-common-deep1-plain", "fused-smem-common-deep1-states", "tile-smem-split3-inline",
                 "tile-smem-nosplit-general"):
        _, budget, args, tags, states, key = _recipe(name)
        assert budget is None
        mb, words = tle.variant_model(*args)
        out.append((name, mb, tags, states, key[0], tle.ALPHABET, words))
    for name, args, tags, states, key in nv.SCORE_KERNELS:
        if "tw4" in name:
            continue
        mb, words = nv.norm_model(*args)
        out.append((name, mb, tags, states, key[0], nv.TEXT_ALPHABET, words))
    out.append(("config2", synth.gen_model_bccwj_shaped(n_patterns=30_000, sample_sentences=50_000), False, False,
                "k_fused", None, None))
    return out


PROFILED = _profiled_models()


def _profiled_text(alphabet, words, rng):
    if alphabet is None:
        text, offs, _ = synth.gen_text(20_000, 40, seed=synth.TEXT_SEED + 47, ragged=True)
        sents = [bytes(text[int(offs[i]):int(offs[i + 1])]) for i in range(len(offs) - 1)]
    else:
        sents = nv.text_for(words, 3_000, rng, lo=1, hi=150) if alphabet is nv.TEXT_ALPHABET else \
            ["".join(rng.choice(list(alphabet), size=int(rng.integers(1, 150)))) +
             (words[i % len(words)] if words and i % 3 == 0 else "") for i in range(3_000)]
        sents = [s.encode() for s in sents]
    sents[11], sents[12], sents[13] = b"", "a\0b".encode(), b"\xe3\x81"
    return _batch(sents)


@pytest.mark.parametrize("name,mb,tags,states,kernel,alphabet,words", PROFILED, ids=[m[0] for m in PROFILED])
def test_profiled_equals_plain(name, mb, tags, states, kernel, alphabet, words):
    """vpt_predict_batch_dev_profiled writes the bytes vpt_predict_batch_dev writes (scores, boundaries, both offset
    arrays, status, states), both equal to the oracle; stage_ms holds three finite times >= 0."""
    torch = _torch()
    p = vb.Predictor(vb.Model.read(mb), predict_tags=tags)
    assert p.kernel_plan(states)["kernel"] == kernel
    text, offs = _profiled_text(alphabet, words, np.random.default_rng(len(name)))
    n, nbytes = len(offs) - 1, int(offs[-1])
    dev = torch.device("cuda:0")
    d_text = torch.zeros(nbytes + 64, dtype=torch.uint8, device=dev)
    d_text[:nbytes] = torch.from_numpy(text.copy()).to(dev)
    d_off = torch.from_numpy(offs.astype(np.int64)).to(dev)
    ws = torch.empty(vb.lib().vpt_workspace_size(n), dtype=torch.uint8, device=dev)

    def run(profiled):
        o = dict(scores=torch.full((nbytes,), SENTINEL, dtype=torch.int32, device=dev),
                 boundaries=torch.full((nbytes,), 0xA5, dtype=torch.uint8, device=dev),
                 bound_offsets=torch.full((n + 1,), SENTINEL, dtype=torch.int64, device=dev),
                 status=torch.full((n,), SENTINEL, dtype=torch.int32, device=dev),
                 char_states=torch.full((nbytes,), SENTINEL, dtype=torch.int32, device=dev) if states else None,
                 type_states=torch.full((nbytes,), SENTINEL, dtype=torch.int32, device=dev) if states else None,
                 char_offsets=torch.full((n + 1,), SENTINEL, dtype=torch.int64, device=dev))
        ptrs = [None if o[k] is None else o[k].data_ptr() for k in ("scores", "boundaries", "bound_offsets", "status",
                                                                      "char_states", "type_states", "char_offsets")]
        args = [p._h, d_text.data_ptr(), d_off.data_ptr(), n, ws.data_ptr(), ws.numel(), *ptrs, _stream_ptr()]
        stage = (C.c_float * 3)(-1.0, -1.0, -1.0)
        rc = vb.lib().vpt_predict_batch_dev_profiled(*args, stage) if profiled else vb.lib().vpt_predict_batch_dev(*args)
        assert rc == 0, _err()
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in o.items() if v is not None}, list(stage)

    plain, _ = run(False)
    prof, stage = run(True)
    assert sorted(plain) == sorted(prof)
    for k in plain:
        assert plain[k].tobytes() == prof[k].tobytes(), k
    assert all(math.isfinite(x) and x >= 0 for x in stage), stage
    o = OraclePredictor(mb, predict_tags=tags)
    sc, bd, boff, st = o.predict_batch(text, offs, nthreads=8)
    nb = int(boff[-1])
    assert prof["bound_offsets"].astype(np.uint64).tolist() == boff.tolist()
    assert ((prof["status"] != 0) == (st != 0)).all() and (st != 0).sum() == 3
    assert np.array_equal(prof["scores"][:nb], sc) and np.array_equal(prof["boundaries"][:nb], bd)
    if states:
        cs, ts, coff = o.predict_batch_states(text, offs, nthreads=8)
        nc = int(coff[-1])
        assert prof["char_offsets"].astype(np.uint64).tolist() == coff.tolist()
        assert np.array_equal(prof["char_states"][:nc].view(np.uint32), cs)
        assert np.array_equal(prof["type_states"][:nc].view(np.uint32), ts)
    # stage_ms is required; a batch of no sentences returns 0 with three zero times
    args = [p._h, d_text.data_ptr(), d_off.data_ptr(), n, ws.data_ptr(), ws.numel()] + [None] * 7 + [_stream_ptr()]
    assert vb.lib().vpt_predict_batch_dev_profiled(*args, None) == INVALID
    assert _err() == "InvalidArgumentError: stage_ms: must not be NULL"
    stage = (C.c_float * 3)(-1.0, -1.0, -1.0)
    args[3] = 0
    assert vb.lib().vpt_predict_batch_dev_profiled(*args, stage) == 0
    assert list(stage) == [0.0, 0.0, 0.0]
