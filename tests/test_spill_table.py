"""The dense node table with a spill table (keys.hpp: slot_of_seeds, builder.cpp: place_keys): inline-format char tables
whose seeds fit the shared-memory budget are placed at a load of 0.75, and the buckets no seed places there go to a
sparse spill table behind the primary slots.  Checked on text made of the n-grams whose records sit in spill slots:
through the host emulator of the kernels' probe sequence (CPU), and through k_fused and k_tile_fast (GPU), against
the oracle.  Probes that ignored the spill seed would miss those records and change the scores."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from vpt_testlib import synth
from vpt_testlib.bincode_model import encode_model
from vpt_testlib.oracle import OraclePredictor

from test_host_tables import emul  # noqa: F401  (fixture: tests/native/host_emul.cpp)

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "vaporetto_b200", "csrc")

ALPHA = [chr(c) for c in range(0x4E00, 0x4E00 + 300)] + [chr(c) for c in range(0x3041, 0x3041 + 40)]


def mid_model(n_patterns, cw, lens, seed):
    """Random char n-grams of the given lengths over ALPHA (rows as wide as the window allows), all type 1-3-grams."""
    rng = np.random.default_rng(seed)
    ng = {}
    while len(ng) < n_patterns:
        n = int(rng.choice(lens))
        ng["".join(rng.choice(ALPHA, size=n))] = rng.integers(-3000, 3000, size=2 * cw - n + 1).tolist()
    tng = {bytes(1 + (k // 6 ** j) % 6 for j in range(n)): rng.integers(-3000, 3000, size=7 - n).tolist()
           for n in (1, 2, 3) for k in range(6 ** n)}
    return encode_model(dict(char_ngrams=list(ng.items()), type_ngrams=list(tng.items()), dict=[],
                             bias=int(rng.integers(-500, 500)), char_window=cw, type_window=3, tag_models=[]))


MODELS = {
    "mid-20k-w3": lambda: mid_model(20_000, 3, (1, 2, 3), seed=11),
    "mid-60k-w3": lambda: mid_model(60_000, 3, (2, 3), seed=12),
    "mid-40k-w4": lambda: mid_model(40_000, 4, (3, 4, 5), seed=13),   # inline rows at r0 = -4: k_tile_fast
}


@pytest.fixture(scope="module")
def spill_lib():
    so = os.path.join(HERE, "native", "libspill_table.so")
    srcs = [os.path.join(HERE, "native", "spill_table.cpp")] + [os.path.join(CSRC, f) for f in
                                                                ("predictor_build.cpp", "builder.cpp", "model.cpp")]
    deps = srcs + [os.path.join(CSRC, f) for f in ("builder.hpp", "keys.hpp", "predictor_build.hpp", "common.hpp")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so] + srcs)
    L = C.CDLL(so)
    L.spill_char_table.restype = C.c_long
    L.spill_char_table.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t]
    return L


def char_table(L, mb):
    """(geometry dict, [(c1, c2, c3)] of the nodes of <= 3 symbols whose records sit in spill slots)."""
    out = np.zeros(7, np.uint64)
    cap = 1 << 20
    syms = np.zeros(3 * cap, np.uint32)
    n = L.spill_char_table(mb, len(mb), out.ctypes.data, syms.ctypes.data, cap)
    assert n >= 0, n
    g = dict(zip(("nodes", "seed_bits", "nslots", "nbuckets", "spill_slots", "spill_buckets", "spilled"), map(int, out)))
    return g, [tuple(int(x) for x in syms[3 * i: 3 * i + 3]) for i in range(n)]


def spill_sentences(nodes, n_sent, seed):
    """Sentences of 6-10 spilled node strings each, with a random character between some of them."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_sent):
        parts = []
        for _ in range(int(rng.integers(6, 11))):
            parts.append("".join(chr(c) for c in nodes[int(rng.integers(len(nodes)))] if c))
            if rng.integers(2):
                parts.append(ALPHA[int(rng.integers(len(ALPHA)))])
        out.append("".join(parts))
    return out


@pytest.fixture(scope="module")
def config2_model():
    return synth.gen_model_bccwj_shaped(n_patterns=300_000, sample_sentences=2_000_000)


def check_layout(g, spilled):
    assert g["seed_bits"] == 8
    assert g["nslots"] <= g["nodes"] / 0.75 + 1                             # primary slots: all nodes at a load of 0.75
    assert g["spill_slots"] > 0 and g["spilled"] > 0 and len(spilled) > 0
    assert g["nbuckets"] + g["spill_buckets"] <= 37632                      # both seed arrays fit the shared-memory budget
    assert g["spill_slots"] < g["nslots"]


def emul_scores(L, mb, text):
    b = text.encode()
    sc = np.zeros(len(b) + 1, np.int32)
    info = np.zeros(4, np.int32)
    n = L.emul_predict(mb, len(mb), 0, b, len(b), sc.ctypes.data, None, None, info.ctypes.data)
    assert n > 0, L.emul_last_error()
    assert info[0] == 1  # inline format
    return sc[: n - 1]


@pytest.mark.parametrize("name", ["config2"] + sorted(MODELS))
def test_spilled_ngrams_on_the_host(emul, spill_lib, name, request):
    mb = request.getfixturevalue("config2_model") if name == "config2" else MODELS[name]()
    g, spilled = char_table(spill_lib, mb)
    check_layout(g, spilled)
    if name == "config2":
        assert g["nodes"] == 300_000 and (g["nslots"] + g["spill_slots"]) * 32 < 0.8 * 22.9e6
    o = OraclePredictor(mb)
    for text in spill_sentences(spilled, 40, seed=len(name)):
        sc, _ = o.predict(text)
        assert emul_scores(emul, mb, text).tolist() == sc.tolist(), text


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["config2"] + sorted(MODELS))
def test_spilled_ngrams_on_the_device(spill_lib, name, request):
    import vaporetto_b200 as vb
    mb = request.getfixturevalue("config2_model") if name == "config2" else MODELS[name]()
    g, spilled = char_table(spill_lib, mb)
    check_layout(g, spilled)
    p = vb.Predictor(vb.Model.read(mb))
    plan = p.kernel_plan()
    assert plan["seeds_smem"] == 1
    assert plan["kernel"] == ("k_tile_fast" if name.endswith("w4") else "k_fused"), plan
    o = OraclePredictor(mb)
    sents = [s.encode() for s in spill_sentences(spilled, 20_000, seed=len(name) + 1)]
    text = np.frombuffer(b"".join(sents), np.uint8)
    offs = np.zeros(len(sents) + 1, np.uint64)
    np.cumsum([len(s) for s in sents], out=offs[1:])
    r = p.predict_batch(text, offs)
    sc, bd, _, _ = o.predict_batch(text, offs, nthreads=8)
    assert np.array_equal(r.scores, sc) and np.array_equal(r.boundaries, bd)
    # the model's own synthetic text too (mostly primary-table probes, and absent keys)
    if name == "config2":
        text, offs, _ = synth.gen_text(20_000, 40)
        r = p.predict_batch(text, offs)
        sc, bd, _, _ = o.predict_batch(text, offs, nthreads=8)
        assert np.array_equal(r.scores, sc) and np.array_equal(r.boundaries, bd)
