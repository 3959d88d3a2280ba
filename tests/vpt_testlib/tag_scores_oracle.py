"""CPU oracle of the tag candidate scores of the compact and spans calls (tests/native/tag_scores_oracle.cpp: the oracle's
fill_tags raw scores per token record), a host build of the kernels' own score code (tests/native/tag_scores_emul.cpp),
and a literal Python restatement of Token::tag_candidates.

TEST INFRASTRUCTURE ONLY.  The libraries are compiled once per source state into the temporary directory (the tree may
be read-only)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from . import oracle
from .spans_oracle import wsconst_mask

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_NATIVE = os.path.join(_ROOT, "tests", "native")
_CSRC = os.path.join(_ROOT, "vaporetto_b200", "csrc")
_CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")


def _build(tag, srcs, deps, flags=()):
    h = hashlib.sha256()
    for f in srcs + deps:
        h.update(open(f, "rb").read())
    so = os.path.join(tempfile.gettempdir(), f"vpt_{tag}_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", *flags, "-o", tmp] + srcs)
        os.replace(tmp, so)
    return C.CDLL(so)


_ora = None


def ora_lib():
    global _ora
    if _ora is None:
        L = _build("tag_scores_oracle", [os.path.join(_NATIVE, "tag_scores_oracle.cpp")],
                   [os.path.join(_NATIVE, "spans_oracle.cpp"), os.path.join(_ROOT, "oracle", "vaporetto_oracle.cpp"),
                    os.path.join(_ROOT, "oracle", "grapheme_tables.hpp")])
        L.ora_last_error.restype = C.c_char_p
        L.ora_model_read.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
        L.ora_model_free.argtypes = [C.c_void_p]
        L.ora_predictor_new.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
        L.ora_predictor_free.argtypes = [C.c_void_p]
        L.ora_predictor_n_tags.argtypes = [C.c_void_p]
        L.ora_compact_tag_scores.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                             C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.ora_spans_tag_scores.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_uint32,
                                           C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64),
                                           C.POINTER(C.c_uint64)]
        _ora = L
    return _ora


class TagScoresOracle:
    """Model::read + Predictor::new(model, true), then per token record of a batch: the token id and, for an id >= 0,
    its score vector, for the compact chain and the spans chain."""

    def __init__(self, model_bytes: bytes):
        L = ora_lib()
        m = C.c_void_p()
        consumed = C.c_size_t()
        rc = L.ora_model_read(model_bytes, len(model_bytes), C.byref(m), C.byref(consumed))
        if rc:
            raise oracle.OracleError(rc, L.ora_last_error().decode())
        p = C.c_void_p()
        rc = L.ora_predictor_new(m, 1, C.byref(p))
        L.ora_model_free(m)
        if rc:
            raise oracle.OracleError(rc, L.ora_last_error().decode())
        self._p = p
        self.n_tags = L.ora_predictor_n_tags(p)

    def __del__(self):
        if getattr(self, "_p", None):
            ora_lib().ora_predictor_free(self._p)
            self._p = None

    def _run(self, fn, text, offsets, *args):
        t = np.frombuffer(bytes(text), np.uint8) if isinstance(text, (bytes, bytearray)) else np.ascontiguousarray(text, np.uint8)
        off = np.ascontiguousarray(offsets, np.uint64)
        cap = max(int(off[-1] - off[0]) if off.size > 1 else 0, 1)
        scap = cap * 8
        while True:
            ids = np.zeros(cap, np.int32)
            sc = np.zeros(scap, np.int32)
            nr, ns = C.c_uint64(), C.c_uint64()
            rc = fn(self._p, t.ctypes.data, off.ctypes.data, off.size - 1, *args, ids.ctypes.data, cap, sc.ctypes.data, scap,
                    C.byref(nr), C.byref(ns))
            if rc == 2:
                cap, scap = max(cap, nr.value), max(scap, ns.value)
                continue
            if rc:
                raise oracle.OracleError(rc, ora_lib().ora_last_error().decode())
            return ids[: nr.value].copy(), sc[: ns.value].copy()

    def compact(self, text, offsets):
        """-> (token ids, concatenated score vectors) of predict + fill_tags on every sentence's raw text."""
        return self._run(ora_lib().ora_compact_tag_scores, text, offsets)

    def spans(self, text, offsets, no_norm: bool = False, wsconst: str = ""):
        """-> (token ids, concatenated score vectors) of token_stream's chain with fill_tags on the filtered sentence."""
        return self._run(ora_lib().ora_spans_tag_scores, text, offsets, int(no_norm), wsconst_mask(wsconst))


_emul = None


def emul_lib():
    global _emul
    if _emul is None:
        srcs = [os.path.join(_NATIVE, "tag_scores_emul.cpp"), os.path.join(_NATIVE, "host_emul.cpp")] + \
               [os.path.join(_CSRC, f) for f in ("predictor_build.cpp", "builder.cpp", "model.cpp", "tags_build.cpp")]
        deps = [os.path.join(_CSRC, f) for f in ("builder.hpp", "keys.hpp", "predictor_build.hpp", "common.hpp", "tags.hpp",
                                                  "tags_token.hpp", "textnorm.hpp")]
        L = _build("tag_scores_emul", srcs, deps, ("-I" + _CUDA_INC,))
        L.emul_predict.restype = C.c_long
        L.emul_predict.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_char_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p]
        L.emul_last_error.restype = C.c_char_p
        L.emul_tag_scores.restype = C.c_long
        L.emul_tag_scores.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64)]
        _emul = L
    return _emul


def tag_candidates(tags, scores):
    """Token::tag_candidates (sentence.rs:1219-1250) restated: `tags` = the token's own tag model (a list of candidate
    lists, one per slot), `scores` = its score vector.  A one-candidate slot gives (tag, 0) and consumes no score, an
    empty slot gives [], a slot of two or more candidates gives (tag, score) pairs from the next scores in order."""
    out, i = [], 0
    for cands in tags:
        if len(cands) == 1:
            out.append([(cands[0], 0)])
        else:
            out.append([(c, int(scores[i + j])) for j, c in enumerate(cands)])
            i += len(cands)
    return out


def first_max(v):
    """Index of the first strict maximum (TagPredictor::predict, predictor.rs:286-304)."""
    best, mx = 0, None
    for j, x in enumerate(v):
        if mx is None or x > mx:
            best, mx = j, x
    return best
