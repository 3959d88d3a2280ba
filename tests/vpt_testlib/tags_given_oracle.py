"""CPU oracle of vpt_predict_tags_batch_dev (tests/native/tags_given_oracle.cpp): the reference's predict_tags on the
caller's 0 / 1 boundaries, over the oracle's Sentence and Predictor.

TEST INFRASTRUCTURE ONLY.  The library is compiled once per source state into the temporary directory (the tree may be
read-only), by partial_oracle's builder."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import oracle
from .partial_oracle import _build

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_SRCS = [os.path.join(_ROOT, "tests", "native", "tags_given_oracle.cpp"),
         os.path.join(_ROOT, "oracle", "vaporetto_oracle.cpp"), os.path.join(_ROOT, "oracle", "grapheme_tables.hpp")]


def lib():
    L = _build("tags_given_oracle", _SRCS)
    L.ora_last_error.restype = C.c_char_p
    L.ora_model_read.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
    L.ora_model_free.argtypes = [C.c_void_p]
    L.ora_predictor_new.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
    L.ora_predictor_free.argtypes = [C.c_void_p]
    L.ora_predictor_n_tags.argtypes = [C.c_void_p]
    L.ora_tags_given.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p]
    return L


def char_offsets(text, offs) -> np.ndarray:
    """Characters per sentence as a prefix (lead bytes of valid UTF-8; what the device counts for a scored sentence)."""
    t = np.asarray(text, np.uint8)
    lead = np.concatenate(([0], np.cumsum((t & 0xC0) != 0x80)))
    return lead[np.asarray(offs, np.int64)] - lead[int(offs[0])]


def bound_offsets(coff) -> np.ndarray:
    """max(n_chars - 1, 0) per sentence as a prefix."""
    nb = np.maximum(np.diff(np.asarray(coff, np.int64)), 1) - 1
    return np.concatenate(([0], np.cumsum(nb)))


class TagsGivenOracle:
    """Model::read + Predictor::new(model, true) + predict_tags on given boundaries, on the CPU."""

    def __init__(self, model_bytes: bytes):
        L = lib()
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
            lib().ora_predictor_free(self._p)
            self._p = None

    def tags(self, text, offs, boff, boundaries, coff):
        """-> (tag_token [chars] int32, tag_cand [chars, n_tags] int32) of the batch `text` / `offs` whose sentence i
        has the boundaries boundaries[boff[i] ..] (None: the predicted ones) and the characters [coff[i], coff[i+1])."""
        t = np.ascontiguousarray(text, np.uint8)
        o = np.ascontiguousarray(offs, np.uint64)
        bo = np.ascontiguousarray(boff, np.uint64)
        co = np.ascontiguousarray(coff, np.uint64)
        bd = None if boundaries is None else np.ascontiguousarray(boundaries, np.uint8)
        nc = int(co[-1])
        tok = np.full(max(nc, 1), -2, np.int32)
        cand = np.full(max(nc * self.n_tags, 1), -2, np.int32)
        rc = lib().ora_tags_given(self._p, t.ctypes.data, o.ctypes.data, o.size - 1, bo.ctypes.data,
                                  None if bd is None else bd.ctypes.data, co.ctypes.data, tok.ctypes.data,
                                  cand.ctypes.data)
        if rc:
            raise oracle.OracleError(rc, lib().ora_last_error().decode())
        return tok[:nc], cand[: nc * self.n_tags].reshape(nc, self.n_tags)
