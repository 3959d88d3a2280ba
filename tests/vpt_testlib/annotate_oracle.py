"""CPU oracle of vpt_annotate_lines (tests/native/annotate_oracle.cpp: Sentence::write_partial_annotation_text and
TokenIterator restated, and the chain of the C header over the oracle's Sentence and Predictor).

TEST INFRASTRUCTURE ONLY.  The library is compiled once per source state into the temporary directory (the tree may be
read-only)."""
from __future__ import annotations

import ctypes as C
import os
import struct

from . import oracle
from .partial_oracle import _build
from .spans_oracle import wsconst_mask

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_SRCS = [os.path.join(_ROOT, "tests", "native", "annotate_oracle.cpp"),
         os.path.join(_ROOT, "oracle", "vaporetto_oracle.cpp"), os.path.join(_ROOT, "oracle", "grapheme_tables.hpp")]


def lib():
    L = _build("annotate_oracle", _SRCS)
    L.ora_last_error.restype = C.c_char_p
    L.ora_model_read.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
    L.ora_model_free.argtypes = [C.c_void_p]
    L.ora_predictor_new.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
    L.ora_predictor_free.argtypes = [C.c_void_p]
    L.ora_predictor_n_tags.argtypes = [C.c_void_p]
    L.ora_write_partial_annotation.restype = C.c_long
    L.ora_write_partial_annotation.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t]
    L.ora_annotate_lines.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int, C.c_uint32, C.c_int, C.c_int32,
                                     C.c_char_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    return L


def _slots(tags) -> bytes:
    out = struct.pack("<I", len(tags))
    for t in tags:
        if t is None:
            out += struct.pack("<i", -1)
        else:
            b = t.encode()
            out += struct.pack("<I", len(b)) + b
    return out


def write(text: str, boundaries, tags=None) -> str:
    """write_partial_annotation_text of a sentence: its text, boundaries (0 / 1 / 2) and, optionally, the tag slots of
    every character ([[tag or None]] per character)."""
    b = text.encode()
    blob = b"".join(_slots(t) for t in tags) if tags is not None else None
    cap = 8 * len(b) + 256 + (len(blob) if blob else 0)
    buf = C.create_string_buffer(cap)
    n = lib().ora_write_partial_annotation(b, len(b), bytes(boundaries), blob, buf, cap)
    assert n >= 0
    return buf.raw[:n].decode()


class AnnotateOracle:
    """Model::read + Predictor::new + the chain of vpt_annotate_lines, on the CPU."""

    def __init__(self, model_bytes: bytes, predict_tags: bool = False):
        L = lib()
        m = C.c_void_p()
        consumed = C.c_size_t()
        rc = L.ora_model_read(model_bytes, len(model_bytes), C.byref(m), C.byref(consumed))
        if rc:
            raise oracle.OracleError(rc, L.ora_last_error().decode())
        p = C.c_void_p()
        rc = L.ora_predictor_new(m, int(predict_tags), C.byref(p))
        L.ora_model_free(m)
        if rc:
            raise oracle.OracleError(rc, L.ora_last_error().decode())
        self._p = p
        self.n_tags = L.ora_predictor_n_tags(p)

    def __del__(self):
        if getattr(self, "_p", None):
            lib().ora_predictor_free(self._p)
            self._p = None

    def lines(self, data: bytes, margin: int = 0, no_norm: bool = False, wsconst: str = "", predict_tags: bool = False,
              rules=None):
        """-> (output bytes, n_lines).  `rules` ({surface: [tag or None]}): PatternMatchTagger after fill_tags, keyed by
        the KyteaFullwidthFilter image of a token unless no_norm."""
        L = lib()
        blob = None
        if rules and predict_tags:
            blob = struct.pack("<I", len(rules))
            for k, v in rules.items():
                kb = k.encode()
                blob += struct.pack("<I", len(kb)) + kb + _slots(v)
        cap = 3 * len(data) + 16
        for _ in range(2):
            buf = C.create_string_buffer(cap)
            n, nl = C.c_uint64(), C.c_uint64()
            rc = L.ora_annotate_lines(self._p, data, len(data), int(no_norm), wsconst_mask(wsconst), int(predict_tags),
                                      margin, blob, buf, cap, C.byref(n), C.byref(nl))
            if rc == 99:
                cap = n.value + 16
                continue
            break
        if rc:
            raise oracle.OracleError(rc, L.ora_last_error().decode())
        return buf.raw[: n.value], int(nl.value)
