"""CPU oracle of vpt_reannotate_lines (tests/native/reannotate_oracle.cpp: the chain of the C header composed from the
restatements of partial_oracle.cpp and annotate_oracle.cpp, over the oracle's Sentence and Predictor), and the host
build of tests/native/reannotate_tags_test.cpp.

TEST INFRASTRUCTURE ONLY.  The libraries are compiled once per source state into the temporary directory (the tree may
be read-only)."""
from __future__ import annotations

import ctypes as C
import os
import struct

from . import oracle
from .annotate_oracle import _slots
from .partial_oracle import _build
from .spans_oracle import wsconst_mask

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_NATIVE = os.path.join(_ROOT, "tests", "native")
_ORACLE = [os.path.join(_ROOT, "oracle", "vaporetto_oracle.cpp"), os.path.join(_ROOT, "oracle", "grapheme_tables.hpp")]
_SRCS = [os.path.join(_NATIVE, "reannotate_oracle.cpp"), os.path.join(_NATIVE, "partial_oracle.cpp"),
         os.path.join(_NATIVE, "annotate_oracle.cpp")] + _ORACLE
_TEST_SRCS = [os.path.join(_NATIVE, "reannotate_tags_test.cpp"), os.path.join(_NATIVE, "partial_oracle.cpp"),
              os.path.join(_ROOT, "vaporetto_b200", "csrc", "partial_parse.hpp"),
              os.path.join(_ROOT, "vaporetto_b200", "csrc", "common.hpp")] + _ORACLE


def lib():
    L = _build("reannotate_oracle", _SRCS)
    L.ora_last_error.restype = C.c_char_p
    L.ora_model_read.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
    L.ora_model_free.argtypes = [C.c_void_p]
    L.ora_predictor_new.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
    L.ora_predictor_free.argtypes = [C.c_void_p]
    L.ora_predictor_n_tags.argtypes = [C.c_void_p]
    L.ora_reannotate_lines.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int, C.c_uint32, C.c_int, C.c_int32,
                                       C.c_int, C.c_char_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_uint64),
                                       C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    return L


def tags_test_lib():
    """tests/native/reannotate_tags_test.cpp: partial_parse.hpp's tag regions against the restatement."""
    L = _build("reannotate_tags_test", _TEST_SRCS, "-O2")
    L.rt_check_all.restype = C.c_long
    L.rt_check_all.argtypes = [C.c_int, C.c_char_p, C.c_size_t]
    return L


def rules_blob(rules) -> bytes:
    """{surface: [tag or None]} in ora_annotate_lines' layout."""
    blob = struct.pack("<I", len(rules))
    for k, v in rules.items():
        kb = k.encode()
        blob += struct.pack("<I", len(kb)) + kb + _slots(v)
    return blob


class ReannotateOracle:
    """Model::read + Predictor::new + the chain of vpt_reannotate_lines, on the CPU."""

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

    def lines(self, data: bytes, margin: int = 0, keep_tags: bool = True, no_norm: bool = False, wsconst: str = "",
              predict_tags: bool = False, rules=None):
        """-> (output bytes, n_lines), or raises oracle.OracleError (code 2 or 5) whose .message is the library's error
        text and .output the output of the lines before the bad one.  `rules` ({surface: [tag or None]}):
        PatternMatchTagger after fill_tags, as AnnotateOracle.lines."""
        L = lib()
        blob = rules_blob(rules) if rules and predict_tags else None
        cap = 3 * len(data) + 16
        for _ in range(2):
            buf = C.create_string_buffer(cap)
            n, nl, el = C.c_uint64(), C.c_uint64(), C.c_uint64()
            rc = L.ora_reannotate_lines(self._p, data, len(data), int(no_norm), wsconst_mask(wsconst), int(predict_tags),
                                        margin, int(keep_tags), blob, buf, cap, C.byref(n), C.byref(nl), C.byref(el))
            if rc == 99:
                cap = n.value + 16
                continue
            break
        if rc:
            e = oracle.OracleError(rc, L.ora_last_error().decode())
            e.message, e.output = L.ora_last_error().decode(), buf.raw[: n.value]
            raise e
        return buf.raw[: n.value], int(nl.value)
