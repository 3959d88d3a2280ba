"""CPU oracle of vpt_tokenize_dev (tests/native/tokenize_doc_oracle.cpp: per document, Sentence::from_raw of the whole
document, the filters, fill_tags and write_tokenized_text over the oracle's Sentence and Predictor), with
PatternMatchTagger applied on top as tag_rules.oracle_tokenize_lines applies it.

TEST INFRASTRUCTURE ONLY.  The library is compiled once per source state into the temporary directory (the tree may be
read-only)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from . import oracle
from .spans_oracle import wsconst_mask
from .tag_rules import parse_tokenized_line, pattern_match_filter, write_tokenized

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_SRCS = [os.path.join(_ROOT, "tests", "native", "tokenize_doc_oracle.cpp"),
         os.path.join(_ROOT, "oracle", "vaporetto_oracle.cpp"),
         os.path.join(_ROOT, "oracle", "grapheme_tables.hpp")]

_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for f in _SRCS:
            h.update(open(f, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"vpt_tokenize_doc_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", tmp, _SRCS[0]])
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.ora_last_error.restype = C.c_char_p
        L.ora_model_read.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
        L.ora_model_free.argtypes = [C.c_void_p]
        L.ora_predictor_new.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
        L.ora_predictor_free.argtypes = [C.c_void_p]
        L.ora_predictor_n_tags.argtypes = [C.c_void_p]
        L.ora_kytea_fullwidth.restype = C.c_uint32
        L.ora_kytea_fullwidth.argtypes = [C.c_uint32]
        L.ora_tokenize_docs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_uint32, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        _lib = L
    return _lib


class TokenizeDocOracle:
    """Model::read + Predictor::new + the per-document tokenized text of vpt_tokenize_dev, on the CPU."""

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

    def tokenize_docs(self, text, offsets, no_norm: bool = False, wsconst: str = "", predict_tags: bool = False,
                      rules=None):
        """-> (list of bytes per document, status uint8 array).  `rules`: {surface: [tag or None]} for
        PatternMatchTagger after fill_tags (predict_tags only; exact for models whose tag strings are not empty)."""
        t = np.frombuffer(bytes(text), np.uint8) if isinstance(text, (bytes, bytearray)) else np.ascontiguousarray(text, np.uint8)
        off = np.ascontiguousarray(offsets, np.uint64)
        n = off.size - 1
        out_off = np.zeros(n + 1, np.uint64)
        status = np.zeros(max(n, 1), np.uint8)
        cap = 64
        for _ in range(2):
            buf = C.create_string_buffer(cap)
            rc = lib().ora_tokenize_docs(self._p, t.ctypes.data, off.ctypes.data, n, int(no_norm), wsconst_mask(wsconst),
                                         int(predict_tags), out_off.ctypes.data, status.ctypes.data, buf, cap)
            if rc == 2:
                cap = int(out_off[-1]) + 64
                continue
            break
        if rc:
            raise oracle.OracleError(rc, lib().ora_last_error().decode())
        raw = buf.raw
        docs = [raw[int(out_off[d]):int(out_off[d + 1])] for d in range(n)]
        if rules is not None and predict_tags:
            fw = lib().ora_kytea_fullwidth
            key = (lambda s: s) if no_norm else (lambda s: "".join(chr(fw(ord(c))) for c in s))
            docs = [write_tokenized(pattern_match_filter(parse_tokenized_line(d.decode()), self.n_tags, rules,
                                                         key)).encode() if d else b"" for d in docs]
        return docs, status[:n]
