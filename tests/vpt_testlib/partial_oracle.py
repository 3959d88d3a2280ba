"""CPU oracle of vpt_tokenize_partial_lines (tests/native/partial_oracle.cpp: Sentence::parse_partial_annotation
restated, and the chain of the C header over the oracle's Sentence and Predictor), and the host build of
tests/native/partial_parse_test.cpp.

TEST INFRASTRUCTURE ONLY.  The libraries are compiled once per source state into the temporary directory (the tree may
be read-only)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

from . import oracle
from . import tag_rules as tr
from .spans_oracle import wsconst_mask

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_NATIVE = os.path.join(_ROOT, "tests", "native")
_ORACLE_SRCS = [os.path.join(_NATIVE, "partial_oracle.cpp"), os.path.join(_ROOT, "oracle", "vaporetto_oracle.cpp"),
                os.path.join(_ROOT, "oracle", "grapheme_tables.hpp")]
_TEST_SRCS = [os.path.join(_NATIVE, "partial_parse_test.cpp"),
              os.path.join(_ROOT, "vaporetto_b200", "csrc", "partial_parse.hpp"),
              os.path.join(_ROOT, "vaporetto_b200", "csrc", "common.hpp")] + _ORACLE_SRCS

_libs = {}


def _build(name: str, srcs, opt: str = "-O2"):
    if name not in _libs:
        h = hashlib.sha256()
        for f in srcs:
            h.update(open(f, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"vpt_{name}_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["g++", opt, "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", tmp, srcs[0]])
            os.replace(tmp, so)
        _libs[name] = C.CDLL(so)
    return _libs[name]


def lib():
    L = _build("partial_oracle", _ORACLE_SRCS)
    L.ora_last_error.restype = C.c_char_p
    L.ora_model_read.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
    L.ora_model_free.argtypes = [C.c_void_p]
    L.ora_predictor_new.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
    L.ora_predictor_free.argtypes = [C.c_void_p]
    L.ora_predictor_n_tags.argtypes = [C.c_void_p]
    L.ora_partial_parse.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.POINTER(C.c_size_t), C.c_char_p,
                                    C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    L.ora_partial_write.restype = C.c_long
    L.ora_partial_write.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
    L.ora_partial_lines.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int, C.c_uint32, C.c_int, C.c_char_p,
                                    C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    return L


def parse_test_lib():
    """tests/native/partial_parse_test.cpp: partial_parse.hpp against the restatement."""
    L = _build("partial_parse_test", _TEST_SRCS, "-O2")
    L.pp_check_all.restype = C.c_long
    L.pp_check_all.argtypes = [C.c_int, C.c_char_p, C.c_size_t]
    return L


def parse(line: bytes):
    """-> (raw text bytes, [marker codes]) or raises oracle.OracleError(kind, ...) with .message and .pos set."""
    L = lib()
    text = C.create_string_buffer(len(line) + 1)
    given = C.create_string_buffer(len(line) + 1)
    tl, ng, pos = C.c_size_t(), C.c_size_t(), C.c_size_t()
    rc = L.ora_partial_parse(line, len(line), text, C.byref(tl), given, C.byref(ng), C.byref(pos))
    if rc:
        e = oracle.OracleError(rc, L.ora_last_error().decode())
        e.message, e.pos = L.ora_last_error().decode(), pos.value
        raise e
    return text.raw[: tl.value], list(given.raw[: ng.value])


def write(line: bytes) -> str:
    """Sentence::from_partial_annotation(line) + write_tokenized_text; raises oracle.OracleError(kind, message)."""
    L = lib()
    cap = 4 * len(line) + 16
    buf = C.create_string_buffer(cap)
    n = L.ora_partial_write(line, len(line), buf, cap)
    if n < 0:
        e = oracle.OracleError(-n, L.ora_last_error().decode())
        e.message = L.ora_last_error().decode()
        raise e
    return buf.raw[:n].decode()


class PartialOracle:
    """Model::read + Predictor::new + the chain of vpt_tokenize_partial_lines, on the CPU."""

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

    def lines(self, data: bytes, no_norm: bool = False, wsconst: str = "", predict_tags: bool = False, rules=None):
        """-> (output bytes, n_lines, error) with error None or (status, message): the output of the lines before
        the first bad line.  `rules` ({surface: [tag or None]}): PatternMatchTagger after fill_tags, keyed by the
        KyteaFullwidthFilter image of a token unless no_norm (exact for models whose tag strings are not empty)."""
        L = lib()
        cap = 4 * len(data) + 16 + (64 * len(data) if predict_tags else 0)
        buf = C.create_string_buffer(cap)
        n, nl, el = C.c_uint64(), C.c_uint64(), C.c_uint64()
        rc = L.ora_partial_lines(self._p, data, len(data), int(no_norm), wsconst_mask(wsconst), int(predict_tags), buf,
                                 cap, C.byref(n), C.byref(nl), C.byref(el))
        if rc not in (0, 2, 5):
            raise oracle.OracleError(rc, L.ora_last_error().decode())
        out = buf.raw[: n.value]
        if rules and predict_tags:
            fw = oracle.lib().ora_kytea_fullwidth
            key = (lambda s: s) if no_norm else (lambda s: "".join(chr(fw(ord(c))) for c in s))
            lines = out.decode().split("\n")
            res = [tr.write_tokenized(tr.pattern_match_filter(tr.parse_tokenized_line(ln), self.n_tags, rules, key))
                   if ln else "" for ln in lines[:-1]]
            out = "".join(ln + "\n" for ln in res).encode()
        return out, int(nl.value), (None if rc == 0 else (rc, L.ora_last_error().decode()))
