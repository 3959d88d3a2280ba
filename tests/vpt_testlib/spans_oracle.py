"""CPU oracle of vpt_token_spans (tests/native/spans_oracle.cpp: vaporetto_tantivy's token_stream restated over the
oracle's Sentence and Predictor), plus literal Python restatements of the filters it composes, for checking it.

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

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_SRCS = [os.path.join(_ROOT, "tests", "native", "spans_oracle.cpp"),
         os.path.join(_ROOT, "oracle", "vaporetto_oracle.cpp"),
         os.path.join(_ROOT, "oracle", "grapheme_tables.hpp")]

_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for f in _SRCS:
            h.update(open(f, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"vpt_spans_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
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
        L.ora_token_spans.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_uint32, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                      C.POINTER(C.c_uint64)]
        _lib = L
    return _lib


def wsconst_mask(wsconst: str) -> int:
    return sum(1 << ("DRHTKOG".index(ch) + 1) for ch in set(wsconst))


class SpansOracle:
    """Model::read + Predictor::new + token_stream for a batch of documents, on the CPU."""

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

    def token_spans(self, text, offsets, no_norm: bool = False, wsconst: str = "", tags: bool = False):
        """-> dict of n_tokens, status, token_ends and (tags) token_ids, token_cands [tokens, n_tags]."""
        t = np.frombuffer(bytes(text), np.uint8) if isinstance(text, (bytes, bytearray)) else np.ascontiguousarray(text, np.uint8)
        off = np.ascontiguousarray(offsets, np.uint64)
        n = off.size - 1
        cap = max(int(off[-1] - off[0]) if n > 0 else 0, 1)
        nt = self.n_tags
        n_tokens = np.zeros(max(n, 1), np.uint32)
        status = np.zeros(max(n, 1), np.uint8)
        ends = np.zeros(cap, np.uint32)
        ids = np.zeros(cap, np.int32)
        cands = np.zeros(cap * max(nt, 1), np.uint8)
        total = C.c_uint64()
        rc = lib().ora_token_spans(self._p, t.ctypes.data, off.ctypes.data, n, int(no_norm), wsconst_mask(wsconst),
                                   int(tags), n_tokens.ctypes.data, status.ctypes.data, ends.ctypes.data,
                                   ids.ctypes.data, cands.ctypes.data, cap, C.byref(total))
        if rc:
            raise oracle.OracleError(rc, lib().ora_last_error().decode())
        k = int(total.value)
        out = {"n_tokens": n_tokens[:n], "status": status[:n], "token_ends": ends[:k]}
        if tags:
            out["token_ids"] = ids[:k]
            out["token_cands"] = cands[: k * max(nt, 1)].reshape(-1, max(nt, 1))[:, :nt]
        return out


# ---- literal restatements, for checking the oracle against a composition of ora_predict ----------------------------

def split_linebreaks(chars, boundaries):
    """SplitLinebreaksFilter (split_linebreaks.rs:9-37): boundary i lies between chars[i] and chars[i + 1]."""
    b = list(boundaries)
    for i in range(len(chars) - 1):
        if chars[i] in "\r\n" or chars[i + 1] in "\r\n":
            b[i] = 1
    return b


def wsconst_filter(types, boundaries, t):
    """KyteaWsConstFilter (kytea_wsconst.rs:27-44) for character type t."""
    b = list(boundaries)
    for i in range(len(types) - 1):
        if types[i] == t and types[i + 1] == t:
            b[i] = 0
    return b


def grapheme_filter(cluster_lengths, boundaries):
    """ConcatGraphemeClustersFilter (concat_grapheme_clusters.rs:10-35): no boundary inside a cluster."""
    b = list(boundaries)
    pos = 0
    for n in cluster_lengths:
        for i in range(pos, pos + n - 1):
            b[i] = 0
        pos += n
    return b


def boundary_pos(text: str, boundaries):
    """lib.rs:179-188: the byte offset of every character after a WordBoundary, then the text's byte length."""
    starts = np.cumsum([0] + [len(c.encode()) for c in text]).tolist()
    return [starts[i + 1] for i, b in enumerate(boundaries) if b == 1] + [len(text.encode())]


def compose(ora: "oracle.OraclePredictor", text: str, no_norm: bool = False, wsconst: str = ""):
    """token_stream's ends for one non-empty document from ora_predict and the literal filters above."""
    pre = text if no_norm else "".join(chr(oracle.lib().ora_kytea_fullwidth(ord(c))) for c in text)
    _, b = ora.predict(pre)
    b = split_linebreaks(text, [int(x) for x in b])
    types = oracle.char_types(pre).tolist()
    for ch in wsconst:
        if ch == "G":
            b = grapheme_filter(oracle.grapheme_lengths(pre), b)
        else:
            b = wsconst_filter(types, b, "DRHTKOG".index(ch) + 1)
    return boundary_pos(text, b)
