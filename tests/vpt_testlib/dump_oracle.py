"""CPU oracle of the predict CLI's score dumps (tests/native/dump_oracle.cpp: main.rs:125-181 with print_scores and
print_tag_scores over the unchanged oracle), and a Python composition of the same output from the per-sentence oracle.

TEST INFRASTRUCTURE ONLY.  The library is compiled once per source state into the temporary directory."""
from __future__ import annotations

import ctypes as C
import os

from . import oracle
from .spans_oracle import wsconst_mask
from .tag_scores_oracle import _build, tag_candidates

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = _build("dump_oracle", [os.path.join(_ROOT, "tests", "native", "dump_oracle.cpp")],
                   [os.path.join(_ROOT, "oracle", "vaporetto_oracle.cpp"), os.path.join(_ROOT, "oracle", "grapheme_tables.hpp")])
        L.ora_last_error.restype = C.c_char_p
        L.ora_model_read.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
        L.ora_model_free.argtypes = [C.c_void_p]
        L.ora_predictor_new.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
        L.ora_predictor_free.argtypes = [C.c_void_p]
        L.ora_dump_lines.restype = C.c_long
        L.ora_dump_lines.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int, C.c_uint32, C.c_int, C.c_int, C.c_int,
                                     C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64)]
        _lib = L
    return _lib


class DumpOracle:
    """Model::read + Predictor::new, then the predict CLI's loop with --scores / --tag-scores over a buffer of lines."""

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
        self.predict_tags = predict_tags

    def __del__(self):
        if getattr(self, "_p", None):
            lib().ora_predictor_free(self._p)
            self._p = None

    def dump_lines(self, data: bytes, no_norm=False, wsconst="", scores=False, tag_scores=False,
                   token_lines: bytes | None = None) -> bytes:
        """The CLI's output for `data`; `token_lines` replaces the token lines (tag rules change only those)."""
        cap = 64 * len(data) + 4096
        while True:
            buf = C.create_string_buffer(cap)
            n = C.c_uint64()
            r = lib().ora_dump_lines(self._p, data, len(data), int(no_norm), wsconst_mask(wsconst), int(self.predict_tags),
                                     int(scores), int(tag_scores), token_lines,
                                     0 if token_lines is None else len(token_lines), buf, cap, C.byref(n))
            if r <= -1000000:
                cap = -r - 1000000 + 16
                continue
            if r < 0:
                raise oracle.OracleError(int(-r), lib().ora_last_error().decode())
            return buf.raw[:r]


def compose(o: oracle.OraclePredictor, so, model: dict, lines, no_norm=False, scores=False, tag_scores=False,
            predict_tags=False) -> bytes:
    """The same output composed in Python from the per-sentence oracles, for lines without wsconst filters: token lines
    from ora_tokenize_lines(_tags), boundary scores from predict, and per token record of fill_tags (`so`, a
    TagScoresOracle) the id and score vector, read through the restated Token::tag_candidates with the tag models of
    `model` (the encode_model dict).  `lines` are str, or bytes for lines the CLI rejects."""
    fw = oracle.lib().ora_kytea_fullwidth
    tms = model.get("tag_models", [])
    out = []
    for line in lines:
        data = (line.encode() if isinstance(line, str) else line) + b"\n"
        tok, _ = o.tokenize_lines(data, no_norm=no_norm, predict_tags=predict_tags or tag_scores)
        if not isinstance(line, str) or line == "" or "\0" in line:
            out.append(b"\n" + (b" \n\n" if tag_scores else b""))
            continue
        s = line if no_norm else "".join(chr(fw(ord(c))) for c in line)
        sc, bd = o.predict(s)[:2]
        blk = "".join(f"{i}:{s[i]}{s[i + 1]} {int(sc[i])}\n" for i in range(len(s) - 1)) + "\n" if scores else ""
        t = tok[:-1].decode()
        out.append(((t + blk + "\n") if no_norm else (t + "\n" + blk)).encode())
        if tag_scores:
            toks, cur = [], s[0]
            for c, b in zip(s[1:], bd.tolist()):
                if b == 1:
                    toks.append(cur)
                    cur = c
                else:
                    cur += c
            toks.append(cur)
            enc = line.encode()
            ids, vec = so.spans(enc, [0, len(enc)], no_norm=no_norm)
            assert len(ids) == len(toks)
            blk, at = "", 0
            for tk, tid in zip(toks, ids.tolist()):
                blk += tk
                if tid >= 0:
                    n = max(8, len(tms[tid]["bias"]))
                    for cands in tag_candidates(tms[tid]["tags"], vec[at:at + n]):
                        blk += "\t" + ",".join(f"{a}:{b}" for a, b in cands)
                    at += n
                blk += "\n"
            out.append((blk + "\n").encode())
    return b"".join(out)
