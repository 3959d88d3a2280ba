"""Test helpers for PatternMatchTagger rules: the C ABI's array layout of a rule dict, a restatement of the filter from
the reference source applied to the oracle's tagged output, and the host build of tests/native/tag_rules_test.cpp."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from vpt_testlib import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
CSRC = os.path.join(os.path.dirname(TESTS), "vaporetto_b200", "csrc")
NONE = 0xFFFFFFFF


def encode(rules) -> tuple:
    """{surface: [tag or None]} (or a list of pairs, duplicates kept) -> (n_rules, surfaces, surface_offsets,
    slot_offsets, slots, tags) as vpt_tag_rules_new takes them; strings may also be bytes (invalid UTF-8 on purpose)."""
    items = list(rules.items()) if isinstance(rules, dict) else list(rules)
    surf, soff, qoff, slots, tags = bytearray(), [0], [0], [], bytearray()
    for key, vals in items:
        surf += key if isinstance(key, bytes) else key.encode()
        soff.append(len(surf))
        for v in vals:
            if v is None:
                slots += [NONE, 0]
            else:
                b = v if isinstance(v, bytes) else v.encode()
                slots += [len(tags), len(b)]
                tags += b
        qoff.append(len(slots) // 2)
    return (len(items), np.frombuffer(bytes(surf) + b"\0", np.uint8), np.array(soff, np.uint64),
            np.array(qoff, np.uint64), np.array(slots + [0, 0], np.uint32), np.frombuffer(bytes(tags) + b"\0", np.uint8),
            len(tags))


def esc(s: str) -> str:
    """write_tokenized_text's escaping (sentence.rs:850-886): '\\' before ' ', '\\' and '/'."""
    return "".join("\\" + c if c in " /\\" else c for c in s)


def pattern_match_filter(tokens, n_tags: int, rules, key=lambda s: s):
    """PatternMatchTagger::filter (vaporetto_rules/src/sentence_filters/pattern_match_tagger.rs:21-41), restated: for
    every token [(surface, [tag or None])] and every slot j < n_tags that is None, a rule for key(surface) sets the slot
    to rules[key(surface)].get(j) (None beyond the rule's entries).  Predicted tags are never overwritten."""
    out = []
    for surface, tags in tokens:
        tags = list(tags) + [None] * (n_tags - len(tags))
        r = rules.get(key(surface))
        if r is not None:
            tags = [t if t is not None else (r[j] if j < len(r) else None) for j, t in enumerate(tags)]
        out.append((surface, tags))
    return out


def write_tokenized(tokens) -> str:
    """Sentence::write_tokenized_text (sentence.rs:850-886): tokens joined by ' ', each followed by '/' + tag for its
    slots up to the last one that has a tag, surfaces and tags escaped."""
    parts = []
    for surface, tags in tokens:
        last = max((j for j, t in enumerate(tags) if t is not None), default=-1)
        parts.append(esc(surface) + "".join("/" + esc(tags[j] or "") for j in range(last + 1)))
    return " ".join(parts)


def filter_tokens(tokens, n_tags: int, rules) -> str:
    """PatternMatchTagger::filter + write_tokenized_text on a sentence given as [(surface, [tag or None])]."""
    return write_tokenized(pattern_match_filter(tokens, n_tags, rules))


def parse_tokenized_line(line: str):
    """The tokens of one line of write_tokenized_text's output as [(surface, [tag or None])]: '\\' escapes the next
    character, ' ' ends a token, '/' starts a tag, an empty tag is None (exact when no tag string is empty)."""
    toks, fields, cur, escape = [], [], [], False
    for c in line:
        if escape:
            cur.append(c)
            escape = False
        elif c == "\\":
            escape = True
        elif c in " /":
            fields.append("".join(cur))
            cur = []
            if c == " ":
                toks.append(fields)
                fields = []
        else:
            cur.append(c)
    fields.append("".join(cur))
    toks.append(fields)
    return [(f[0], [t if t else None for t in f[1:]]) for f in toks]


def oracle_tokenize_lines(o: oracle.OraclePredictor, data: bytes, rules, no_norm=False, wsconst="") -> tuple:
    """The `predict` CLI loop with --predict-tags and PatternMatchTagger right after fill_tags: the oracle's tagged
    output (ora_tokenize_lines_tags), every token's slots filled by pattern_match_filter.  The filter sees the sentence
    that was predicted, so unless no_norm a token is matched by the KyteaFullwidthFilter image of its surface (one
    character for one: the tokens of both sentences line up).  Rejected lines stay empty.  Exact for models whose tag
    strings are not empty (model_tags_nonempty): an empty field of the output is then None."""
    out, n_lines = o.tokenize_lines(data, no_norm=no_norm, wsconst=wsconst, predict_tags=True)
    fw = oracle.lib().ora_kytea_fullwidth
    key = (lambda s: s) if no_norm else (lambda s: "".join(chr(fw(ord(c))) for c in s))
    lines = out.decode().split("\n")
    assert lines[-1] == ""
    res = [write_tokenized(pattern_match_filter(parse_tokenized_line(ln), o.n_tags, rules, key)) if ln else ""
           for ln in lines[:-1]]
    return "".join(ln + "\n" for ln in res).encode(), n_lines


def model_tags_nonempty(model_bytes: bytes) -> bool:
    """Whether every tag candidate of the model is a non-empty string (read through a host-only predictor)."""
    import vaporetto_b200 as vb
    p = vb.Predictor(vb.Model.read(model_bytes), predict_tags=True, device=-1)
    L = vb.lib()
    for t in range(L.vpt_tag_n_tokens(p._h)):
        for k in range(p.n_tags):
            for c in range(L.vpt_tag_n_candidates(p._h, t, k)):
                if not L.vpt_tag_string(p._h, t, k, c):
                    return False
    return True


def native_lib():
    """tests/native/tag_rules_test.cpp with the product's tag_rules.cpp, built for the host."""
    so = os.path.join(TESTS, "native", "libtag_rules_test.so")
    srcs = [os.path.join(TESTS, "native", "tag_rules_test.cpp"), os.path.join(CSRC, "tag_rules.cpp")]
    deps = srcs + [os.path.join(CSRC, f) for f in ("tag_rules.hpp", "tags.hpp", "tags_token.hpp", "textnorm.hpp", "common.hpp")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in deps):
        # (tags.hpp declares the launch interface next to the tables: cuda_runtime.h for the types only, nothing is linked)
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        tmp = so + ".%d.tmp" % os.getpid()
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wextra", "-I" + cuda_inc,
                               "-o", tmp] + srcs)
        os.replace(tmp, so)
    L = C.CDLL(so)
    L.tr_new.restype = C.c_void_p
    L.tr_new.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                         C.c_char_p, C.c_size_t]
    L.tr_free.argtypes = [C.c_void_p]
    L.tr_capacity.restype = C.c_uint32
    L.tr_capacity.argtypes = [C.c_void_p]
    L.tr_find.restype = C.c_int32
    L.tr_find.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_int]
    L.tr_suffix.restype = C.c_long
    L.tr_suffix.argtypes = [C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_int, C.c_void_p, C.c_char_p, C.c_char_p,
                            C.c_size_t]
    return L


class HostRules:
    """The builder's table on the host (tr_new); raises ValueError(code, message) on a rejected rule set."""

    def __init__(self, L, rules, n_tags: int):
        self.L = L
        n, surf, soff, qoff, slots, tags, tags_len = encode(rules)
        err = C.create_string_buffer(512)
        self.h = L.tr_new(n, surf.ctypes.data, soff.ctypes.data, qoff.ctypes.data, slots.ctypes.data, tags.ctypes.data,
                          tags_len, n_tags, err, 512)
        if not self.h:
            code, msg = err.value.decode().split(" ", 1)
            raise ValueError(int(code), msg)
        self.n_tags = n_tags

    def find(self, surface: str, norm: bool = False) -> int:
        b = surface.encode()
        return self.L.tr_find(self.h, b, len(b), int(norm))

    def suffix(self, surface: str, model_tags, norm: bool = False) -> str:
        """The writer's suffix for a token with the given model tags (list of str/None per slot, or None: no model)."""
        b = surface.encode()
        ref, mb = None, bytearray()
        if model_tags is not None:
            r = []
            for t in model_tags:
                if t is None:
                    r += [NONE, 0]
                else:
                    r += [len(mb), len(t.encode())]
                    mb += t.encode()
            ref = np.array(r + [0, 0], np.uint32)
        cap = 1 << 16
        out = C.create_string_buffer(cap)
        n = self.L.tr_suffix(self.h, self.n_tags, b, len(b), int(norm), None if ref is None else ref.ctypes.data,
                             bytes(mb) + b"\0", out, cap)
        assert 0 <= n <= cap
        return out.raw[:n].decode()

    def __del__(self):
        if getattr(self, "h", None):
            self.L.tr_free(self.h)
