"""Sentences whose token ends sit exactly on the edges of k_tags' chunk and ring arithmetic, and a model that tags them.

k_tags (csrc/tags.cu) walks a sentence 32 characters per step.  Before step c0 it decodes 128-byte windows, from the
4-byte aligned position b0 & ~3 on, until it holds min(n, c0 + 33) characters (decode_window, kernels_common.cuh); each
window appends its characters to a 256-slot ring of byte positions, so after the step's decoding the ring holds the
characters [nd - 256, nd).  A lane whose character e ends a token needs the byte position of the token's first
character s and of character e + 1 (or b1 for the sentence's last character):

  as at first   s in this step: ring slot s.  Otherwise only when e - s < 216 (`near`): ring slot s, read in THIS step
                -- not live once nd - 256 > s (a "stale" slot: the token silently lost its tags); e - s >= 216: the token
                is "unserved" (left to the host path by the batch calls, written untagged by the lines paths).
  now           s in this step: ring slot s.  Otherwise a carry, read from ring slot s at the end of the step that holds
                character s - 1 (the previous token's end), where it is always live.

Every case built here is checked against this restatement: a construction that misses the edge it names raises.

The model (`model`) makes the boundaries exact, as reference_kat.TOKENIZED_ESCAPE does: bias -1, char_window 1 and a
unigram (term, [0, 2]) for one terminator character per UTF-8 width, so a token ends after every terminator.  Every
character used maps to itself under KyteaFullwidthFilter, so the cases mean the same with and without no_norm.  A
known target token is fill * (L - 1) + term; its tag model has a bias and char n-gram weights (term and fill + term at
rel 0, pad at rel 1), so its tags depend on the pattern-id states around the token end (`expected_cands`).  Each known
target has an unknown twin of the same length that differs in one character.
"""
from __future__ import annotations

import bisect
import functools
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

RING = 256
STEP = 32
WINDOW = 128
NEAR = RING - 40  # the `near` limit of the first k_tags: e - s < 216

# per UTF-8 width: fill (target tokens), twin (one character of a twin), term (ends every token), pad (other tokens)
CHARS = {
    1: ("$", "~", "#", "^"),
    2: ("é", "è", "ß", "ñ"),
    3: ("あ", "い", "。", "う"),
    4: ("\U0001d538", "\U0001d539", "\U0001f600", "\U0001d53b"),
}
TAGS = [["A", "B"], ["C", "D", "E"]]


def fill(w):
    return CHARS[w][0]


def twin_char(w):
    return CHARS[w][1]


def term(w):
    return CHARS[w][2]


def pad(w):
    return CHARS[w][3]


# ---- the arithmetic, restated ------------------------------------------------------------------------------------

def step_nd(lead: List[int], nbytes: int, align: int) -> List[int]:
    """nd after the decoding of every step: `lead` = byte positions of the characters from b0, `align` = b0 % 4."""
    n = len(lead)
    nd, w, out = 0, -align, []
    for c0 in range(0, n, STEP):
        need = min(n, c0 + STEP + 1)
        while nd < need and w < nbytes:
            nd += bisect.bisect_left(lead, min(w + WINDOW, nbytes)) - bisect.bisect_left(lead, max(w, 0))
            w += WINDOW
        out.append(nd)
    return out


def live(nd: int, c: int) -> bool:
    return nd - RING <= c < nd


def locate(nd: List[int], n: int, s: int, e: int, fixed: bool) -> Tuple[str, Optional[int]]:
    """How k_tags finds the first byte of the token [s, e] of a sentence of n characters (nd: step_nd()): ("ok", step
    whose ring slot s is read), ("stale", step) or ("unserved", None); ("ok", None) for s == 0 (the carry's initial
    value)."""
    k = e // STEP
    # the end of the token (character e + 1) comes from the ring of the same step: always live
    assert e + 1 == n or live(nd[k], e + 1)
    if s >= k * STEP:
        assert live(nd[k], s)
        return "ok", k
    if fixed:
        if s == 0:
            return "ok", None
        kp = (s - 1) // STEP
        assert live(nd[kp], s), "the carry must always read a live slot"
        return "ok", kp
    if e - s >= NEAR:
        return "unserved", None
    return ("ok" if live(nd[k], s) else "stale"), k


def uniform_lead(w: int, n: int) -> List[int]:
    return [w * i for i in range(n)]


@functools.lru_cache(maxsize=None)
def uniform_nd(w: int, n: int, align: int) -> Tuple[int, ...]:
    return tuple(step_nd(uniform_lead(w, n), w * n, align))


def outcome(w: int, n: int, align: int, s: int, e: int, fixed: bool) -> str:
    """locate() for a sentence of n characters of UTF-8 width w."""
    return locate(uniform_nd(w, n, align), n, s, e, fixed)[0]


def shortest_stale(w: int, align: int, tail: int = 160) -> Tuple[int, int]:
    """(L, s) of the shortest token that reads a stale slot at the first k_tags in a sentence of width-`w` characters
    starting at b0 % 4 == align, followed by `tail` characters; the smallest s among those of that length."""
    for L in range(2, NEAR + 1):
        for s in range(0, 2 * RING):
            if outcome(w, s + L + tail, align, s, s + L - 1, fixed=False) == "stale":
                return L, s
    raise AssertionError("no stale slot below the near limit")


# ---- cases ---------------------------------------------------------------------------------------------------------

@dataclass
class Case:
    kind: str                 # the edge
    w: int                    # UTF-8 width of every character
    align: int                # b0 % 4 the sentence must start at
    tokens: List[str]         # the sentence's tokens
    target: int               # index of the token on the edge
    known: bool = True        # the target is a known token (False: its twin)
    old: str = "ok"           # what the first k_tags does with the target
    sentence: str = field(init=False)

    def __post_init__(self):
        self.sentence = "".join(self.tokens)

    def span(self) -> Tuple[int, int]:
        s = sum(len(t) for t in self.tokens[: self.target])
        return s, s + len(self.tokens[self.target]) - 1


def target_token(w: int, L: int) -> str:
    return fill(w) * (L - 1) + term(w)


def twin_token(w: int, L: int) -> str:
    t = list(target_token(w, L))
    t[(L - 1) // 2] = twin_char(w)
    return "".join(t)


def pad_token(w: int, n: int) -> str:
    return pad(w) * (n - 1) + term(w)


def _case(kind, w, align, P, L, S, check=None) -> List[Case]:
    """The target token of L characters behind P and ahead of S characters of pad tokens, and its twin."""
    out = []
    for known in (True, False):
        toks = ([pad_token(w, P)] if P else []) + [target_token(w, L) if known else twin_token(w, L)] + \
               ([pad_token(w, S)] if S else [])
        c = Case(kind, w, align, toks, 1 if P else 0, known)
        s, e = c.span()
        n = len(c.sentence)
        c.old = outcome(w, n, align, s, e, fixed=False)
        assert outcome(w, n, align, s, e, fixed=True) == "ok"
        if check is not None:
            assert check(c, s, e, n), (kind, w, align, P, L, S)
        out.append(c)
    return out


def window_ends_inside(w, align, pos_char) -> bool:
    """A 128-byte decode window ends strictly inside character `pos_char` of a sentence of width-w characters."""
    b = w * pos_char
    return any(b < x < b + w for x in range(WINDOW - align, b + w + WINDOW, WINDOW))


def edge_cases() -> List[Case]:
    cases: List[Case] = []
    for w in (1, 2, 3, 4):
        for align in range(4):
            L, s = shortest_stale(w, align)
            cases += _case("stale", w, align, s, L, 160, lambda c, s_, e, n: c.old == "stale")
            cases += _case("stale-1", w, align, s + 1, L - 1, 160, lambda c, s_, e, n: c.old == "ok")
            # either side of the first k_tags' near limit
            cases += _case("len216", w, align, 5, NEAR, 40, lambda c, s_, e, n: c.old != "unserved")
            cases += _case("len217", w, align, 5, NEAR + 1, 40, lambda c, s_, e, n: c.old == "unserved")
            for L in (33, 100):
                # token ends at lane 0 and lane 31 of a step
                for lane in (0, 31):
                    P = (lane - (L - 1)) % STEP + STEP * 4
                    cases += _case("lane%d" % lane, w, align, P, L, 7, lambda c, s_, e, n, ln=lane: e % STEP == ln)
            for steps in (1, 2, 8):
                cases += _case("steps%d" % steps, w, align, STEP, STEP * steps, 3,
                               lambda c, s_, e, n, k=steps: s_ % STEP == 0 and e // STEP - s_ // STEP + 1 == k
                               and (e + 1) % STEP == 0)
            # (in a sentence of one width, a window ends inside a character only where w * p + align is not a multiple
            # of 4 for some p: width 2 at odd alignments, width 3 always, width 4 when unaligned)
            for which, L in (("first", 150), ("last", 150)):
                P = next((P for P in range(1, 400) if window_ends_inside(w, align, P if which == "first" else P + L - 1)), None)
                if P is not None:
                    cases += _case("window-" + which, w, align, P, L, 9,
                                   lambda c, s_, e, n, wh=which: window_ends_inside(w, align, s_ if wh == "first" else e))
            for L in (2, 40, 100, 300):
                cases += _case("whole%d" % L, w, align, 0, L, 0, lambda c, s_, e, n: s_ == 0 and e + 1 == n)
    return cases


LONG_KNOWN = "$" * 69_999 + "#"       # a known one-token line of 70 000 bytes
LONG_PREFIX = "$" * 65_535            # a known token: the first 65 535 bytes of LONG_UNKNOWN and of LONG_KNOWN
LONG_UNKNOWN = "$" * 70_000 + "#"     # 70 001 bytes: must not be looked up as its prefix


def known_tokens(cases: List[Case]) -> List[str]:
    out = dict.fromkeys(c.tokens[c.target] for c in cases if c.known)
    out[LONG_KNOWN] = None
    out[LONG_PREFIX] = None
    return list(out)


def tag_model(token: str) -> dict:
    """Slot 0: bias [0, 1] + term at rel 0 [2, 0] + (fill, term) at rel 0 [0, 2] -> B; + pad at rel 1 [3, 0] -> A.
    Slot 1: a bias of 10 on candidate len(token) % 3."""
    w = len(token[-1].encode("utf-8"))
    L = len(token)
    b1 = [10 if k == L % 3 else 0 for k in range(3)]
    return dict(token=token, tags=TAGS,
                char_ngrams=[(term(w), [(0, [2, 0, 0, 0, 0])]), (fill(w) + term(w), [(0, [0, 2, 0, 0, 0])]),
                             (pad(w), [(1, [3, 0, 0, 0, 0])])],
                type_ngrams=[], bias=[0, 1] + b1)


def expected_cands(token: str, next_char: Optional[str]) -> List[int]:
    """The candidates tag_model(token) chooses for `token` followed by `next_char` (None: the sentence's end)."""
    w = len(token[-1].encode("utf-8"))
    assert len(token) >= 2 and token[-2:] == fill(w) + term(w)
    return [0 if next_char == pad(w) else 1, len(token) % 3]


def model(cases: List[Case], extra_tag_models=()) -> dict:
    return dict(char_ngrams=[(term(w), [0, 2]) for w in CHARS], type_ngrams=[], dict=[], bias=-1, char_window=1,
                type_window=1, tag_models=[tag_model(t) for t in known_tokens(cases)] + list(extra_tag_models))


def expected_sentence_cands(sentence_tokens: List[str], known: set) -> List[List[int]]:
    """Per character: the candidates of the token ending there (-1 elsewhere and for unknown tokens)."""
    out = []
    text = "".join(sentence_tokens)
    pos = 0
    for t in sentence_tokens:
        out += [[-1, -1]] * (len(t) - 1)
        pos += len(t)
        out.append(expected_cands(t, text[pos] if pos < len(text) else None) if t in known else [-1, -1])
    return out


# ---- layout of a batch / a buffer of lines ------------------------------------------------------------------------

def aligned_batch(sentences: List[Tuple[str, int]]) -> Tuple[List[str], List[int]]:
    """(sentence, align) pairs -> the sentence list with short pad sentences ('^' * k) in front of those that need them
    so that every sentence starts at its byte offset % 4, and the indices of the original sentences."""
    out, idx, off = [], [], 0
    for s, align in sentences:
        k = (align - off) % 4
        if k:
            out.append("^" * k)
            off += k
        idx.append(len(out))
        out.append(s)
        off += len(s.encode("utf-8"))
    return out, idx


def aligned_lines(sentences: List[Tuple[str, int]], crlf_every: int = 3) -> bytes:
    """One line per sentence, every `crlf_every`-th ending in "\\r\\n", each starting at its byte offset % 4 (short
    '^' lines in between)."""
    parts, off = [], 0
    for i, (s, align) in enumerate(sentences):
        k = (align - off) % 4
        if k:
            k = k if k >= 2 else k + 4
            parts.append(b"^" * (k - 1) + b"\n")
            off += k
        b = s.encode("utf-8") + (b"\r\n" if i % crlf_every == crlf_every - 1 else b"\n")
        parts.append(b)
        off += len(b)
    return b"".join(parts)
