"""Lines and documents whose features sit exactly on the 128-byte window and 4-byte lane edges of the byte-window
kernels (lines.cu k_tok_write / k_tok_write_tags / k_wsconst / k_grapheme, spans.cu k_split_linebreaks / k_token_ends /
k_span_count, evaluate.cu k_gold_parse / k_eval).

The window arithmetic, restated.  One warp walks one line (document) whose bytes are [o0, o1) of the text it sees:

  a0 = o0 & ~3          the aligned word the walk starts from
  b0 = o0 - a0          (0..3) the line's first byte, in window coordinates
  b1 = o1 - a0 - trim   the line's end; trim is 1 for '\\n', 2 for '\\r\\n' (line paths), 0 for documents
  window k              coordinates [w0, w0 + 128) with w0 = 128 * k; everything that spans windows is a register carry
  lane                  (x - w0) // 4 holds the 4-byte word of coordinate x; x % 4 is its byte in the lane

k_tok_write takes a single-window register path when b1 <= 128, the streaming path otherwise.  k_span_count reads the
boundary bytes of a document as aligned words from bound_offsets & ~3, so there the coordinates are
r = bound_offsets % 4 and r + n_chars - 1.  k_eval walks boundaries, not bytes: 32 per step.

Coordinates are those of the device buffer, so every layout here states how a caller's offsets become device offsets
and checks it (`line_buffer`, `doc_batch`).  A case is built from the text in front of its feature, the feature's bytes
and the text after it (`_case`): the feature's position is measured from that text, the Case holds the feature's bytes
and its constructor raises unless those bytes are at that position of the payload and the position lands on the
coordinate the case names.  So no case drifts off its edge when a string is edited.
"""
from __future__ import annotations

import bisect
import os
import re
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple, Union

from .bincode_model import encode_model

WINDOW = 128
LANE = 4
EVAL_STEP = 32
CHUNK_BYTES = 16 << 20      # capi.cpp chunk_bytes() without VPT_CHUNK_BYTES
CHUNK_SENTENCES = 262144    # capi.cpp chunk_sentences() without VPT_CHUNK_SENTENCES


def coords(o0: int, o1: int, trim: int = 0) -> Tuple[int, int, int]:
    """(a0, b0, b1) of the line [o0, o1) of the device text."""
    a0 = o0 & ~3
    return a0, o0 - a0, o1 - a0 - trim


def locate(x: int) -> Dict[str, int]:
    """Window k, its w0, the lane and the byte in the lane of window coordinate x."""
    k = x // WINDOW
    return {"window": k, "w0": WINDOW * k, "lane": (x - WINDOW * k) // LANE, "byte": x % LANE}


def streaming(b1: int) -> bool:
    """k_tok_write's choice: the streaming path (else the single-window register path)."""
    return b1 > WINDOW


@dataclass
class Case:
    """A line or document (`payload`, without its terminator) built for one edge of one kernel family.  Byte `at` of
    the payload is the feature; it lands on window coordinate `coord` when the payload starts at b0.  `feature` holds
    the feature's bytes, byte `k` of them being byte `at` of the payload."""
    kernel: str
    edge: str
    b0: int
    payload: bytes
    at: int
    coord: int
    feature: bytes
    k: int = 0
    end: bytes = b"\n"            # line terminator (line paths): b"\n" or b"\r\n"
    bound_r: Optional[int] = None  # spans runs: the bound_offsets % 4 the document needs
    info: dict = field(default_factory=dict)

    def __post_init__(self):
        if not 0 <= self.b0 < 4:
            raise ValueError(f"{self.kernel} {self.edge}: b0 {self.b0}")
        if not 0 <= self.at < len(self.payload):
            raise ValueError(f"{self.kernel} {self.edge}: feature byte {self.at} outside the payload")
        if not self.feature or self.payload[self.at - self.k:self.at - self.k + len(self.feature)] != self.feature:
            raise ValueError(f"{self.kernel} {self.edge}: the feature {self.feature!r} is not at byte {self.at - self.k}")
        if self.b0 + self.at != self.coord:
            raise ValueError(f"{self.kernel} {self.edge}: feature at {self.b0 + self.at}, the edge is {self.coord}")
        if self.kernel != "gold_err":
            self.payload.decode("utf-8")

    @property
    def b1(self) -> int:
        return self.b0 + len(self.payload)

    @property
    def key(self):
        return (self.kernel, self.edge, self.b0 if self.bound_r is None else self.bound_r)


def _b(x: Union[str, bytes]) -> bytes:
    return x.encode() if isinstance(x, str) else x


def _case(kernel: str, edge: str, b0: int, head, feature, tail, coord: int, k: int = 0, **kw) -> Case:
    """The payload head + feature + tail; the feature byte is byte k of `feature`, measured from `head`."""
    h, f = _b(head), _b(feature)
    return Case(kernel, edge, b0, h + f + _b(tail), len(h) + k, coord, f, k, **kw)


# ---- fillers of an exact byte length ---------------------------------------------------------------------------------

def fill(n: int, alphabet: str) -> str:
    """Exactly n bytes: the alphabet's characters in turn, ASCII 'a' where the next one does not fit."""
    out, left, i = [], n, 0
    while left:
        c = alphabet[i % len(alphabet)]
        i += 1
        if len(c.encode()) > left:
            c = "a"
        out.append(c)
        left -= len(c.encode())
    return "".join(out)


TOK_ALPHA = "ab#c d/é\\あx😀y"  # escapes, word ends of the tag model, every UTF-8 width
GOLD_ALPHA = "ab cd# éf あg"      # valid gold text (no escapes, no double spaces) without tags


def gold_fill(n: int) -> str:
    s = fill(n, GOLD_ALPHA)
    if s.endswith(" "):
        s = s[:-1] + "z"
    return s


# ---- models ------------------------------------------------------------------------------------------------------

TERM = "#"  # maps to itself under KyteaFullwidthFilter: a token ends after every '#'
TAG_STRINGS = [["a/b c\\d", "x"], ["y", "/ \\"]]  # both chosen strings need every escape


def model_all() -> bytes:
    """No features, bias 1: every boundary is a word boundary, every character after the first gets a ' '."""
    return encode_model(dict(bias=1))


def model_none() -> bytes:
    return encode_model(dict(bias=-1))


def model_tag() -> bytes:
    """Bias -1 and a unigram that ends a token after every '#'; the one-character token '#' has two tag slots whose
    chosen strings hold ' ', '/' and '\\'."""
    return encode_model(dict(char_ngrams=[(TERM, [0, 2])], bias=-1, char_window=1, type_window=1,
                             tag_models=[dict(token=TERM, tags=TAG_STRINGS, char_ngrams=[], type_ngrams=[],
                                              bias=[3, 0, 0, 3])]))


TAG_SUFFIX = "/a\\/b\\ c\\\\d/\\/\\ \\\\"  # what the writer puts after the token '#' (escaped)
TAG_RULES = {"x#": ["r/1", None, "q \\"], "ab#": ["ab"]}  # PatternMatchTagger rules for tokens of TOK_ALPHA lines


# ---- cases: tok_write and tagged_sentence (lines, also documents) -------------------------------------------------

EDGE_COORDS = (3, 4, 63, 64, 126, 127, 128, 129, 255, 256)
B1S = (127, 128, 129, 255, 256, 257)
ESCAPES = " /\\"


def tok_cases() -> List[Case]:
    out = []
    for b0 in range(4):
        for x in EDGE_COORDS:
            for e in ESCAPES:
                out.append(_case("tok", f"esc{e!r}@{x}", b0, fill(x - b0, TOK_ALPHA), e, fill(60, TOK_ALPHA), x))
        for w, ch in ((2, "é"), (3, "あ"), (4, "😀")):
            for j in range(1, w):
                x = WINDOW - j
                out.append(_case("tok", f"char{w}@{x}", b0, fill(x - b0, TOK_ALPHA), ch, fill(40, TOK_ALPHA), x))
        for b1 in B1S:
            for end in (b"\n", b"\r\n"):
                name = f"b1={b1}" + ("/crlf" if end == b"\r\n" else "")
                out.append(_case("tok", name, b0, fill(b1 - b0 - 1, TOK_ALPHA), "\\", "", b1 - 1, end=end))
        # tagged_sentence: the one-character token '#' ending on 127 (suffix before the ' ' of byte 128) and 128
        for x in (127, 128):
            out.append(_case("tags", f"suffix@{x}", b0, TERM * (x - b0), TERM + "x", (TERM + "x#") * 30 + TERM * 8, x))
    return out


# ---- cases: k_wsconst ----------------------------------------------------------------------------------------------

# per class (types 1..6 = D R H T K O): a pair of different characters of that class, also after KyteaFullwidthFilter
WS_PAIRS = {"D": ("１", "2"), "R": ("ｂ", "c"), "H": ("あ", "い"), "T": ("ア", "ｲ"), "K": ("漢", "字"), "O": ("★", "😀")}
WS_FILL = {"D": "aあ", "R": "1あ", "H": "aア", "T": "aあ", "K": "aあ", "O": "aあ"}  # alternating, never a pair of cls


def wsconst_cases() -> List[Case]:
    out = []
    for b0 in range(4):
        for cls, (A, B) in WS_PAIRS.items():
            # A ends on 127, B starts on 128; and A straddling the edge with B right after it
            head = fill(128 - b0 - len(A.encode()), WS_FILL[cls])
            out.append(_case("wsconst", f"pair{cls}@127|128", b0, head + A, B, fill(30, WS_FILL[cls]), 128,
                             info={"cls": cls, "first": len(head)}))
            if len(A.encode()) > 1:
                head = fill(127 - b0, WS_FILL[cls])
                out.append(_case("wsconst", f"pair{cls}@straddle", b0, head + A, B, fill(30, WS_FILL[cls]),
                                 127 + len(A.encode()), info={"cls": cls, "first": len(head)}))
        # a last window of continuation bytes only: '😀' from 127 to the line's end, after another O character
        head = fill(127 - b0 - 3, "aあ")
        out.append(_case("wsconst", "cont-only", b0, head + "★", "😀", "", 127, info={"cls": "O", "first": len(head)}))
    return out


# ---- cases: k_grapheme ---------------------------------------------------------------------------------------------

RI = "\U0001F1E6"


def _cluster(b0: int, before: str, after: str):
    """`before` ends on 127 and `after` starts on 128 (behind 'a' filler); -> (head, index of the character boundary
    between them)."""
    head = "a" * (128 - b0 - len(before.encode())) + before
    return head, len(head) - 1


def grapheme_cases(docs: bool = False) -> List[Case]:
    out = []
    for b0 in range(4):
        clusters = {
            "extend": ("e", "́̂"),
            "zwj": ("\U0001F468‍", "\U0001F469"),
            "hangul": ("ᄀ", "ᅡᆨ"),
            "gb9c": ("क्", "ष"),
            "ri-odd": (RI * 3, RI * 3),
            "ri-even": (RI * 2, RI * 3),
            "prepend0600": ("؀", "a"),
            "prepend110bd": ("\U000110bd", "a"),
        }
        if docs:
            clusters["crlf"] = ("\r", "\n")
        for name, (before, after) in clusters.items():
            head, k = _cluster(b0, before, after)
            if name == "ri-even":
                k += 1  # the even run ends a pair on the edge: the live boundary is the one after
            out.append(_case("grapheme", f"{name}@127|128", b0, head, after, "a" * 140, 128, info={"boundary": k}))
    return out


# ---- cases: the span kernels (documents) -----------------------------------------------------------------------------

def span_cases() -> List[Case]:
    out = []
    for b0 in range(4):
        for x in (126, 127, 128, 129):
            for lb in ("\n", "\r"):
                out.append(_case("spans", f"lb{lb!r}@{x}", b0, fill(x - b0, "ab#cé"), lb, fill(60, "ab#cé"), x))
        for x in (127, 128):
            # a token starts on x: '#' ends on x - 1
            out.append(_case("spans", f"tok@{x}", b0, "a" * (x - 1 - b0), TERM + "b", "a" * 20 + TERM + "bb", x, k=1))
    for r in range(4):
        for nb in (127, 128, 129):
            # nb + 1 characters, a word end at both ends of the boundary run
            chars = (TERM + "ab" + TERM + "c" + "d" * 3) * 40
            b0 = (r + 1) % 4
            c = _case("spans", f"run{nb}", b0, chars[:nb - 1], TERM, "e", b0 + nb - 1, bound_r=r, info={"nb": nb})
            assert len(c.payload.decode()) == nb + 1
            out.append(c)
    return out


# ---- cases: gold_line (evaluate) -------------------------------------------------------------------------------------

def _bs_case(b0: int, x: int, L: int, esc: str) -> Case:
    """A run of L backslashes whose last one is on x, then the byte `esc`."""
    return _case("gold", f"bs{L}@{x}/{esc!r}", b0, gold_fill(x - L + 1 - b0) + "\\" * (L - 1), "\\" + esc,
                 "q " + gold_fill(150), x, info={"L": L})


def gold_cases() -> List[Case]:
    out = []
    for b0 in range(4):
        for L in range(1, 10):
            for x in list(range(124, 133)) + list(range(0, 9)):
                if x - L + 1 < b0:
                    continue
                for esc in (" ", "/", "\\", "k"):
                    out.append(_bs_case(b0, x, L, esc))
        # a tag field open across the edge, and a token of four fields over it
        out.append(_case("gold", "field@120..135", b0, gold_fill(120 - b0), "/" + "t" * 14 + " ", gold_fill(40), 120))
        out.append(_case("gold", "fields@124..133", b0, gold_fill(124 - b0), "/u/v\\ w/x/y z ", gold_fill(40), 124))
        # the one-character token '#' (tagged by model_tag) on 127, its first '/' on 128
        out.append(_case("gold", "tagpos@128", b0, gold_fill(125 - b0) + TERM + " ", TERM + TAG_SUFFIX + " ",
                         gold_fill(40), 128, k=1))
        # multi-byte characters across the edge
        for w, ch in ((2, "é"), (3, "あ"), (4, "😀")):
            for j in range(1, w):
                out.append(_case("gold", f"char{w}@{128 - j}", b0, gold_fill(128 - j - b0), ch, gold_fill(40), 128 - j))
    return out


# error lines: (kind, bytes ending in the feature, bytes after it)
ERR_FEATURES = {
    "DoubleWs": (b"  ", b"b"),
    "Slash": (b" /", b"b"),
    "NUL": (b"\x00", b"b"),
    "EndWs": (b" ", b""),
}
UTF8_BAD = {
    "utf8-missing": (b"\xe3\x81", b"a"),
    "utf8-surrogate": (b"\xed\xa0\x80", b"a"),
    "utf8-overlong3": (b"\xe0\x80\x80", b"a"),
    "utf8-overlong2": (b"\xc0\x80", b"a"),
    "utf8-stray": (b"a\x80", b"a"),
}


def gold_error_cases() -> List[Case]:
    out = []
    for b0 in range(4):
        for x in (127, 128):
            for kind, (feat, tail) in ERR_FEATURES.items():
                out.append(_case("gold_err", f"{kind}@{x}", b0, gold_fill(x - b0 - len(feat) + 1), feat,
                                 tail + (b" " + gold_fill(30).encode() if tail else b""), x, k=len(feat) - 1,
                                 info={"kind": kind}))
        for kind, (feat, tail) in UTF8_BAD.items():
            k = 1 if kind == "utf8-stray" else 0  # the lead byte on 127; the stray continuation on 128
            out.append(_case("gold_err", f"{kind}@{127 + k}", b0, gold_fill(127 - b0), feat, tail + b" " + gold_fill(30).encode(),
                             127 + k, k=k, info={"kind": kind}))
    return out


def gold_error_multi() -> List[Tuple[str, List[bytes], int]]:
    """(name, lines, index of the line the first error is reported for): an error in window 2 and a later one in
    window 3 of the same line; a line whose first error is in window 3 ahead of a line that errs on its first byte."""
    a = (gold_fill(200) + "  " + gold_fill(100) + "\x00" + gold_fill(40)).encode()
    b = (gold_fill(300) + " /" + gold_fill(40)).encode()
    good = gold_fill(40).encode()
    return [("window2-then-3", [good, a, good], 1), ("window3-before-line-start", [good] * 3 + [b, good, b" a", good], 3)]


# ---- cases: k_eval (evaluate; model_tag) ----------------------------------------------------------------------------

NBS = (31, 32, 33, 63, 64, 65)


def sys_bounds(raw: str) -> List[int]:
    """model_tag's boundaries: after every '#'."""
    return [1 if c == TERM else 0 for c in raw[:-1]]


def gold_text(raw: str, bounds: List[int], tags: Dict[int, List[Optional[str]]] = None) -> str:
    """A gold line: tokens of `raw` split at `bounds`, the token ending on character i followed by tags[i] fields."""
    tags = tags or {}
    out = []
    for i, c in enumerate(raw):
        out.append("\\" + c if c in " /\\" else c)
        if i + 1 == len(raw) or bounds[i]:
            for t in tags.get(i, []):
                out.append("/" + ("".join("\\" + x if x in " /\\" else x for x in t) if t else ""))
            if i + 1 < len(raw):
                out.append(" ")
    return "".join(out)


def eval_cases() -> List[Tuple[str, str, str]]:
    """(name, gold line, the same line with its feature removed) for k_eval.  Raw text: 'x' and '#' characters."""
    out = []
    for nb in NBS:
        raw = "".join(TERM if i % 5 == 4 else "x" for i in range(nb + 1))
        sb = sys_bounds(raw)
        out.append((f"nb={nb}", gold_text(raw, sb), None))
        if nb >= 33:
            # a disagreement on boundary 31, a shared one on 32 (and the reverse: shared 31, disagreement 32, shared 33)
            r = list(raw)
            r[31], r[32] = "x", TERM
            r = "".join(r)
            g = sys_bounds(r)
            g[31] = 1
            out.append((f"nb={nb}/dis31-shared32", gold_text(r, g), gold_text(r, sys_bounds(r))))
            r = list(raw)
            r[31], r[32], r[33] = TERM, "x", TERM
            r = "".join(r)
            g = sys_bounds(r)
            g[32] = 1
            out.append((f"nb={nb}/shared31-dis32", gold_text(r, g), gold_text(r, sys_bounds(r))))
        # a disagreement on boundary 31 and no other boundary after it: the last token's `matched`
        r = "".join(TERM if (i % 5 == 4 and i < 31) else "x" for i in range(nb + 1))
        g = sys_bounds(r)
        g[min(31, nb - 1)] ^= 1
        out.append((f"nb={nb}/dis31-to-end", gold_text(r, g), gold_text(r, sys_bounds(r))))
        # tags: the one-character token '#' ending in the second step, its record behind the first step's tokens
        if nb >= 33:
            r = "".join(TERM if i in (4, 9, 14, 19, 24, 29, 32, 33) else "x" for i in range(nb + 1))
            right = {33: [TAG_STRINGS[0][0], TAG_STRINGS[1][1]]}  # what model_tag chooses
            wrong = {33: [TAG_STRINGS[0][1], TAG_STRINGS[1][0]]}
            out.append((f"nb={nb}/tags-right", gold_text(r, sys_bounds(r), right), gold_text(r, sys_bounds(r), wrong)))
            out.append((f"nb={nb}/tags-wrong", gold_text(r, sys_bounds(r), wrong), gold_text(r, sys_bounds(r), right)))
    return out


# ---- layouts: how offsets become device offsets ------------------------------------------------------------------

def _env_int(name: str) -> int:
    """atoll() of an environment variable, as capi.cpp reads its tuning knobs."""
    m = re.match(r"\s*([+-]?\d+)", os.environ.get(name, ""))
    return int(m.group(1)) if m else 0


def chunk_bytes() -> int:
    """capi.cpp chunk_bytes(): VPT_CHUNK_BYTES when >= 64, else 16 MiB (read at every call)."""
    x = _env_int("VPT_CHUNK_BYTES")
    return x if x >= 64 else CHUNK_BYTES


def chunk_sentences() -> int:
    """capi.cpp chunk_sentences(): VPT_CHUNK_SENTENCES when >= 1024, else 262144.  The library reads it once, at its
    first batch call, so this holds while the variable does not change in the process."""
    x = _env_int("VPT_CHUNK_SENTENCES")
    return x if x >= 1024 else CHUNK_SENTENCES


def ramp_schedule(total: int, big: int, small_up: int, small_down: int) -> List[int]:
    """capi.cpp ramp_schedule: the nominal chunk sizes of a pipeline over `total` units."""
    up, down = [], []
    v = max(small_up, 1)
    while v < big:
        up.append(v)
        v *= 2
    v = max(small_down, 1)
    while v < big:
        down.append(v)
        v *= 2
    s = sum(up) + sum(down)
    if total <= s + big:
        c = max(min(big, (total + 3) // 4), min(small_up, big))
        return [min(c, total - lo) for lo in range(0, total, c)]
    middle = total - s
    nmid = (middle + big - 1) // big
    return up + [middle // nmid + (1 if i < middle % nmid else 0) for i in range(nmid)] + down[::-1]


def line_chunk_count(n_bytes: int, big: Optional[int] = None) -> int:
    """Chunks line_chunks (capi.cpp) cuts a buffer of n_bytes into, at most (a cut moves forward to a line end)."""
    big = chunk_bytes() if big is None else big
    return len(ramp_schedule(n_bytes, big, big // 8, big // 8))


def span_chunks(offs: List[int], cs: Optional[int] = None, big: Optional[int] = None) -> List[Tuple[int, int]]:
    """capi.cpp span_chunks: the (first document, documents) chunks vpt_token_spans cuts a batch into: the ramp over
    chunk_sentences(), each cut again where its text passes the byte budget (chunk_bytes(), from 1/8 of it over the
    first three chunks)."""
    cs = chunk_sentences() if cs is None else cs
    big = chunk_bytes() if big is None else big
    out: List[Tuple[int, int]] = []
    lo = 0
    for sz in ramp_schedule(len(offs) - 1, cs, cs // 8, cs // 4):
        end = lo + sz
        while lo < end:
            budget = max(big >> (3 - len(out)), 1) if len(out) < 3 else big
            hi = bisect.bisect_right(offs, offs[lo] + budget, lo + 1, end + 1) - 1
            hi = max(hi, lo + 1)
            out.append((lo, hi - lo))
            lo = hi
    return out


def line_buffer(cases: List[Case], lead: bytes = b"") -> Tuple[bytes, List[int]]:
    """The case lines behind `lead`, each behind a short '^' padding line so that it starts at its b0 mod 4; -> (buffer,
    byte offset of every case line).  The line pipeline copies each chunk to the start of a device buffer from
    cudaMalloc (256-byte aligned) and the kernels see offsets from the chunk's first byte, so in a buffer of one chunk
    the device b0 of a line is its offset mod 4; the buffer is checked to be one chunk."""
    parts, offs, o = [lead], [], len(lead)
    for c in cases:
        k = (c.b0 - o) % 4
        if k:
            parts.append(b"^" * (k - 1) + b"\n")
            o += k
        offs.append(o)
        b = c.payload + c.end
        parts.append(b)
        o += len(b)
    data = b"".join(parts)
    if line_chunk_count(len(data)) != 1:
        raise ValueError(f"{len(data)} bytes: more than one line chunk")
    for c, off in zip(cases, offs):
        trim = len(c.end)
        _, b0, b1 = coords(off, off + len(c.payload) + trim, trim)
        if (b0, b1) != (c.b0, c.b1):
            raise AssertionError((c.key, b0, b1))
    return data, offs


def _nb(nchars: int) -> int:
    return nchars - 1 if nchars > 0 else 0


def doc_batch(cases: List[Case]) -> Tuple[bytes, List[int], List[int]]:
    """The case documents with filler documents between them: a document of m ASCII characters (m - 1 boundaries) sets
    bound_offsets mod 4 for the cases that need it, a one-character document of 1..3 bytes (no boundary) sets the byte
    offset mod 4 to b0.  -> (text, offsets [n + 1], indices of the case documents).  Offsets mod 4 are device offsets
    mod 4: the batch calls copy the text to (offset & 15) of an aligned buffer, the device calls add the text's address
    mod 16 (0 for a fresh torch allocation: checked by the caller).  bound_offsets are chunk-local in vpt_token_spans
    (the device call runs the batch as one), so a batch with such cases is checked to be one span chunk."""
    docs: List[bytes] = []
    idx = []
    o = bo = 0

    def add(b: bytes):
        nonlocal o, bo
        docs.append(b)
        o += len(b)
        bo += _nb(len(b.decode()))

    for c in cases:
        if c.bound_r is not None and (bo - c.bound_r) % 4:
            add(b"z" * ((c.bound_r - bo) % 4 + 1))
        k = (c.b0 - o) % 4
        if k:
            add({1: "z", 2: "é", 3: "あ"}[k].encode())
        assert o % 4 == c.b0 and (c.bound_r is None or bo % 4 == c.bound_r)
        idx.append(len(docs))
        add(c.payload)
    offs = [0]
    for d in docs:
        offs.append(offs[-1] + len(d))
    if any(c.bound_r is not None for c in cases) and len(span_chunks(offs)) != 1:
        raise ValueError(f"{len(docs)} documents, {offs[-1]} bytes: more than one span chunk")
    return b"".join(docs), offs, idx


def line_cases() -> List[Case]:
    return tok_cases() + wsconst_cases() + grapheme_cases()


def doc_cases() -> List[Case]:
    return tok_cases() + wsconst_cases() + grapheme_cases(docs=True)


def all_cases() -> List[Case]:
    return doc_cases() + span_cases() + gold_cases() + gold_error_cases()
