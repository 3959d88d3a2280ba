"""Models whose weight rows sit exactly on the edges of the windows each scoring kernel accepts, and batches whose
sentences put those rows against their neighbours at exactly the separator gap.

The builder's row merge and trim (builder.cpp build_patterns), the row extents of the node table (build_node_table:
smin, smax, rel_min, rel_max, fast, r0, has_overflow), the type-scorer choice (predictor_build.cpp) and the kernel
plan (kernel_plan.hpp plan(): kernel, gap, lag and template switches) are restated here.  Every case names the edge
it was made for and `Case.model()` raises when the restated builder does not put it there, so a test that uses a
case really reaches its edge.

Weight rows, with the oracle's convention: the row (off, w) of a pattern whose last character is character c adds
w[k] to boundary c + off + k (boundary j lies between characters j and j + 1).  In a tile, boundary j of a sentence
sits on the slot of its character j, and `gap` separator slots lie between neighbouring sentences: the row of a
sentence's first character reaches r0 slots in front of it, the row of its last character r0 + 5 slots behind it.
"""
from __future__ import annotations

import numpy as np

from . import tile_edges as te
from .bincode_model import encode_model

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
INLINE_WIDTH = 6          # kInlineWidth
COMMON_GAP = 2            # fused_detail::kCommonGap
OVF_LIMIT = 32000         # overflow offsets are 16-bit

PAT = "人火星地球猫社長"   # pattern characters (kanji)
FILL = "山川木あいうカキaZ1、"  # characters no pattern uses, of several character types
SAME_TYPE_FILL = "山"      # a pattern-free character of the pattern characters' type


def wrap32(x: int) -> int:
    return ((int(x) - I32_MIN) & 0xFFFFFFFF) + I32_MIN


# ---- the builder, restated --------------------------------------------------------------------------------------

def _accumulate(dst, src):
    """Adds row src = (off, w) into dst, aligned on the smaller offset, wrapping (builder.cpp accumulate)."""
    lo = min(dst[0], src[0])
    hi = max(dst[0] + len(dst[1]), src[0] + len(src[1]))
    out = [0] * (hi - lo)
    for k, v in enumerate(dst[1]):
        out[dst[0] - lo + k] = v
    for k, v in enumerate(src[1]):
        out[src[0] - lo + k] = wrap32(out[src[0] - lo + k] + v)
    return (lo, out)


def merged_rows(md, predict_tags):
    """{pattern: (off, w) trimmed of zeros at both ends, or None for a pattern without a row} of the char patterns
    (build_patterns: union of equal strings, suffix sums, trim), and the unwrapped sums of every merged entry."""
    cw = md["char_window"]
    own, raw = {}, {}

    def add(key, off, w):
        if own.get(key) is None:
            own[key] = (off, list(w))
            raw[key] = (off, list(w))
        else:
            own[key] = _accumulate(own[key], (off, w))
            raw[key] = _accumulate_raw(raw[key], (off, w))
    for s, w in md.get("char_ngrams", []):
        add(s, -cw, w)
    for word, w, _ in md.get("dict", []):
        add(word, -len(word), w)
    if predict_tags:
        for tm in md.get("tag_models", []):
            for s, _ in tm.get("char_ngrams", []):
                own.setdefault(s, None)
                raw.setdefault(s, None)
    keys = sorted(own, key=lambda s: s.encode())
    for p in sorted(keys, key=lambda s: len(s.encode())):
        for j in range(1, len(p)):
            if p[j:] in own:
                src = own[p[j:]]
                if src is not None:
                    own[p] = src if own[p] is None else _accumulate(own[p], src)
                    raw[p] = raw[p[j:]] if raw[p] is None else _accumulate_raw(raw[p], raw[p[j:]])
                break
    rows = {}
    for p in keys:
        r = own[p]
        if r is None:
            rows[p] = None
            continue
        off, w = r
        lo, hi = 0, len(w)
        while lo < hi and w[lo] == 0:
            lo += 1
        while hi > lo and w[hi - 1] == 0:
            hi -= 1
        rows[p] = (off + lo, w[lo:hi])
    return rows, raw


def _accumulate_raw(dst, src):
    lo = min(dst[0], src[0])
    hi = max(dst[0] + len(dst[1]), src[0] + len(src[1]))
    out = [0] * (hi - lo)
    for k, v in enumerate(dst[1]):
        out[dst[0] - lo + k] = v
    for k, v in enumerate(src[1]):
        out[src[0] - lo + k] += v
    return (lo, out)


def restate(md, predict_tags=False):
    """The facts of the device model (DevModel) that plan() reads, restated from the model dict."""
    cw, tw = md["char_window"], md["type_window"]
    tms = md.get("tag_models", []) if predict_tags else []
    tags = len(tms) > 0
    tng = md.get("type_ngrams", [])
    has_char = bool(md.get("char_ngrams") or md.get("dict")) and cw > 0
    has_type = bool(tng) and tw > 0
    type_variant = 0 if not has_type else (3 if tags else (2 if tw <= 3 else 1))
    tag_tng = [t for tm in tms for t, _ in tm.get("type_ngrams", [])]
    cache = False
    tt_present, tt_depth = False, 0
    if type_variant == 2:
        cache = True
    elif type_variant in (1, 3):
        in_window = all(len(t) <= 2 * tw and len(w) + len(t) <= 2 * tw + 1 for t, w in tng)
        tps_max = max(len(t) for t in [t for t, _ in tng] + tag_tng)
        if type_variant == 3 and tw <= 3 and in_window and tps_max <= 3:
            cache = True
        else:
            tt_present, tt_depth = True, tps_max
    f = dict(type_cache_window=tw if cache else 0, tt_present=tt_present, tt_max_depth=tt_depth,
             type_a=cache and tw == 3 and all(len(t) <= 3 for t, _ in tng), emit_states=tags,
             ct_present=False, fast=True, r0=0, has_overflow=False, max_depth=0, rel_min=0, rel_max=0,
             smin=None, smax=None, rows={}, raw={})
    if not has_char:
        return f
    rows, raw = merged_rows(md, predict_tags)
    f.update(ct_present=True, rows=rows, raw=raw, max_depth=max(len(p) for p in rows))
    live = [(p, r) for p, r in rows.items() if r is not None and r[1]]
    if live:
        f["rel_min"] = min(r[0] for _, r in live)
        f["rel_max"] = max(r[0] + len(r[1]) for _, r in live)
    short = [r for p, r in live if len(p) <= 3]
    if short:
        f["smin"] = min(r[0] for r in short)
        f["smax"] = max(r[0] + len(r[1]) for r in short)
    fast = not tt_present and (not short or f["smax"] - f["smin"] <= INLINE_WIDTH)
    r0 = f["smin"] if short else (max(f["rel_min"], f["rel_max"] - INLINE_WIDTH) if live else 0)
    if r0 < -24 or r0 > 18:
        fast = False
    if fast and live and (f["rel_min"] < -OVF_LIMIT or f["rel_max"] > OVF_LIMIT):
        fast = False
    f.update(fast=fast, r0=r0,
             has_overflow=fast and bool(live) and (f["rel_min"] < r0 or f["rel_max"] > r0 + INLINE_WIDTH))
    return f


# ---- plan(), restated -------------------------------------------------------------------------------------------

def inline_rows(f):
    return (not f["ct_present"] or f["fast"]) and not f["tt_present"]


def tile_gap(f):
    tw = max(2, f["type_cache_window"] - 1)
    if not inline_rows(f):
        return tw
    r0 = f["r0"] if f["ct_present"] else 0
    return max(tw, -r0 - 1, r0 + INLINE_WIDTH - 1)


def fused_lag(f):
    r0 = f["r0"] if f["ct_present"] else 0
    return max(-r0, f["type_cache_window"], 1)


def fused_shape_ok(f):
    if not inline_rows(f):
        return False
    r0 = f["r0"] if f["ct_present"] else 0
    tw = f["type_cache_window"]
    if r0 < -5 or r0 > 0 or tw < 0 or tw > 3 or tile_gap(f) > 8:
        return False
    if f["emit_states"] and f["ct_present"] and f["max_depth"] == 0:
        return False
    return fused_lag(f) + max(tw, 1) <= 6


def tile_shape_ok(f):
    r0 = f["r0"] if f["ct_present"] else 0
    return inline_rows(f) and -8 <= r0 <= 2 and tile_gap(f) <= 8 and f["type_cache_window"] <= 3


PLAN_FIELDS = ("kernel", "common_shape", "deep", "r0_fixed", "general", "split3", "overflow", "gap", "lag")


def plan(f):
    """The fields PLAN_FIELDS of vpt_predictor_kernel_plan for the restated model facts f."""
    p = dict(kernel="", common_shape=0, deep=0, r0_fixed=0, general=0, split3=0, overflow=0, gap=0, lag=0)
    if fused_shape_ok(f):
        gap = tile_gap(f)
        p.update(kernel="k_fused", gap=gap, lag=fused_lag(f),
                 common_shape=int(f["type_a"] and f["type_cache_window"] == 3 and f["ct_present"] and f["r0"] == -3
                                  and gap == COMMON_GAP),
                 deep=0 if not f["ct_present"] or f["max_depth"] <= 3 else (2 if f["has_overflow"] else 1))
        return p
    tile_general = (not inline_rows(f) and f["type_cache_window"] <= 3 and f["max_depth"] <= 3
                    and f["tt_max_depth"] <= 4)
    if tile_shape_ok(f) or tile_general:
        p.update(kernel="k_tile_fast", gap=tile_gap(f), general=int(tile_general),
                 r0_fixed=int(not tile_general and f["ct_present"] and f["r0"] == -3),
                 split3=int(f["type_a"] and f["type_cache_window"] == 3),
                 overflow=int(not tile_general and f["ct_present"] and f["has_overflow"]))
        return p
    p["kernel"] = "k_score_fast" if inline_rows(f) else "k_score_general"
    return p


def library_plan(plan_dict):
    return {k: plan_dict[k] for k in PLAN_FIELDS}


# ---- the model builder ------------------------------------------------------------------------------------------

def _row(rng, length, base, lo, hi, lim=3000):
    """A raw row of `length` entries whose entry k sits at relative offset base + k: nonzero exactly on [lo, hi]
    (random values of magnitude <= lim, never zero), zero elsewhere."""
    assert base <= lo <= hi <= base + length - 1, (base, lo, hi, length)
    w = [0] * length
    for rel in range(lo, hi + 1):
        v = int(rng.integers(1, lim + 1)) * (1 if rng.random() < 0.5 else -1)
        w[rel - base] = v
    return w


def build_model(cw, ng_lens=(1, 2, 3), rows=((-3, 2),), tw=0, tng_lens=(), dict_lens=(), long_range=None,
                tags=0, bias=None, seed=0, n_per_len=12):
    """A model dict: every character of PAT as a 1-gram, `n_per_len` random n-grams over PAT of each further length in
    `ng_lens`, dictionary words over PAT of the lengths in `dict_lens`, type n-grams of the lengths in `tng_lens`
    (type window `tw`) and `tags` tag models.  The rows of the patterns of at most three characters are nonzero
    exactly on the relative range rows[i % len(rows)] (inclusive), so that r0 = min(lo) and the row width is
    max(hi) + 1 - r0; the rows of longer n-grams and of dictionary words on `long_range` (clipped to what each row
    can hold; default: their whole row)."""
    rng = np.random.default_rng(seed)
    alpha = list(PAT)

    def word(n):
        return "".join(rng.choice(alpha, size=n))
    strings = list(alpha) if 1 in ng_lens else []
    seen = set(strings)
    for n in ng_lens:
        if n == 1:
            continue
        for _ in range(n_per_len):
            s = word(n)
            if s not in seen:
                seen.add(s)
                strings.append(s)
    cng, i = [], 0
    for s in strings:
        n = len(s)
        if n <= 3:
            lo, hi = rows[i % len(rows)]
            i += 1
        else:
            lo, hi = long_range if long_range else (-cw, cw - n)
            lo, hi = max(lo, -cw), min(hi, cw - n)
        cng.append((s, _row(rng, 2 * cw - n + 1, -cw, lo, hi)))
    dic, dseen = [], set()
    for n in dict_lens:
        for _ in range(1 if n > 64 else 6):
            s = word(n)
            if s in dseen:
                continue
            dseen.add(s)
            lo, hi = long_range if long_range else (-n, 0)
            lo, hi = max(lo, -n), min(hi, 0)
            dic.append((s, _row(rng, n + 1, -n, lo, hi), ""))
    tng = {}
    for L in tng_lens:
        for _ in range(30 if L > 1 else 6):
            t = bytes(rng.integers(1, 7, size=L).tolist())
            tng[t] = rng.integers(-3000, 3000, size=max(2 * tw - L + 1, 1)).tolist()
    tms = []
    for t in range(tags):
        cn = [(word(int(rng.integers(1, 4))), [(int(rng.integers(0, cw + 1)), rng.integers(-99, 99, size=2).tolist())])
              for _ in range(5)]
        tn = [(bytes(rng.integers(1, 7, size=int(rng.integers(1, 3))).tolist()),
               [(int(rng.integers(0, max(tw, 1))), rng.integers(-99, 99, size=2).tolist())]) for _ in range(3)] if tw else []
        tms.append(dict(token=word(2) + str(t), tags=[["x", "y"]], char_ngrams=cn, type_ngrams=tn, bias=[1, 2]))
    return dict(char_ngrams=cng, type_ngrams=list(tng.items()), dict=dic,
                bias=int(rng.integers(-500, 500)) if bias is None else bias,
                char_window=cw, type_window=tw, tag_models=tms)


def window_for(lo, hi, maxlen=3):
    """The smallest char window whose n-gram rows (lengths 1..maxlen) can hold entries at lo and hi."""
    return max(1, -lo, hi + maxlen)


# ---- the cases --------------------------------------------------------------------------------------------------

class Case:
    """A model made for one edge: `edge` names it, `on_edge(f, plan)` tells whether the restated builder put the model
    there, `expect` the plan fields it must get.  `gap_side`: which term of the separator gap the char rows make tight
    ("left": -r0 - 1, "right": r0 + 5), for the gap liveness check."""

    def __init__(self, name, edge, model_args, expect, on_edge, tags=False, states=False, gap_sides=(), values=None):
        self.name, self.edge, self.model_args, self.expect = name, edge, model_args, expect
        self.on_edge, self.tags, self.states, self.gap_sides, self.values = on_edge, tags, states, gap_sides, values
        self._md = None

    def model_dict(self):
        if self._md is None:
            md = build_model(**self.model_args)
            if self.values:
                self.values(md)
            self._md = md
        return self._md

    def facts(self):
        return restate(self.model_dict(), self.tags)

    def plan(self):
        return plan(self.facts())

    def model(self):
        """Model bytes; raises if the model is not on its edge or does not get the expected plan."""
        f = self.facts()
        p = plan(f)
        if not self.on_edge(f, p):
            raise AssertionError(f"{self.name}: model missed its edge ({self.edge}): r0 {f['r0']}, smin {f['smin']}, "
                                 f"smax {f['smax']}, rel {f['rel_min']}..{f['rel_max']}, plan {p}")
        for k, v in self.expect.items():
            if p[k] != v:
                raise AssertionError(f"{self.name}: restated plan {p} has {k} = {p[k]}, the case expects {v}")
        return encode_model(self.model_dict())


def _r0_width(r0, width):
    def f(fa, p):
        return fa["fast"] and fa["r0"] == r0 and fa["smax"] - fa["smin"] == width
    return f


def _all(*preds):
    return lambda f, p: all(q(f, p) for q in preds)


def _tw(tw):
    return lambda f, p: f["type_cache_window"] == tw


def _sides(r0):
    """The char terms of the gap that are tight (>= every other term) at window start r0."""
    s = []
    if -r0 - 1 >= r0 + INLINE_WIDTH - 1:
        s.append("left")
    if r0 + INLINE_WIDTH - 1 >= -r0 - 1:
        s.append("right")
    return tuple(s)


def fused_tw_max(r0):
    """The largest type window k_fused accepts at window start r0 (-1: none)."""
    return max([tw for tw in range(4) if max(-r0, tw, 1) + max(tw, 1) <= 6], default=-1)


def _window_case(r0, tw, width=INLINE_WIDTH, tng=None, tags=False, name=None, edge=None, seed=0):
    hi = r0 + width - 1
    tng = tuple(range(1, min(2 * tw, 3) + 1)) if tng is None else tng
    args = dict(cw=window_for(r0, hi), rows=((r0, hi),) if width <= INLINE_WIDTH else ((r0, r0 + 5), (hi - 5, hi)),
                tw=tw, tng_lens=tng if tw else (), tags=2 if tags else 0, seed=seed + 100 * tw + (r0 + 40))
    return args


def window_cases():
    out = []
    # k_fused: every (r0, tw) it accepts, rows of full width (weight in entries 0 and 5)
    for tw in range(4):
        for r0 in range(-5, 1):
            if fused_tw_max(r0) < tw:
                continue
            gap = max(max(2, tw - 1), -r0 - 1, r0 + 5)
            lag = max(-r0, tw, 1)
            out.append(Case(f"fused-r0{r0:+d}-tw{tw}", f"k_fused accepts r0 {r0}, type window {tw}",
                            _window_case(r0, tw), dict(kernel="k_fused", gap=gap, lag=lag, general=0),
                            _all(_r0_width(r0, 6), _tw(tw)), gap_sides=_sides(r0)))
    # ... and the first neighbour it refuses: r0 one below its range and r0 = 1 for every type window, the next type
    # window for every r0
    refused = set()
    for tw in range(4):
        lo = min(r0 for r0 in range(-5, 1) if fused_tw_max(r0) >= tw)
        refused |= {(lo - 1, tw), (1, tw)}
    for r0 in range(-5, 1):
        refused.add((r0, fused_tw_max(r0) + 1))
    for r0, tw in sorted(refused):
        if tw <= 3:
            exp = dict(kernel="k_tile_fast", general=0, gap=max(max(2, tw - 1), -r0 - 1, r0 + 5),
                       split3=int(tw == 3))
            on = _all(_r0_width(r0, 6), _tw(tw))
            sides = _sides(r0)
        else:   # type window 4: the type automaton, general rows
            exp = dict(kernel="k_tile_fast", general=1, gap=2)
            on = lambda f, p: f["tt_present"] and not f["fast"]
            sides = ()
        out.append(Case(f"fused-refuses-r0{r0:+d}-tw{tw}", f"k_fused refuses r0 {r0}, type window {tw}",
                        _window_case(r0, tw, tng=(1, 2, 3, 4) if tw == 4 else None), exp, on, gap_sides=sides))
    # k_tile_fast's inline window ends and its refusals
    for r0, tw in ((-8, 2), (-7, 1), (2, 2), (2, 0)):
        out.append(Case(f"tile-r0{r0:+d}-tw{tw}", f"k_tile_fast accepts r0 {r0}",
                        _window_case(r0, tw), dict(kernel="k_tile_fast", general=0, gap=max(2, -r0 - 1, r0 + 5)),
                        _all(_r0_width(r0, 6), _tw(tw)), gap_sides=_sides(r0)))
    for r0 in (-9, 3):
        out.append(Case(f"tile-refuses-r0{r0:+d}", f"k_tile_fast refuses r0 {r0}",
                        _window_case(r0, 2), dict(kernel="k_score_fast"), _r0_width(r0, 6)))
    # k_score_fast's window range and row width, and the neighbours that fall to general rows
    for r0, tw in ((-24, 2), (18, 1), (-12, 3)):
        out.append(Case(f"score-fast-r0{r0:+d}", f"k_score_fast accepts r0 {r0}", _window_case(r0, tw),
                        dict(kernel="k_score_fast"), _r0_width(r0, 6)))
    for r0, tw in ((-25, 2), (19, 1)):
        out.append(Case(f"general-r0{r0:+d}", f"r0 {r0} is past the shuffle gather: general rows",
                        _window_case(r0, tw), dict(kernel="k_tile_fast", general=1),
                        lambda f, p, r0=r0: not f["fast"] and f["r0"] == r0 and f["smax"] - f["smin"] == 6))
    for r0, tw, kern in ((-12, 2, "k_score_fast"), (-3, 3, "k_fused")):
        out.append(Case(f"width7-r0{r0:+d}", f"short rows 7 wide at r0 {r0}: general rows ({kern} at width 6)",
                        _window_case(r0, tw, width=7), dict(kernel="k_tile_fast", general=1),
                        lambda f, p, r0=r0: not f["fast"] and f["smin"] == r0 and f["smax"] - f["smin"] == 7))
    return out


def type_cases():
    out = []
    # type window 3 without split tables: a type n-gram of four types
    for r0, kern, split in ((-3, "k_fused", 1), (-3, "k_fused", 0), (0, "k_fused", 0), (-6, "k_tile_fast", 1),
                            (-6, "k_tile_fast", 0), (1, "k_tile_fast", 0)):
        tng = (1, 2, 3) if split else (1, 2, 3, 4)
        exp = dict(kernel=kern, gap=max(2, -r0 - 1, r0 + 5))
        if kern == "k_fused":
            exp.update(common_shape=int(split and r0 == -3), lag=max(-r0, 3))
        else:
            exp.update(split3=split)
        out.append(Case(f"tw3-{'split' if split else 'nosplit'}-{kern}-r0{r0:+d}",
                        f"type window 3 {'with' if split else 'without'} split tables in {kern}",
                        _window_case(r0, 3, tng=tng), exp,
                        lambda f, p, split=split: f["type_cache_window"] == 3 and bool(f["type_a"]) == bool(split)))
    # tag predictors: pattern-id states (the direct type-state table) at both tile kernels
    for r0, tw, kern in ((-3, 2, "k_fused"), (-7, 2, "k_tile_fast"), (-4, 3, "k_tile_fast"), (-12, 1, "k_score_fast")):
        out.append(Case(f"tags-{kern}-r0{r0:+d}-tw{tw}", f"tag predictor, {kern} at r0 {r0}, type window {tw}",
                        _window_case(r0, tw, tags=True), dict(kernel=kern), _all(_r0_width(r0, 6), _tw(tw)),
                        tags=True, states=True, gap_sides=_sides(r0) if kern != "k_score_fast" else ()))
    return out


def overflow_cases():
    out = []

    def ovf(left, right):
        def f(fa, p):
            return (fa["fast"] and fa["has_overflow"] and (fa["rel_min"] == fa["r0"] - 1) == left
                    and (fa["rel_max"] == fa["r0"] + INLINE_WIDTH + 1) == right
                    and fa["r0"] - 1 <= fa["rel_min"] and fa["rel_max"] <= fa["r0"] + INLINE_WIDTH + 1)
        return f
    # dictionary rows one entry left of the window (k_fused), and on both sides (k_tile_fast at r0 -6: a row ending
    # at the word's last boundary is one past the window [-6, 0))
    out.append(Case("overflow-dict-left-fused", "dictionary rows one entry left of k_fused's window",
                    dict(cw=5, rows=((-3, 2),), tw=2, tng_lens=(1, 2, 3), dict_lens=(4, 5, 9), long_range=(-4, 0), seed=11),
                    dict(kernel="k_fused", deep=2), ovf(True, False), gap_sides=("left", "right")))
    out.append(Case("overflow-ngram-right-fused", "4-gram rows one entry right of k_fused's window",
                    dict(cw=7, ng_lens=(1, 2, 3, 4), rows=((-3, 2),), tw=3, tng_lens=(1, 2, 3), long_range=(-3, 3), seed=12),
                    dict(kernel="k_fused", deep=2, common_shape=1), ovf(False, True), gap_sides=("left", "right")))
    out.append(Case("overflow-dict-both-tile", "dictionary rows one entry out on both sides of k_tile_fast's window",
                    dict(cw=6, rows=((-6, -1),), tw=2, tng_lens=(1, 2, 3), dict_lens=(7, 8, 12), long_range=(-7, 0), seed=13),
                    dict(kernel="k_tile_fast", overflow=1), ovf(True, True), gap_sides=("left",)))
    out.append(Case("deep-dict-inside-fused", "dictionary rows that end exactly on k_fused's window edge",
                    dict(cw=5, rows=((-3, 2),), tw=2, tng_lens=(1, 2, 3), dict_lens=(4, 6), long_range=(-3, 0), seed=14),
                    dict(kernel="k_fused", deep=1),
                    lambda f, p: f["fast"] and not f["has_overflow"] and f["rel_min"] == f["r0"], gap_sides=("left", "right")))
    # the 16-bit overflow offset: a dictionary word of 32 000 characters keeps inline rows, one of 32 001 does not
    out.append(Case("dict-32000", "dictionary word of 32 000 characters: overflow offset at its 16-bit limit",
                    dict(cw=5, rows=((-3, 2),), tw=2, tng_lens=(1, 2), dict_lens=(OVF_LIMIT, 5), seed=15),
                    dict(kernel="k_fused", deep=2), lambda f, p: f["fast"] and f["rel_min"] == -OVF_LIMIT))
    out.append(Case("dict-32001", "dictionary word of 32 001 characters: past the 16-bit limit, general rows",
                    dict(cw=5, rows=((-3, 2),), tw=2, tng_lens=(1, 2), dict_lens=(OVF_LIMIT + 1, 5), seed=16),
                    dict(kernel="k_score_general"), lambda f, p: not f["fast"] and f["rel_min"] == -OVF_LIMIT - 1))
    return out


# weight values: bias and the row of 人 make boundaries score exactly these (with tw = 0 nothing else adds)
EXACT = (0, 1, I32_MIN, I32_MAX, -1, 2)
VALUE_BIAS = 12345
BIG = 1 << 30


def _set_values(r0, width):
    """Model edits of the weight-value cases: 人's row makes boundaries score EXACT (bias VALUE_BIAS); 火's row is
    all BIG, so that runs of 火 wrap the device sums; the 2-gram 星火 adds I32_MAX to 火's row, so its merged row wraps
    in the builder; 社's row cancels the 2-gram 猫社's own row, so that 猫社's merged row trims to empty."""
    def edit(md):
        cw = md["char_window"]
        # (no other pattern ends with 火, so that a run of 火 adds 火's row alone)
        cng = {s: w for s, w in md["char_ngrams"] if s == "火" or not s.endswith("火")}
        base = -cw
        vals = [wrap32(v - VALUE_BIAS) for v in EXACT]
        w = [0] * (2 * cw)
        for k in range(width):
            w[r0 + k - base] = vals[k % len(vals)] if k < len(vals) else 777
        cng["人"] = w
        cng["火"] = [BIG if r0 <= rel < r0 + width else 0 for rel in range(base, base + 2 * cw)]
        w2 = [0] * (2 * cw - 1)
        for k in range(width):
            w2[r0 + k - base] = I32_MAX - k
        cng["星火"] = w2
        soc = cng["社"]
        cng["猫社"] = [-v for v in soc[: 2 * cw - 1]]
        md["char_ngrams"] = list(cng.items())
        md["bias"] = VALUE_BIAS
    return edit


def value_cases():
    out = []
    for r0, width, kern in ((-3, 6, "k_fused"), (-7, 6, "k_tile_fast"), (-12, 6, "k_score_fast"), (-3, 7, "k_tile_fast")):
        hi = r0 + width - 1
        args = dict(cw=window_for(r0, hi), rows=((r0, r0 + 5), (hi - 5, hi)), tw=0, tags=1, seed=21 + r0 + width)
        exp = dict(kernel=kern, general=int(width > 6))

        def on(f, p, r0=r0, width=width):
            rows, raw = f["rows"], f["raw"]
            wraps = any(v != wrap32(v) for v in raw["星火"][1])
            return f["smin"] == r0 and f["smax"] - f["smin"] == width and wraps and rows["猫社"] is not None \
                and rows["猫社"][1] == [] and rows["人"][0] == r0
        out.append(Case(f"values-{kern}-r0{r0:+d}-w{width}", f"exact, wrapping and cancelling weights in {kern}",
                        args, exp, on, tags=True, states=True, values=_set_values(r0, width),
                        gap_sides=_sides(r0) if width == 6 and kern != "k_score_fast" else ()))
    return out


def all_cases():
    return window_cases() + type_cases() + overflow_cases() + value_cases()


# the plans the cases must reach between them (kernel, and for the tile kernels the switches that change code paths)
MATRIX = (
    ("k_fused", "r0 0, tw 3, not common, gap 5, lag 3", dict(kernel="k_fused", common_shape=0, gap=5, lag=3)),
    ("k_fused", "r0 -5, tw 1, gap 4, lag 5", dict(kernel="k_fused", gap=4, lag=5)),
    ("k_fused", "common shape", dict(kernel="k_fused", common_shape=1)),
    ("k_fused", "deep 1", dict(kernel="k_fused", deep=1)),
    ("k_fused", "deep 2", dict(kernel="k_fused", deep=2)),
    ("k_tile_fast", "split3, gap 6", dict(kernel="k_tile_fast", split3=1, gap=6, general=0)),
    ("k_tile_fast", "gap 7", dict(kernel="k_tile_fast", gap=7, general=0)),
    ("k_tile_fast", "type window 3, no split", dict(kernel="k_tile_fast", split3=0, general=0)),
    ("k_tile_fast", "overflow", dict(kernel="k_tile_fast", overflow=1)),
    ("k_tile_fast", "general", dict(kernel="k_tile_fast", general=1)),
    ("k_score_fast", "", dict(kernel="k_score_fast")),
    ("k_score_general", "", dict(kernel="k_score_general")),
)


# ---- sentences ----------------------------------------------------------------------------------------------------

EDGE_LENS = (1, 2, 3, 8)


def _sentence_lens(f, rng, n):
    """Sentence lengths: 1, 2, 3 and about 8 characters, plus ones long enough for the row's first and last kept
    entries to land on the first and last boundaries (c = -r0 and c = n - 2 - (r0 + w - 1) both inside the sentence),
    and some that cross several 32-character chunks."""
    r0, w = f["r0"], (f["smax"] - f["smin"]) if f["smin"] is not None else INLINE_WIDTH
    need = max(-r0 + 2, r0 + w + 2, 4)
    pool = list(EDGE_LENS) + [7, 9, need, need + 1] + [40, 70]
    return [pool[i % len(pool)] if pool[i % len(pool)] < 40 else int(rng.integers(33, 100)) for i in range(n)]


def _edge_chars(f, L):
    """The characters of a sentence of L characters whose row's first kept entry lands on its first boundary and
    whose last kept entry lands on its last boundary (those that exist)."""
    r0 = f["r0"]
    w = (f["smax"] - f["smin"]) if f["smin"] is not None else INLINE_WIDTH
    return [c for c in (-r0, L - 2 - (r0 + w - 1)) if 0 <= c < L]


def _row_width(f):
    return (f["smax"] - f["smin"]) if f["smin"] is not None else INLINE_WIDTH


def sentences(f, pl, n, seed=0):
    """n sentences over PAT and FILL, laid out as one group of a tile with pl["gap"] separator slots: the first and
    last characters of every sentence are pattern characters (their rows reach into the separator gap), and so are
    the characters whose row's first kept entry lands on the sentence's first boundary and whose last kept entry
    lands on its last boundary, and one character whose row crosses each 32-slot chunk edge of the tile."""
    rng = np.random.default_rng(seed)
    lens = _sentence_lens(f, rng, n)
    total = int(sum(lens))
    pat = np.array(list(PAT), "<U1")
    fill = np.array(list(FILL), "<U1")
    chars = np.where(rng.random(total) < 0.75, pat[rng.integers(len(pat), size=total)], fill[rng.integers(len(fill), size=total)])
    r0, w, gap = f["r0"], _row_width(f), max(pl["gap"], 1)
    # slot -> index into chars, for the character slots of the group's tile
    first = gap * (np.arange(n) + 1) + np.concatenate([[0], np.cumsum(lens)[:-1]])
    slot_of = {}
    pos = 0
    for k, L in enumerate(lens):
        for c in [0, L - 1] + _edge_chars(f, L):
            chars[pos + c] = pat[rng.integers(len(pat))]
        for i in range(L):
            slot_of[int(first[k]) + i] = pos + i
        pos += L
    end = int(first[-1]) + lens[-1]
    for e in range(32, end, 32):
        src = [slot_of[s] for s in range(e - r0 - w + 1, e - r0) if s in slot_of]
        if src:
            chars[src[int(rng.integers(len(src)))]] = pat[rng.integers(len(pat))]
    out, pos = [], 0
    for L in lens:
        out.append("".join(chars[pos:pos + L].tolist()))
        pos += L
    return out


def check_group_edges(f, pl, sents):
    """Raises unless the group of sentences `sents` (one tile: the fast path of k_fused or one range of k_tile_fast)
    puts rows on the edges the batch is made for: every sentence starts and ends with a pattern character, with its
    neighbours exactly `gap` slots away; there are sentences of 1, 2 and 3 characters and ones on whose first and last
    boundary a row's first and last kept entries land; and rows cross every 32-slot chunk edge of the tile that a
    character's row can reach."""
    gap = pl["gap"]
    nch = [len(s) for s in sents]
    offs = np.concatenate([[0], np.cumsum([len(s.encode()) for s in sents])]).tolist()
    got = te.classify(pl, offs, nch)
    assert got == ("fast",) or got == ("ranges", [(0, len(sents), False)]), f"the group is not one tile: {got}"
    assert all(s[0] in PAT and s[-1] in PAT for s in sents), "a sentence edge without a pattern character"
    assert {1, 2, 3} <= set(nch), "no sentences of 1, 2 and 3 characters"
    r0, w = f["r0"], _row_width(f)
    # (a row entirely left of its character lands on no sentence's last boundary, one entirely right on no first one)
    full = [s for s in sents if len(_edge_chars(f, len(s))) == int(r0 <= 0) + int(r0 + w - 1 >= -1)]
    assert full and all(all(s[c] in PAT for c in _edge_chars(f, len(s))) for s in sents), \
        "no row lands on a sentence's first and last boundary"
    slot, pat_slots, char_slots = gap, [], []
    for s in sents:
        pat_slots += [slot + i for i, ch in enumerate(s) if ch in PAT]
        char_slots += range(slot, slot + len(s))
        slot += len(s) + gap
    ps, cs = np.array(pat_slots), np.array(char_slots)
    reach = [e for e in range(32, slot - gap, 32) if np.any((cs + r0 < e) & (cs + r0 + w - 1 >= e))]
    assert len(reach) >= (slot // 32) // 2, "too few chunk edges in reach of a row"
    for e in reach:
        assert np.any((ps + r0 < e) & (ps + r0 + w - 1 >= e)), f"no row crosses the chunk edge at slot {e}"


def batch(case, f, pl, n_groups, seed=0):
    """n_groups groups of 64 edge sentences (each checked with check_group_edges for the tile kernels), a last
    partial group, and the sentences the case's weight values need: (text uint8, offsets uint64, sentences)."""
    sents = []
    for g in range(n_groups):
        grp = sentences(f, pl, te.GROUP, seed=seed * 7919 + g)
        if pl["kernel"] in ("k_fused", "k_tile_fast") and g < 4:
            check_group_edges(f, pl, grp)
        sents += grp
    sents += extra_sentences(case, f)
    sents += sentences(f, pl, 37, seed=seed + 1)
    enc = [s.encode() for s in sents]
    offs = np.zeros(len(enc) + 1, np.uint64)
    np.cumsum([len(e) for e in enc], out=offs[1:])
    return np.frombuffer(b"".join(enc), np.uint8), offs, sents


def extra_sentences(case, f):
    """Sentences a case's weights need beyond the edge groups: the exact-value and wrapping runs of the value cases,
    the long dictionary words in their sentences."""
    out = []
    if case.values:
        out += [value_sentence(), WRAP_RUN, "山星火山星火火", "猫社" * 3, "人"]
    for word, _, _ in case.model_dict().get("dict", []):
        if len(word) > 64:
            out.append("山" + word + "火")
    return out


WRAP_RUN = "火" * 40


def value_sentence():
    """A sentence in which 人's row lands whole: its boundaries -r0 .. -r0 + w - 1 around 人 score bias + row."""
    return SAME_TYPE_FILL * 30 + "人" + SAME_TYPE_FILL * 30


# ---- gap liveness, with the oracle --------------------------------------------------------------------------------

def gap_probe(f, pl, side, seed=0):
    """(sentence with a pattern character on the probed edge, the same with that character replaced by a pattern-free
    one of its type, boundary index): sentences A and B scored as one sentence with gap - 1 pattern-free characters
    between them (the gap one slot short).  "left": B's first character against A's last boundary; "right": A's last
    character against B's first boundary."""
    rng = np.random.default_rng(seed)
    gap = pl["gap"]
    n = max(8, -f["r0"] + 2, f["r0"] + 8)
    a = "".join(rng.choice(list(PAT), size=n))
    b = "".join(rng.choice(list(PAT), size=n))
    mid = SAME_TYPE_FILL * (gap - 1)
    if side == "left":
        return a + mid + b, a + mid + SAME_TYPE_FILL + b[1:], len(a) - 2
    return a + mid + b, a[:-1] + SAME_TYPE_FILL + mid + b, len(a) + gap - 1
