"""Models and text on which KyteaFullwidthFilter changes what a model matches.

The predict CLI and every tokenizing entry point score KyteaFullwidthFilter(text) unless no_norm, and each kernel maps
the code points on the fly (kytea_fullwidth, csrc/textnorm.hpp).  The models of tile_edges draw their patterns from
characters the filter keeps or from half-width ones the filter moves away (`a` becomes `ａ`, which no pattern holds), so
they never show whether a kernel matched the filtered character.  The models here draw their patterns over filter
images (plus kana, kanji and 2- and 4-byte fixed points), and the text spells the images through their sources: the
half-width letters, digits and punctuation, and the dashes and half-width CJK punctuation.  A pattern then matches only
when the kernel maps the character; the dashes also change type (Other to Katakana), so every type n-gram and the
`wsconst K` filter see different input under the filter.

The filter tables come from the fixture tests/golden/kytea_fullwidth_map.json, not from the library.
"""
from __future__ import annotations

import json
import os

import numpy as np

from . import tile_edges as te
from .bincode_model import encode_model

_GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "golden")
FILTER = {chr(int(k)): chr(v) for k, v in json.load(open(os.path.join(_GOLDEN, "kytea_fullwidth_map.json"))).items()}

SOURCES = "".join(sorted(FILTER))                                                    # every character the filter changes
IMAGES = "".join(sorted(set(FILTER.values())))                                       # what they become
FIXED = "".join(c for c in map(chr, range(0x20, 0x7F)) if c not in FILTER)           # printable ASCII the filter keeps
SPELLINGS = {img: "".join(s for s in SOURCES if FILTER[s] == img) for img in IMAGES}  # image -> its sources
DASHES = SPELLINGS["ー"]                                                              # U+2013 U+2015 U+2500 U+FF0D

# the images patterns are drawn from: every type the filter produces (Roman, Digit, Other, and Katakana from the
# dashes), images with one source and with several (ー has four, 。 two)
PATTERN_IMAGES = "ＡＢａｂ１２ー。，”−「」・〜"
# pattern characters: those images, kana and kanji, and fixed points of 2 and 4 bytes
PATTERN_ALPHABET = PATTERN_IMAGES + "あいアイ人猫éß𠀋𩸽"
# text characters: the pattern characters, every source of their images, and some 1-byte fixed points
TEXT_ALPHABET = PATTERN_ALPHABET + "".join(SPELLINGS[c] for c in PATTERN_IMAGES) + "#|~"


def normalize(text: str) -> str:
    """KyteaFullwidthFilter by the fixture's table."""
    return "".join(FILTER.get(c, c) for c in text)


def source_spellings(word: str, rng) -> str:
    """`word` with every image spelled by one of its sources, chosen at random (ー: one of its four dashes)."""
    return "".join(SPELLINGS[c][int(rng.integers(len(SPELLINGS[c])))] if c in SPELLINGS else c for c in word)


def _words(rng, n, draws):
    """The distinct ones of `draws` random words of n pattern characters, each with an image in it (so its source
    spelling differs from it)."""
    alpha = list(PATTERN_ALPHABET)
    out = {}
    for _ in range(draws):
        w = list(rng.choice(alpha, size=n))
        w[int(rng.integers(n))] = PATTERN_IMAGES[int(rng.integers(len(PATTERN_IMAGES)))]
        out["".join(w)] = None
    return list(out)


def _weights(rng, n):
    """n weights, none zero (so no row is trimmed and every row keeps the extent the model gives it)."""
    w = rng.integers(-3000, 3000, size=n)
    return np.where(w == 0, 1, w).tolist()


def norm_model(cw, tw, ng_lens, dict_lens, tags=0, seed=1, ng_weights=None):
    """(model bytes, long patterns: dictionary words, then n-grams) in the shape of
    tile_edges.variant_model(cw, tw, ng_lens, dict_lens, tags) -- the same windows, n-gram and dictionary lengths,
    pattern counts and tag count -- with patterns over images: char n-grams and dictionary words over PATTERN_ALPHABET,
    every type n-gram up to length 3, and tag models whose tokens and char n-grams are images.  `ng_weights`: length
    of every char n-gram's weight vector (default: the window's 2 * cw - n + 1)."""
    rng = np.random.default_rng(seed)
    cng = {}
    for n in ng_lens:
        for w in _words(rng, n, 60):
            cng[w] = _weights(rng, ng_weights or max(2 * cw - n + 1, 0))
    dic = [(w, _weights(rng, len(w) + 1), "") for n in dict_lens for w in _words(rng, n, 20)]
    tng = {}
    for n in (1, 2, 3):
        if n <= 2 * tw:
            for k in range(6 ** n):
                tng[bytes(1 + (k // 6 ** j) % 6 for j in range(n))] = _weights(rng, 2 * tw - n + 1)
    tms = []
    tokens = list(PATTERN_IMAGES[:tags])   # one-character tokens: frequent enough in the text to be tagged often
    for t in range(tags):
        cn = [(w, [(int(rng.integers(0, cw + 1)), rng.integers(-99, 99, size=2).tolist())])
              for w in _words(rng, int(rng.integers(1, 3)), 5)]
        tn = [(bytes(rng.integers(1, 7, size=int(rng.integers(1, 4))).tolist()),
               [(int(rng.integers(0, tw + 1)), rng.integers(-99, 99, size=2).tolist())]) for _ in range(3)]
        tms.append(dict(token=tokens[t], tags=[["x", "y"]], char_ngrams=cn, type_ngrams=tn, bias=[1, 2]))
    mb = encode_model(dict(char_ngrams=list(cng.items()), type_ngrams=list(tng.items()), dict=dic,
                           bias=int(rng.integers(-500, 500)), char_window=cw, type_window=tw, tag_models=tms))
    return mb, [w for w in [d[0] for d in dic] + list(cng) if len(w) >= 4]   # (tile_edges places the first ones first)


def recipes():
    """tile_edges.variant_recipes() with the model arguments for norm_model: (name, VPT_SEED_BUDGET or None, model
    arguments, predict_tags, with_states, expected plan key)."""
    return [("norm-" + name, budget, args, tags, states, key)
            for name, budget, args, tags, states, key in te.variant_recipes()]


def _key(kernel):
    return (kernel,) + (0,) * (len(te.PLAN_KEYS) - 1)


# The one-warp-per-sentence kernels (no tile geometry): (name, model arguments, predict_tags, with_states, key).
#   k_score_general: char window 4 makes the char rows general (a unigram's row spans 8 positions, the inline window 6),
#     type window 4 needs the type automaton; dictionary words of 4 and more characters make the tables too deep for
#     k_tile_fast's general variant.
#   k_score_fast: inline rows whose window starts at -10: char window 10 with n-gram weight vectors of 6 (shorter than
#     the window's 2 * cw - n + 1, which the format allows) put every short row on [-10, -4); both tile kernels refuse a
#     window start below -8 (k_fused: below -5).
SCORE_KERNELS = []
for _tags, _states in ((0, False), (2, True)):
    _form = "states" if _states else "plain"
    SCORE_KERNELS += [
        (f"score-general-cw4-{_form}", (4, 2, (1, 2, 3), (4, 6), _tags), bool(_tags), _states, _key("k_score_general")),
        (f"score-general-tw4-{_form}", (3, 4, (1, 2, 3), (4, 5), _tags), bool(_tags), _states, _key("k_score_general")),
        (f"score-fast-{_form}", (10, 3, (1, 2, 3), (4, 7), _tags, 1, 6), bool(_tags), _states, _key("k_score_fast")),
    ]


def text_for(words, n, rng, lo=5, hi=60):
    """n sentences of TEXT_ALPHABET characters (no line terminators), every third with a source spelling of one of
    `words` in it."""
    alpha = np.array(list(TEXT_ALPHABET))
    out = []
    for i in range(n):
        s = "".join(alpha[rng.integers(len(alpha), size=int(rng.integers(lo, hi)))].tolist())
        if words and i % 3 == 0:
            at = int(rng.integers(len(s) + 1))
            s = s[:at] + source_spellings(words[int(rng.integers(len(words)))], rng) + s[at:]
        out.append(s)
    return out
