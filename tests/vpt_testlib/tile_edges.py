"""Batches whose 64-sentence groups sit exactly on the edges of a scoring kernel's tile buffers.

The fit tests of the kernels are restated here (fused_kernel.cuh k_fused, kernels.cu k_tile_fast) and every group
built for an edge is checked against them: a construction that misses its edge raises, so a test that uses these
batches really reaches the edge it names.

k_fused, per group of sentences [0, ns) with byte offsets off[]:
  fast path  ((off[ns] - (off[0] & ~15) + 15) & ~15) + 16 <= text_cap  and  gap + chars + gap * ns <= slot_cap
             (and every sentence non-empty, valid, without NUL)
  otherwise  ranges [k0, k1): the longest prefix whose every sentence t passes
             ((off[t+1] - (off[k0] & ~15) + 15) & ~15) + 16 <= text_cap  and  gap + chars[k0..t] + gap * (t+1-k0) <= slot_cap;
             a sentence that fits no range on its own is walked by one warp
k_tile_fast: always the ranges, with the slot test ((slots + 8 + 255) & ~255) <= slot_cap.
"""
from __future__ import annotations

import numpy as np

GROUP = 64
HALO = 8      # slots a warp range of k_fused re-reads in front of its first output
WARPS = 8     # warps per sub-block


def utf8_len(c: str) -> int:
    return len(c.encode("utf-8"))


def by_length(alphabet):
    """{1: [...], 2: [...], 3: [...], 4: [...]}: the characters of `alphabet` by UTF-8 length."""
    out = {1: [], 2: [], 3: [], 4: []}
    for c in dict.fromkeys(alphabet):
        out[utf8_len(c)].append(c)
    assert all(out[k] for k in out), "the alphabet needs characters of every UTF-8 length"
    return out


# ---- the fit tests, restated -----------------------------------------------------------------------------------

def text_fits(plan, off0, end):
    a0 = off0 & ~15
    return ((end - a0 + 15) & ~15) + 16 <= plan["text_cap"]


def slots_fit(plan, slots):
    if plan["kernel"] == "k_tile_fast":
        return ((slots + 8 + 255) & ~255) <= plan["slot_cap"]
    return slots <= plan["slot_cap"]


def slot_limit(plan):
    """The largest slot count of a tile that passes the slot test."""
    return plan["slot_cap"] - 8 if plan["kernel"] == "k_tile_fast" else plan["slot_cap"]


def group_slots(plan, nchars):
    return plan["gap"] + int(sum(nchars)) + plan["gap"] * len(nchars)


def classify(plan, offs, nchars):
    """How a group (absolute byte offsets offs[0..ns], characters per sentence) is processed:
    ("fast",) for the fused fast path, else ("ranges", [(k0, k1, single), ...])."""
    ns = len(nchars)
    if plan["kernel"] == "k_fused" and min(nchars) > 0 and text_fits(plan, offs[0], offs[ns]) and \
            slots_fit(plan, group_slots(plan, nchars)):
        return ("fast",)
    out = []
    k0 = 0
    csum = np.concatenate([[0], np.cumsum(nchars)])
    while k0 < ns:
        k1 = ns
        for t in range(k0, ns):
            slots = plan["gap"] + int(csum[t + 1] - csum[k0]) + plan["gap"] * (t + 1 - k0)
            if not (text_fits(plan, offs[k0], offs[t + 1]) and slots_fit(plan, slots)):
                k1 = t
                break
        single = k1 == k0
        out.append((k0, k0 + 1 if single else k1, single))
        k0 = k0 + 1 if single else k1
    return ("ranges", out)


# ---- construction ----------------------------------------------------------------------------------------------

class EdgeBatch:
    """Builds a batch group by group; every edge group records what it was made for and is checked on add."""

    def __init__(self, plan, alphabet, seed=0):
        self.plan = plan
        self.alpha = by_length(alphabet)
        self._alpha_np = {k: np.array(v, "<U1") for k, v in self.alpha.items()}
        self.rng = np.random.default_rng(seed)
        self.sents = []       # str per sentence
        self.nbytes = 0
        self.edges = []       # (name, group index)

    def _draw(self, lens):
        out = np.empty(len(lens), "<U1")
        for k in (1, 2, 3, 4):
            sel = np.nonzero(lens == k)[0]
            if sel.size:
                out[sel] = self._alpha_np[k][self.rng.integers(len(self._alpha_np[k]), size=sel.size)]
        return "".join(out.tolist())

    def chars(self, n, lens=(1, 2, 3, 4)):
        """n random characters whose UTF-8 lengths are drawn from `lens`."""
        return self._draw(self.rng.choice(np.asarray(lens), size=n))

    def compose(self, nchars, nbytes):
        """A sentence of exactly nchars characters and nbytes bytes (nchars <= nbytes <= 4 * nchars)."""
        assert nchars <= nbytes <= 4 * nchars, (nchars, nbytes)
        extra = nbytes - nchars
        lens = np.ones(nchars, np.int64)
        n4 = min(nchars, extra // 3)
        lens[:n4] = 4
        rem = extra - 3 * n4
        if rem:
            lens[n4] = 1 + rem
        self.rng.shuffle(lens)
        return self._draw(lens)

    def pad_to(self, mod):
        """Adds a filler group whose byte count makes the next group start at a byte offset = mod (mod 16)."""
        assert len(self.sents) % GROUP == 0
        want = (mod - self.nbytes) % 16
        sents = [self.chars(int(self.rng.integers(10, 40)), (1, 3)) for _ in range(GROUP)]
        total = sum(len(s.encode()) for s in sents)
        sents[-1] += self.alpha[1][0] * ((want - total) % 16)
        self.add(sents)

    def add(self, sents, edge=None, expect=None):
        """Appends one group (a list of sentences); `expect` is checked against the restated fit tests."""
        assert len(self.sents) % GROUP == 0 and 0 < len(sents) <= GROUP
        offs = [self.nbytes]
        for s in sents:
            offs.append(offs[-1] + len(s.encode()))
        nch = [len(s) for s in sents]
        got = classify(self.plan, offs, nch)
        if expect is not None:
            ok = expect(got, offs, nch)
            assert ok, f"edge construction missed its edge: {edge}: {got[0]} {got[1][:4] if len(got) > 1 else ''}"
        if edge is not None:
            self.edges.append((edge, len(self.sents) // GROUP))
        self.sents += sents
        self.nbytes = offs[-1]
        return got

    def filler(self, n_groups, lo=20, hi=60):
        """Groups of ordinary sentences (most take the fused fast path)."""
        lens = self.rng.integers(lo, hi + 1, size=n_groups * GROUP)
        text = self.chars(int(lens.sum()), (1, 3, 3, 3, 2, 4))
        cut = np.concatenate([[0], np.cumsum(lens)])
        for g in range(n_groups):
            self.add([text[cut[i]:cut[i + 1]] for i in range(g * GROUP, (g + 1) * GROUP)])

    def arrays(self):
        enc = [s.encode() for s in self.sents]
        offs = np.zeros(len(enc) + 1, np.uint64)
        np.cumsum([len(e) for e in enc], out=offs[1:])
        return np.frombuffer(b"".join(enc), np.uint8), offs


def _compose_group(b, nchars, nbytes, k):
    """k sentences with nchars characters and nbytes bytes in all."""
    per_c = _split(nchars, k, b.rng)
    extra = nbytes - nchars
    assert 0 <= extra <= 3 * nchars
    sents = []
    for c in per_c:
        take = min(extra, 3 * c)
        extra -= take
        sents.append(b.compose(c, c + take))
    return sents


def _split(total, parts, rng, lo=1):
    """`parts` positive integers >= lo that add up to total."""
    assert total >= lo * parts
    cuts = np.sort(rng.choice(total - lo * parts + parts - 1, size=parts - 1, replace=False)) if parts > 1 else np.array([], np.int64)
    sizes = np.diff(np.concatenate([[-1], cuts, [total - lo * parts + parts - 1]])) - 1 + lo
    assert sizes.sum() == total and sizes.min() >= lo
    return [int(x) for x in sizes]


def is_fast(got, offs, nch):
    return got[0] == "fast"


def is_one_range(got, offs, nch):
    return got[0] == "ranges" and got[1] == [(0, len(nch), False)]


def first_range_ends(k):
    def f(got, offs, nch):
        return got[0] == "ranges" and got[1][0] == (0, k, False) and len(got[1]) > 1
    return f


def slow(got, offs, nch):
    return got[0] == "ranges"


def single_at(k0):
    def f(got, offs, nch):
        return got[0] == "ranges" and any(r == (k0, k0 + 1, True) for r in got[1])
    return f


def range_at(k0):
    def f(got, offs, nch):
        return got[0] == "ranges" and any(r[0] == k0 and not r[2] for r in got[1]) and not any(r[2] for r in got[1])
    return f


# ---- the edge groups -------------------------------------------------------------------------------------------

def slot_edges(b: EdgeBatch):
    """Groups of 1-byte characters with S = limit - 1, limit, limit + 1 slots (the text is far below its cap)."""
    pl, gap = b.plan, b.plan["gap"]
    lim = slot_limit(pl)
    fits = is_fast if pl["kernel"] == "k_fused" else is_one_range
    for d in (-1, 0, 1):
        S = lim + d
        sizes = _split(S - gap * (GROUP + 1), GROUP, b.rng)
        sents = [b.chars(n, (1,)) for n in sizes]
        b.add(sents, f"slots S = limit{d:+d}", fits if d <= 0 else slow)


def text_edges(b: EdgeBatch):
    """Groups whose text span is the last 16-byte unit that fits and the first that does not, with off[0] % 16 in
    {0, 1, 15}.  Not reachable for k_tile_fast with valid text and no trimmed line terminators: its text cap needs more
    characters than its slot cap holds (invalid sentences count no characters, trimmed bytes count in the span)."""
    pl, gap = b.plan, b.plan["gap"]
    if pl["kernel"] == "k_tile_fast":
        assert (pl["text_cap"] - 16 - 15) > 4 * (slot_limit(pl) - gap * 2), "k_tile_fast text edge became reachable"
        return
    fits = is_fast
    for lo in (0, 1, 15):
        for d in (0, 1):
            b.pad_to(lo)
            nbytes = pl["text_cap"] - 16 - lo + d   # end - a0 = text_cap - 16 (+1)
            # as few characters as the bytes allow (4-byte characters), so that the slot test passes
            nch_total = min(slot_limit(pl) - gap * (GROUP + 1) - 1, nbytes)
            nch_total = max(nch_total - 64, (nbytes + 3) // 4)
            sents = _compose_group(b, nch_total, nbytes, GROUP)
            b.add(sents, f"text span {'+1' if d else 'at the cap'}, off[0] % 16 = {lo}", fits if d == 0 else slow)


def split_edges(b: EdgeBatch):
    """Slow-path groups whose first range fills the slot limit exactly, followed by the rest of the group, and
    single sentences of exactly one range and one slot more (the one-warp walk)."""
    pl, gap = b.plan, b.plan["gap"]
    lim = slot_limit(pl)
    k = 40
    sizes = _split(lim - gap * (k + 1), k, b.rng)
    sents = [b.chars(n, (1, 3)) for n in sizes] + [b.chars(int(b.rng.integers(20, 60)), (1, 3)) for _ in range(GROUP - k)]
    b.add(sents, "first range at the slot limit", first_range_ends(k))
    # text: the first range's span exactly at the cap (fused only, see text_edges)
    if pl["kernel"] == "k_fused":
        b.pad_to(0)
        nbytes = pl["text_cap"] - 16
        k = 32
        nch = (nbytes + 3) // 4 + 40
        sents = _compose_group(b, nch, nbytes, k)
        sents += [b.chars(int(b.rng.integers(20, 60)), (3,)) for _ in range(GROUP - k)]
        b.add(sents, "first range at the text cap", first_range_ends(k))
    # one sentence of exactly one range (gap + n + gap = limit), and one slot more
    for d in (0, 1):
        n = lim - 2 * gap + d
        for pos in (0, 17):
            sents = [b.chars(int(b.rng.integers(5, 30)), (1, 3)) for _ in range(GROUP)]
            sents[pos] = b.chars(n, (1,))
            b.add(sents, f"sentence of one range{' + 1 slot' if d else ''} at {pos}", single_at(pos) if d else range_at(pos))


def _sizes_around(b: EdgeBatch, S, spans):
    """GROUP sentence sizes (characters) that fill a tile of exactly S slots and keep every slot span [f, f + n) of
    `spans` inside one sentence (no sentence end, no separator slot inside a span)."""
    gap = b.plan["gap"]
    spans = sorted(spans)
    sizes, cur = [], gap            # cur: slot of the next sentence's first character
    for k in range(GROUP):
        left = GROUP - k
        if left == 1:
            e = S - gap
        else:
            avg = (S - gap - cur - gap * (left - 1)) / left
            e = cur + max(1, int(round(avg * (b.rng.uniform(0.8, 1.2) if left > 4 else 1.0))))
            moved = True
            while moved:
                moved = False
                for f, n in spans:
                    if f < e + gap and e < f + n:          # the end or the separator slots would cut the span
                        e = f - gap if f - gap > cur else f + n
                        moved = True
        for f, n in spans:
            assert not (cur <= f < e) or f + n <= e, "span cut by a sentence end"
            assert not (e <= f < e + gap), "span on separator slots"
        assert e > cur, "no room left for the remaining sentences"
        sizes.append(e - cur)
        cur = e + gap
    assert sum(sizes) + gap * (GROUP + 1) == S
    return sizes


def word_edges(b: EdgeBatch, words):
    """Fast-path groups (k_fused) or one-range groups (k_tile_fast) in which long patterns (dictionary words, long
    n-grams) start at the tile's first character, end at its last one, and sit at every warp's range start
    (R = ceil(S / 8); k_fused re-reads HALO slots in front of it): starting 1 slot before it, ending on it, starting
    at the first halo slot and one slot before the halo, one placement per group.  Every word is checked in place."""
    pl, gap = b.plan, b.plan["gap"]
    words = [w for w in words if 4 <= len(w) <= 12]
    if not words:
        assert pl["deep"] == 0 and not pl["overflow"], "a model with long patterns needs some to place"
        return
    fits = is_fast if pl["kernel"] == "k_fused" else is_one_range
    wi = 0

    def nxt():
        nonlocal wi
        wi += 1
        return words[(wi - 1) % len(words)]
    for S in (slot_limit(pl) // 2, slot_limit(pl)):
        R = (S + WARPS - 1) // WARPS
        for where in ("start - 1", "end on start", "halo start", "halo start - 1"):
            w_first, w_last = nxt(), nxt()
            place = [(gap, w_first), (S - gap - len(w_last), w_last)]   # the tile's first / last characters
            for wv in range(1, WARPS):
                w = nxt()
                back = {"start - 1": 1, "end on start": len(w) - 1, "halo start": HALO, "halo start - 1": HALO + 1}[where]
                place.append((wv * R - back, w))
            sizes = _sizes_around(b, S, [(f, len(w)) for f, w in place])
            first = gap * (np.arange(GROUP) + 1) + np.concatenate([[0], np.cumsum(sizes)[:-1]])   # slot of each sentence's first character
            sents = [list(b.chars(n, (1, 2, 3))) for n in sizes]
            at = []
            for f, w in place:
                k = int(np.searchsorted(first, f, side="right")) - 1
                j = f - int(first[k])
                assert 0 <= j and j + len(w) <= sizes[k]
                sents[k][j:j + len(w)] = list(w)
                at.append((k, j, w))
            for k, j, w in at:  # no placement overwrote another
                assert "".join(sents[k][j:j + len(w)]) == w
            b.add(["".join(x) for x in sents], f"long words at tile and warp edges ({where}), S = {S}", fits)


def build(plan, alphabet, words, n_groups, seed=0, tail=63, every=12):
    """A batch of at least n_groups groups: the edge groups above, repeated all through the batch with `every` filler
    groups in front of each maker (so that every round of groups over the sub-blocks holds edge and slow-path groups),
    ending with a partial group of `tail` sentences."""
    b = EdgeBatch(plan, alphabet, seed)
    makers = [slot_edges, text_edges, split_edges, lambda x: word_edges(x, words)]
    while True:
        for mk in makers:
            b.filler(every)
            mk(b)
        if len(b.sents) // GROUP >= n_groups:
            break
    if tail:
        b.add([b.chars(int(b.rng.integers(1, 50)), (1, 2, 3, 4)) for _ in range(tail)], f"partial last group of {tail}")
    return b


# ---- models that reach every kernel variant --------------------------------------------------------------------

ALPHABET = "あいうえおかきくけこアイウエオ人火星地球猫社長aB1。、éß𠀋𩸽"


def variant_model(cw, tw, ng_lens, dict_lens, tags=0, seed=1):
    """(model bytes, long patterns): char n-grams of the given lengths and dictionary words of the given lengths over
    ALPHABET, every type n-gram up to length 3, `tags` tag models."""
    from .bincode_model import encode_model
    rng = np.random.default_rng(seed)
    alpha = list(ALPHABET)

    def word(n):
        return "".join(rng.choice(alpha, size=n))
    cng = {}
    for n in ng_lens:
        for _ in range(60):
            cng[word(n)] = rng.integers(-3000, 3000, size=max(2 * cw - n + 1, 0)).tolist()
    dic = {}
    for n in dict_lens:
        for _ in range(20):
            dic[word(n)] = None
    dic = [(w, rng.integers(-3000, 3000, size=len(w) + 1).tolist(), "") for w in dic]
    tng = {}
    for n in (1, 2, 3):
        if n <= 2 * tw:
            for k in range(6 ** n):
                tng[bytes(1 + (k // 6 ** j) % 6 for j in range(n))] = rng.integers(-3000, 3000, size=2 * tw - n + 1).tolist()
    tms = []
    for t in range(tags):
        cn = [(word(int(rng.integers(1, 4))), [(int(rng.integers(0, cw + 1)), rng.integers(-99, 99, size=2).tolist())])
              for _ in range(5)]
        tn = [(bytes(rng.integers(1, 7, size=int(rng.integers(1, 4))).tolist()),
               [(int(rng.integers(0, tw + 1)), rng.integers(-99, 99, size=2).tolist())]) for _ in range(3)]
        tms.append(dict(token=word(2) + str(t), tags=[["x", "y"]], char_ngrams=cn, type_ngrams=tn, bias=[1, 2]))
    mb = encode_model(dict(char_ngrams=list(cng.items()), type_ngrams=list(tng.items()), dict=dic, bias=int(rng.integers(-500, 500)),
                           char_window=cw, type_window=tw, tag_models=tms))
    return mb, [w for w in list(cng) + [d[0] for d in dic] if len(w) >= 4]


PLAN_KEYS = ("kernel", "seeds_smem", "common_shape", "deep", "states", "r0_fixed", "general", "split3", "overflow")


def plan_key(plan):
    return tuple(plan[k] for k in PLAN_KEYS)


def all_plan_keys():
    """Every variant the dispatch can launch: the 24 of k_fused and the 20 instantiations of k_tile_fast."""
    keys = set()
    for seeds in (0, 1):
        for common in (0, 1):
            for deep in (0, 1, 2):
                for states in (0, 1):
                    keys.add(("k_fused", seeds, common, deep, states, 0, 0, 0, 0))
        for split3 in (0, 1):
            for r0 in (0, 1):
                for ovf in (0, 1):
                    keys.add(("k_tile_fast", seeds, 0, 0, 0, r0, 0, split3, ovf))
            keys.add(("k_tile_fast", seeds, 0, 0, 0, 0, 1, split3, 0))
    return keys


# k_tile_fast with the window start -3 compiled in: a model with r0 = -3 and inline rows has lag 3 and a type window of
# at most 3, so it always passes k_fused's shape test (the only other refusal, pattern-id states of a char table with no
# patterns, needs a char table without patterns, which is never built).
UNREACHABLE = {k: "r0 = -3 with inline rows always takes k_fused" for k in all_plan_keys() if k[0] == "k_tile_fast" and k[5]}


def variant_recipes():
    """(name, VPT_SEED_BUDGET or None, model arguments, predict_tags, with_states, expected plan key)."""
    out = []
    for seeds, budget in ((1, None), (0, "3")):
        for common, (cw, tw) in ((1, (3, 3)), (0, (2, 2))):
            for deep, ng, dl in ((0, (1, 2, 3), ()), (1, (1, 2, 3, 4), ()), (2, (1, 2, 3), (4, 6, 8, 9))):
                for states in (0, 1):
                    name = f"fused-{'smem' if seeds else 'gmem'}-{'common' if common else 'other'}-deep{deep}-{'states' if states else 'plain'}"
                    out.append((name, budget, (cw, tw, ng, dl, 2), True, bool(states),
                                ("k_fused", seeds, common, deep, states, 0, 0, 0, 0)))
        for split3, (cw, tw, ng) in ((1, (4, 3, (3, 4, 5))), (0, (5, 2, (5, 6)))):
            for ovf, dl in ((0, ()), (1, (8, 9, 10))):
                name = f"tile-{'smem' if seeds else 'gmem'}-{'split3' if split3 else 'nosplit'}-{'overflow' if ovf else 'inline'}"
                out.append((name, budget, (cw, tw, ng, dl, 0), False, False, ("k_tile_fast", seeds, 0, 0, 0, 0, 0, split3, ovf)))
            name = f"tile-{'smem' if seeds else 'gmem'}-{'split3' if split3 else 'nosplit'}-general"
            out.append((name, budget, (4, 3 if split3 else 2, (1, 2, 3), (), 0), False, False,
                        ("k_tile_fast", seeds, 0, 0, 0, 0, 1, split3, 0)))
    return out
