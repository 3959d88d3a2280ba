"""CPU restatement of the reference's `evaluate` command (evaluate/src/main.rs:69-195) and of the tokenized-text parser
it calls (`Sentence::parse_tokenized`, sentence.rs:285-406), for the tests of vpt_evaluate_lines.

TEST INFRASTRUCTURE ONLY.  Prediction comes from the CPU oracle's restatement of the `predict` CLI loop
(OraclePredictor.tokenize_lines, same pre-filter, post-filters and tag prediction); the metric is main.rs's own loop,
with per-sentence vectors, the sequential `matched` flag and list-of-Optional equality of the tags, so the device's
per-position reformulation is checked against the original loop.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

INVALID_ARGUMENT = 2
IO_ERROR = 5


class GoldError(Exception):
    """An error that stops the CLI: code (VaporettoError code), message as vpt_evaluate_lines words it, line index."""

    def __init__(self, code: int, msg: str, line: Optional[int] = None):
        super().__init__(msg)
        self.code, self.msg, self.line = code, msg, line


def _tok_err(what: str) -> GoldError:
    return GoldError(INVALID_ARGUMENT, "InvalidArgumentError: tokenized_text: " + what)


def parse_tokenized(line: str) -> Tuple[str, List[int], List[List[Optional[str]]]]:
    """Sentence::from_tokenized (sentence.rs:285-467): (raw text, boundaries (1 = WordBoundary), tags per character,
    each list n_tags long).  One documented difference: a line that yields no character (a lone '\\') is the
    "must contain at least one character" error; the reference divides by zero at sentence.rs:450."""
    if not line:
        raise _tok_err("must contain at least one character")
    text: List[str] = []
    boundaries: List[int] = []
    tag_str: Optional[List[str]] = None
    prev_boundary = False
    escape = False
    tags_tmp: List[List[str]] = []
    for c in line:
        if not escape and c == "\\":
            escape = True
        elif not escape and c == " ":
            if not text:
                raise _tok_err("must not start with a whitespace")
            if prev_boundary:
                raise _tok_err("must not contain consecutive whitespaces")
            if tag_str is not None:
                tags_tmp[-1].append("".join(tag_str))
                tag_str = None
            prev_boundary = True
        elif not escape and c == "/":
            if not text or prev_boundary:
                raise _tok_err("a slash must follow a character")
            if tag_str is not None:
                tags_tmp[-1].append("".join(tag_str))
            tag_str = []
        else:
            escape = False
            if c == "\0":
                raise _tok_err("must not contain NULL")
            if tag_str is not None:
                tag_str.append(c)
                continue
            if text:
                boundaries.append(1 if prev_boundary else 0)
            prev_boundary = False
            text.append(c)
            tags_tmp.append([])
    if prev_boundary:
        raise _tok_err("must not end with a whitespace")
    if tag_str is not None:
        tags_tmp[-1].append("".join(tag_str))
    if not text:
        raise _tok_err("must contain at least one character")
    n_tags = max(len(x) for x in tags_tmp)
    tags = [[t if t else None for t in ts] + [None] * (n_tags - len(ts)) for ts in tags_tmp]
    return "".join(text), boundaries, tags


def bufread_lines(data: bytes) -> List[bytes]:
    """BufRead::lines: split at '\\n', drop one '\\r' before it; a final line without '\\n' keeps its bytes."""
    if not data:
        return []
    parts = data.split(b"\n")
    if parts[-1] == b"":
        parts.pop()
        return [p[:-1] if p.endswith(b"\r") else p for p in parts]
    return [p[:-1] if p.endswith(b"\r") else p for p in parts[:-1]] + [parts[-1]]


def _system(oracle, raw: str, no_norm: bool, wsconst: str, predict_tags: bool):
    """predict + post-filters (+ fill_tags) of one sentence, read back from the predict CLI restatement's output:
    (boundaries, tags per character as fill_tags leaves them: n_tags slots, or None when fill_tags did not run)."""
    out, _ = oracle.tokenize_lines(raw.encode("utf-8"), no_norm=no_norm, wsconst=wsconst, predict_tags=predict_tags)
    assert out.endswith(b"\n")
    text, bounds, tags = parse_tokenized(out[:-1].decode("utf-8"))
    assert text == raw
    if not (predict_tags and oracle.n_tags > 0):
        return bounds, None
    k = oracle.n_tags
    # write_tokenized_text prints the slots up to the last one with a tag; fill_tags made k slots per character
    return bounds, [t[:k] + [None] * (k - len(t)) for t in tags]


def evaluate_lines(oracle, data: bytes, no_norm: bool = False, wsconst: str = "", predict_tags: bool = False):
    """main.rs:86-192 over `data` -> (counts dict as vpt_evaluate_lines returns it, per-line [tp, tn, fp, fn, n_sys,
    n_ref, n_cor] lists).  Raises GoldError for the first bad line."""
    lines = bufread_lines(data)
    per_line = []
    results = []
    for i, b in enumerate(lines):
        try:
            line = b.decode("utf-8")
        except UnicodeDecodeError:
            raise GoldError(IO_ERROR, f"stream did not contain valid UTF-8 (line {i})", i)
        if not line:
            per_line.append(None)
            continue
        try:
            raw, ref_b, tags = parse_tokenized(line)
        except GoldError as e:
            raise GoldError(e.code, f"{e.msg} (line {i})", i)
        ref_t = tags
        # unless --no-norm the sentence is rebuilt from the filtered raw text: no tags (n_tags 0)
        sys_t = tags if no_norm else [[] for _ in tags]
        sys_b, filled = _system(oracle, raw, no_norm, wsconst, predict_tags)
        if filled is not None:
            sys_t = filled
        per_line.append(len(results))
        results.append((ref_b, ref_t, sys_b, sys_t))
    counts = {"n_lines": len(lines), "n_sentences": len(results)}
    counts.update(char_metric(results))
    counts.update(word_metric(results))
    rows = []
    for r in per_line:
        if r is None:
            rows.append([0] * 7)
        else:
            c = char_metric([results[r]])
            w = word_metric([results[r]])
            rows.append([c["tp"], c["tn"], c["fp"], c["fn"], w["n_sys"], w["n_ref"], w["n_cor"]])
    return counts, rows


def char_metric(results) -> dict:
    """main.rs:121-139."""
    n_tp = n_tn = n_fp = n_fn = 0
    for rs_b, _, hs_b, _ in results:
        for r, h in zip(rs_b, hs_b):
            if r == h:
                if h == 1:
                    n_tp += 1
                else:
                    n_tn += 1
            elif h == 1:
                n_fp += 1
            else:
                n_fn += 1
    return {"tp": n_tp, "tn": n_tn, "fp": n_fp, "fn": n_fn}


def word_metric(results) -> dict:
    """main.rs:149-184 (Nagata 1994)."""
    n_sys = n_ref = n_cor = 0
    for refs_b, refs_t, syss_b, syss_t in results:
        matched = True
        for r_b, r_t, s_b, s_t in zip(refs_b, refs_t, syss_b, syss_t):
            if r_b == s_b:
                if s_b == 1:
                    if matched and r_t == s_t:
                        n_cor += 1
                    matched = True
                    n_ref += 1
                    n_sys += 1
            else:
                if s_b == 1:
                    n_sys += 1
                else:
                    n_ref += 1
                matched = False
        if matched and refs_t[-1] == syss_t[-1]:
            n_cor += 1
        n_sys += 1
        n_ref += 1
    return {"n_sys": n_sys, "n_ref": n_ref, "n_cor": n_cor}
