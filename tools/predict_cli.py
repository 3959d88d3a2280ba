#!/usr/bin/env python
"""The reference's `predict` command (predict/src/main.rs) on top of the line stream (vpt_line_stream_*, the loop of
vpt_tokenize_lines fed in pieces): stdin lines -> space-separated tokens on stdout, everything between the two (line
splitting, full-width pre-filter, scoring, --wsconst post-filters, output text) on the GPU.

    python tools/predict_cli.py --model model.bin[.zst] [--no-norm] [--wsconst D] [--wsconst R] ... \
        [--predict-tags] [--scores] [--tag-scores] < in.txt > out.txt

Input of any size is read in pieces of up to 16 MiB, and the output is written as it comes: memory does not grow with the
input.  When nothing more is waiting on stdin, the output of every complete line read so far is written and flushed, so
an interactive session or a slow producer gets each line back as soon as it is entered, as with the reference.

--scores and --tag-scores print the reference's dumps behind each token line, written on the device as well
(vpt_line_stream_new_scores): every boundary's characters and score, and every token's tag candidates with their scores.
Three differences from the reference, where it panics or prints stale data: --tag-scores needs --predict-tags (the
parser reports an error; the reference panics, as it does for a model without tag slots, which the library refuses); a
rejected line (empty, NUL, invalid UTF-8) prints the tag block " " + two newlines, without the stale candidates the
reference copies from an earlier line; a token whose tag slots list more candidates than its score vector holds prints
its surface alone.  For tag candidate scores as data, call the library: Predictor.predict_batch_compact(...,
tags=True, tag_scores=True) or Predictor.token_spans(..., tags=True, tag_scores=True) and the result's
tag_candidates(r) for a batch, Predictor.store_tag_scores(True) + Token.tag_candidates() for one sentence.

--tag-rules FILE is an extension: the reference CLI has no such option.  With --predict-tags it runs vaporetto_rules'
PatternMatchTagger right after the tag prediction: every tag slot the model left empty for a token whose surface has
a rule gets the rule's tag.  FILE holds one rule per line, written as one token of the tokenized format
(Sentence::from_tokenized): `surface/tag1//tag3`, '\' escaping the next character; an empty tag field leaves its slot
alone.  Unless --no-norm, tokens are matched by their full-width-normalised form, so write full-width surfaces.

--partial-annotation is an extension as well: stdin holds partially annotated lines in the format of the reference's
Sentence::from_partial_annotation (the train CLI's --part corpora: '|' a boundary, '-' none, ' ' for the model to
decide, after every character but the last).  The model predicts the rest, --wsconst runs, then the given markers win;
tags follow with --predict-tags (input tags are dropped).  An empty line gives an empty line; a malformed line stops the
command with its 0-based line number (vpt_line_stream_new_partial).  It cannot be combined with --scores or
--tag-scores.

--write-partial-annotation is an extension too: the output lines are in the format of the reference's
Sentence::write_partial_annotation_text ('|' a boundary, '-' none, ' ' unknown, tags unescaped), and --margin N leaves
every boundary whose score lies strictly between -N and N unknown for an annotator to resolve (default 0: none); tokens
next to an unknown boundary get no tags (vpt_line_stream_new_annotate).  It cannot be combined with --scores or
--tag-scores.

--partial-annotation --write-partial-annotation re-annotates a partially annotated corpus, the second round of the
domain-adaptation loop: the given '|' / '-' and every character's input tags are written back as given, the model
decides each ' ' and leaves open those scoring strictly between -N and N (--margin N); --drop-input-tags drops the
input tags instead, so that --predict-tags may fill them again (vpt_line_stream_new_reannotate)."""
import argparse
import os
import select
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

READ_BYTES = 16 << 20  # largest piece read from stdin at once


def input_waiting(f) -> bool:
    """Whether more input can be read from `f` without waiting (a full pipe, a file); False where that cannot be told."""
    try:
        return bool(select.select([f], [], [], 0)[0])
    except (OSError, ValueError):
        return False


def read_model(path: str) -> bytes:
    """The CLI reads a zstd-compressed model (main.rs:110-111); the library decodes it (vpt_model_read_zstd)."""
    with open(path, "rb") as f:
        return f.read()


def parse_tag_rule(line: str, lineno: int):
    """One line of a --tag-rules file -> (surface, [tag or None per slot]), as Sentence::from_tokenized reads a token
    (sentence.rs:285-467): '\\' escapes the next character, '/' starts a tag, an empty tag is None.  A second token
    (an unescaped ' ') or an empty surface is an error naming the line (1-based)."""
    fields, cur, escape = [], [], False
    for c in line:
        if escape:
            cur.append(c)
            escape = False
        elif c == "\\":
            escape = True
        elif c == "/":
            fields.append("".join(cur))
            cur = []
        elif c == " ":
            raise ValueError(f"--tag-rules line {lineno}: one token per line (found a space)")
        else:
            cur.append(c)
    fields.append("".join(cur))
    if not fields[0]:
        raise ValueError(f"--tag-rules line {lineno}: empty surface")
    return fields[0], [t if t else None for t in fields[1:]]


def read_tag_rules(path: str) -> dict:
    """The rules of a --tag-rules file (UTF-8, one rule per line; a line break ends a rule, '\\r\\n' included; a
    surface given twice is an error, as a HashMap holds one entry per key)."""
    rules = {}
    with open(path, "rb") as f:
        for i, raw in enumerate(f.read().decode("utf-8").splitlines(), 1):
            surface, tags = parse_tag_rule(raw, i)
            if surface in rules:
                raise ValueError(f"--tag-rules line {i}: duplicate surface")
            rules[surface] = tags
    return rules


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description="A program to perform word segmentation (vaporetto_b200).")
    ap.add_argument("--model", required=True, help="The model file to use when analyzing text")
    ap.add_argument("--wsconst", action="append", default=[], choices=list("DRHTKOG"),
                    help="Do not segment some character types: D Digit, R Roman, H Hiragana, T Katakana, K Kanji, O Other, G Grapheme cluster")
    ap.add_argument("--predict-tags", action="store_true", help="Predicts POS tags")
    ap.add_argument("--scores", action="store_true", help="Prints boundary scores")
    ap.add_argument("--tag-scores", action="store_true", help="Prints tag scores (needs --predict-tags)")
    ap.add_argument("--no-norm", action="store_true", help="Do not normalize input strings before prediction")
    ap.add_argument("--tag-rules", metavar="FILE",
                    help="Extension (not in the reference CLI): PatternMatchTagger rules, one `surface/tag1//tag3` per "
                         "line, filling the tags the model leaves empty; needs --predict-tags")
    ap.add_argument("--partial-annotation", action="store_true",
                    help="Extension: the input lines are partially annotated ('|' boundary, '-' none, ' ' unknown); "
                         "the given markers are kept, the model decides the rest")
    ap.add_argument("--write-partial-annotation", action="store_true",
                    help="Extension: write partially annotated lines ('|' boundary, '-' none, ' ' unknown)")
    ap.add_argument("--drop-input-tags", action="store_true",
                    help="With --partial-annotation --write-partial-annotation: drop the input's tags instead of "
                         "writing them back")
    ap.add_argument("--margin", type=int, default=0, metavar="N",
                    help="With --write-partial-annotation: boundaries scoring strictly between -N and N stay unknown")
    ap.add_argument("--device", type=int, default=0, help="CUDA device ordinal")
    args = ap.parse_args(argv)
    if args.tag_rules and not args.predict_tags:
        ap.error("--tag-rules needs --predict-tags")
    if args.tag_scores and not args.predict_tags:
        ap.error("--tag-scores needs --predict-tags")
    if args.partial_annotation and (args.scores or args.tag_scores):
        ap.error("--partial-annotation cannot be combined with --scores or --tag-scores")
    if args.write_partial_annotation and (args.scores or args.tag_scores):
        ap.error("--write-partial-annotation cannot be combined with --scores or --tag-scores")
    if args.drop_input_tags and not (args.partial_annotation and args.write_partial_annotation):
        ap.error("--drop-input-tags needs --partial-annotation and --write-partial-annotation")
    if args.margin and not args.write_partial_annotation:
        ap.error("--margin needs --write-partial-annotation")
    if not 0 <= args.margin <= 2**31 - 1:
        ap.error("--margin must be in 0..2147483647")
    rules = None
    if args.tag_rules:
        try:
            rules = read_tag_rules(args.tag_rules)
        except (ValueError, UnicodeDecodeError) as e:
            ap.error(str(e))

    import vaporetto_b200 as vb
    print("Loading model file...", file=sys.stderr)
    predictor = vb.Predictor(vb.Model.read_zstd(read_model(args.model)), predict_tags=args.predict_tags, device=args.device)
    tagger = vb.PatternMatchTagger(predictor, rules) if rules is not None else None
    print("Start tokenization", file=sys.stderr)
    inp, out = sys.stdin.buffer, sys.stdout.buffer
    t0 = time.perf_counter()
    kind = ("reannotate" if args.partial_annotation and args.write_partial_annotation else
            "partial" if args.partial_annotation else "annotate" if args.write_partial_annotation else "tokenize")
    with predictor.line_stream(kind=kind, no_norm=args.no_norm, wsconst="".join(args.wsconst), predict_tags=args.predict_tags,
                               tag_rules=tagger, scores=args.scores, tag_scores=args.tag_scores,
                               margin=args.margin, keep_tags=not args.drop_input_tags) as stream:
        while True:
            data = inp.read1(READ_BYTES)
            if not data:
                break
            out.write(stream.feed(data))
            if len(data) < READ_BYTES and not input_waiting(inp):
                # nothing more has arrived: hand back every complete line now (an interactive session, a slow producer)
                out.write(stream.flush())
                out.flush()
        rest, _ = stream.finish()
        out.write(rest)
    dt = time.perf_counter() - t0
    out.flush()
    print(f"Elapsed: {dt} [sec]", file=sys.stderr)
    return 0


if __name__ == "__main__":
    sys.exit(main())
