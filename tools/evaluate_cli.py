#!/usr/bin/env python
"""The reference's `evaluate` command (evaluate/src/main.rs) on top of the evaluate line stream (vpt_line_stream_*, the
loop of vpt_evaluate_lines fed in pieces): a gold corpus in the tokenized
format on stdin, precision / recall / F1 on stdout, everything between the two (line splitting, gold parsing, full-width
pre-filter, scoring, --wsconst post-filters, tag prediction, both metrics) on the GPU.

    python tools/evaluate_cli.py --model model.bin[.zst] [--predict-tags] [--wsconst K] ... [--no-norm] \\
        [--metric char|word] < gold.tok
"""
import argparse
import decimal
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
READ_BYTES = 16 << 20  # largest piece read from stdin at once: a corpus of any size is evaluated in bounded memory


def rust_f64(x: float) -> str:
    """Rust's `Display` for f64 (what `println!("{}")` prints): the shortest digits that round-trip, never in exponent
    form ("1", "0.5", "0.000005", "10000000000000000"), "NaN", "inf", "-inf"."""
    if math.isnan(x):
        return "NaN"
    if math.isinf(x):
        return "inf" if x > 0 else "-inf"
    s = format(decimal.Decimal(repr(x)), "f")  # repr: shortest round-trip digits; Decimal 'f': no exponent
    if "." in s:
        s = s.rstrip("0").rstrip(".")
    return s


def ratio(a: float, b: float) -> float:
    """a / b in f64 as Rust computes it: 0 / 0 is NaN, x / 0 is inf."""
    if b == 0:
        return math.nan if a == 0 or math.isnan(a) else math.copysign(math.inf, a)
    return a / b


def report(counts: dict, metric: str) -> str:
    """The lines main.rs:140-143 (char) or :188-190 (word) print."""
    if metric == "char":
        tp, tn, fp, fn = (counts[k] for k in ("tp", "tn", "fp", "fn"))
        precision = ratio(float(tp), float(tp + fp))
        recall = ratio(float(tp), float(tp + fn))
    else:
        precision = ratio(float(counts["n_cor"]), float(counts["n_sys"]))
        recall = ratio(float(counts["n_cor"]), float(counts["n_ref"]))
    f1 = ratio(2.0 * precision * recall, precision + recall)
    out = f"Precision: {rust_f64(precision)}\nRecall: {rust_f64(recall)}\nF1: {rust_f64(f1)}\n"
    if metric == "char":
        out += f"TP: {tp}, TN: {tn}, FP: {fp}, FN: {fn}\n"
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description="A program to evaluate the accuracy of Vaporetto (vaporetto_b200).")
    ap.add_argument("--model", required=True, help="The model file to use when analyzing text (raw or zstd)")
    ap.add_argument("--predict-tags", action="store_true", help="Predicts POS tags")
    ap.add_argument("--wsconst", action="append", default=[], choices=list("DRHTKOG"),
                    help="Do not segment some character types: D Digit, R Roman, H Hiragana, T Katakana, K Kanji, O Other, G Grapheme cluster")
    ap.add_argument("--no-norm", action="store_true", help="Do not normalize input strings before prediction")
    ap.add_argument("--metric", choices=["char", "word"], default="char",
                    help="Evaluation metric: char evaluates each character boundary; word evaluates each word (Nagata's method)")
    ap.add_argument("--device", type=int, default=0, help="CUDA device ordinal")
    args = ap.parse_args(argv)

    import vaporetto_b200 as vb
    print("Loading model file...", file=sys.stderr)
    with open(args.model, "rb") as f:
        model = vb.Model.read_zstd(f.read())
    predictor = vb.Predictor(model, predict_tags=args.predict_tags, device=args.device)
    print("Start tokenization", file=sys.stderr)
    try:
        with predictor.line_stream("evaluate", no_norm=args.no_norm, wsconst="".join(args.wsconst),
                                   predict_tags=args.predict_tags) as stream:
            while True:
                data = sys.stdin.buffer.read1(READ_BYTES)
                if not data:
                    break
                stream.feed(data)
            counts = stream.finish()
    except vb.VaporettoError as e:
        print(f"Error: {e}", file=sys.stderr)
        return 1
    sys.stdout.write(report(counts, args.metric))
    return 0


if __name__ == "__main__":
    sys.exit(main())
