#!/usr/bin/env python
"""The reference's `predict` command (predict/src/main.rs) on top of the line stream (vpt_line_stream_*, the loop of
vpt_tokenize_lines fed in pieces): stdin lines -> space-separated tokens on stdout, everything between the two (line
splitting, full-width pre-filter, scoring, --wsconst post-filters, output text) on the GPU.

    python tools/predict_cli.py --model model.bin[.zst] [--no-norm] [--wsconst D] [--wsconst R] ... < in.txt > out.txt

Input of any size is read in pieces of up to 16 MiB, and the output is written as it comes: memory does not grow with the
input.  When nothing more is waiting on stdin, the output of every complete line read so far is written and flushed, so
an interactive session or a slow producer gets each line back as soon as it is entered, as with the reference.

Options not on the device path (--scores, --tag-scores) are rejected; use the Sentence API
(vaporetto_b200.Sentence / include/vaporetto_b200.hpp) for tags."""
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


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description="A program to perform word segmentation (vaporetto_b200).")
    ap.add_argument("--model", required=True, help="The model file to use when analyzing text")
    ap.add_argument("--wsconst", action="append", default=[], choices=list("DRHTKOG"),
                    help="Do not segment some character types: D Digit, R Roman, H Hiragana, T Katakana, K Kanji, O Other, G Grapheme cluster")
    ap.add_argument("--predict-tags", action="store_true", help="Predicts POS tags")
    ap.add_argument("--no-norm", action="store_true", help="Do not normalize input strings before prediction")
    ap.add_argument("--device", type=int, default=0, help="CUDA device ordinal")
    args = ap.parse_args(argv)

    import vaporetto_b200 as vb
    print("Loading model file...", file=sys.stderr)
    predictor = vb.Predictor(vb.Model.read_zstd(read_model(args.model)), predict_tags=args.predict_tags, device=args.device)
    print("Start tokenization", file=sys.stderr)
    inp, out = sys.stdin.buffer, sys.stdout.buffer
    t0 = time.perf_counter()
    with predictor.line_stream(no_norm=args.no_norm, wsconst="".join(args.wsconst), predict_tags=args.predict_tags) as stream:
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
