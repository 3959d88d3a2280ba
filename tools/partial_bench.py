#!/usr/bin/env python
"""Cost of vpt_tokenize_partial_lines next to vpt_tokenize_lines on the same raw text, in one process.

A synthetic model with tag models and text of the benchmark's config-2 shape (tests/vpt_testlib/synth.py, seeded: lines
of 40 characters) give the raw lines (at least --mb MB); the partially annotated input is the same lines with every
marker ' ' (0 % given) or every marker from the model's own segmentation (100 % given).  After a warm-up, the calls
alternate for --reps rounds, tags off and on; the script prints the median seconds of each, the rates in GB/s of the
call's input, and the card's name, power limit and max SM clock.  It also times the per-sentence host path the device
call replaces (Sentence.from_raw + predict + boundaries set by hand + fill_tags + write_tokenized_text) on a sample of
--host-lines lines.

    python tools/partial_bench.py [--mb 100] [--reps 5] [--host-lines 2000]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().split(", ") + ["", "", ""])[:3]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def annotate_all(tokenized: bytes) -> bytes:
    """Every marker given: '-' inside a token, '|' between tokens, from tokenize_lines output without tags."""
    out = []
    for line in tokenized.decode().split("\n")[:-1]:
        toks, cur, esc = [], [], False
        for c in line:
            if esc:
                cur.append(c)
                esc = False
            elif c == "\\":
                esc = True
            elif c == " ":
                toks.append("".join(cur))
                cur = []
            else:
                cur.append(c)
        toks.append("".join(cur))
        out.append("|".join("-".join(t) for t in toks))
    return ("\n".join(out) + "\n").encode()


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=100.0, help="size of the raw text in MB (at least)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-lines", type=int, default=2000)
    args = ap.parse_args(argv)

    import numpy as np
    import vaporetto_b200 as vb
    from vpt_testlib import synth
    mb = synth.gen_model_bccwj_shaped(n_patterns=100_000, sample_sentences=200_000, tag_models=2_000)
    p = vb.Predictor(vb.Model.read(mb), predict_tags=True)
    text, offs, _ = synth.gen_text(100_000, 40, seed=synth.TEXT_SEED + 77)
    raw_block = b"\n".join(text[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)) + b"\n"
    reps = max(1, int(args.mb * 1e6 / len(raw_block)) + 1)
    raw = raw_block * reps
    none_given = ("\n".join(" ".join(line) for line in raw_block.decode().split("\n")[:-1]) + "\n").encode() * reps
    all_given = annotate_all(p.tokenize_lines(raw_block)[0].tobytes()) * reps

    out = np.empty(6 * len(all_given) + 16, np.uint8)
    out.fill(0)
    res = dict(card(), raw_mb=round(len(raw) / 1e6, 1), lines=raw.count(b"\n"))
    for tags in (False, True):
        calls = {
            "tokenize_lines": (lambda: p.tokenize_lines(raw, out=out, predict_tags=tags), len(raw)),
            "partial_0pct": (lambda: p.tokenize_partial_lines(none_given, out=out, predict_tags=tags), len(none_given)),
            "partial_100pct": (lambda: p.tokenize_partial_lines(all_given, out=out, predict_tags=tags), len(all_given)),
        }
        # warm-up, and the checks that both partial inputs reproduce what they should
        plain = p.tokenize_lines(raw, predict_tags=tags)[0].tobytes()
        assert p.tokenize_partial_lines(none_given, predict_tags=tags)[0].tobytes() == plain
        assert p.tokenize_partial_lines(all_given, predict_tags=tags)[0].tobytes() == plain
        times = {k: [] for k in calls}
        for _ in range(args.reps):
            for k, (fn, _) in calls.items():
                t0 = time.perf_counter()
                fn()
                times[k].append(time.perf_counter() - t0)
        sfx = "_tags" if tags else ""
        for k, (_, nbytes) in calls.items():
            s = statistics.median(times[k])
            res[k + sfx + "_s"] = round(s, 4)
            res[k + sfx + "_input_gb_s"] = round(nbytes / 1e9 / s, 3)

    # the host path the device call replaces, per sentence
    lines = raw_block.decode().split("\n")[: args.host_lines]
    given = annotate_all(p.tokenize_lines(("\n".join(lines) + "\n").encode())[0].tobytes()).decode().split("\n")
    t0 = time.perf_counter()
    for line, ann in zip(lines, given):
        s = vb.Sentence.from_raw(line)
        p.predict(s)
        b = s.boundaries_mut()
        for i, m in enumerate(ann[1::2]):
            if m in "|-":
                b[i] = 1 if m == "|" else 0
        s.fill_tags()
        s.write_tokenized_text()
    dt = time.perf_counter() - t0
    n_host = sum(len(x.encode()) + 1 for x in lines)
    res.update(host_lines=len(lines), host_s=round(dt, 4), host_input_mb_s=round(n_host / 1e6 / dt, 3))
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
