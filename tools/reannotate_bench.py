#!/usr/bin/env python
"""Cost of vpt_reannotate_lines next to vpt_annotate_lines on the raw text and vpt_tokenize_partial_lines on the same
partially annotated input, in one process.

A synthetic model with tag models and text of the benchmark's config-2 shape (tests/vpt_testlib/synth.py, seeded: lines
of 40 characters) give the raw lines (at least --mb MB), as in tools/partial_bench.py.  The partially annotated inputs
are those lines with 0 % of the markers given (every marker ' ') and with 30 % given (each marker of the model's own
segmentation kept with probability 0.3, else ' '; one character in ten carries an input tag "/名詞").  Tags are
predicted in every call; the margin is the median |score| of a sample (about half of the undecided boundaries stay
open).  After a warm-up, the calls alternate for --reps rounds through the C ABI into one preallocated pinned buffer; the
script prints the median, min and max seconds of each, the rates in GB/s of the call's input, the ratios to the two
neighbouring calls, and the card's name, power limit and max SM clock read in the same run.  It checks on the timed
output that the 0 % input gives annotate_lines' output.

    python tools/reannotate_bench.py [--mb 100] [--reps 7]
"""
import argparse
import json
import os
import random
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


def partial_input(tokenized: bytes, share: float, tag_share: float, rng) -> bytes:
    """The lines of tokenize_lines' output (without tags) with a share of the markers given, the rest ' ', and an input
    tag on a share of the characters."""
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
        chars = [c for t in toks for c in t]
        marks = [m for t in toks for m in "-" * (len(t) - 1) + "|"][:-1]
        parts = []
        for i, c in enumerate(chars):
            parts.append(c + ("/名詞" if rng.random() < tag_share else ""))
            if i < len(marks):
                parts.append(marks[i] if rng.random() < share else " ")
        out.append("".join(parts))
    return ("\n".join(out) + "\n").encode()


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=100.0, help="size of the raw text in MB (at least)")
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args(argv)

    import ctypes as C
    import numpy as np
    import torch
    import vaporetto_b200 as vb
    from vpt_testlib import synth
    mb = synth.gen_model_bccwj_shaped(n_patterns=100_000, sample_sentences=200_000, tag_models=2_000)
    p = vb.Predictor(vb.Model.read(mb), predict_tags=True)
    text, offs, _ = synth.gen_text(100_000, 40, seed=synth.TEXT_SEED + 77)
    raw_block = b"\n".join(text[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)) + b"\n"
    reps = max(1, int(args.mb * 1e6 / len(raw_block)) + 1)
    raw = raw_block * reps
    tok_block = p.tokenize_lines(raw_block)[0].tobytes()
    rng = random.Random(20)
    inputs = {"0pct": partial_input(tok_block, 0.0, 0.0, rng) * reps,
              "30pct": partial_input(tok_block, 0.3, 0.1, rng) * reps}
    sample = p.predict_batch(text[: int(offs[2000])], offs[:2001] - offs[0])
    mid = int(np.median(np.abs(sample.scores[: int(sample.bound_offsets[-1])])))

    out = torch.empty(20 * max(len(x) for x in inputs.values()) + 16, dtype=torch.uint8).pin_memory()
    L, n, nl = vb.lib(), C.c_uint64(), C.c_uint64()

    def check(rc):
        vb._check(rc)
        return n.value

    res = dict(card(), raw_mb=round(len(raw) / 1e6, 1), lines=raw.count(b"\n"), margin=mid,
               input_mb={k: round(len(v) / 1e6, 1) for k, v in inputs.items()})
    calls = {"annotate_raw": (lambda: check(L.vpt_annotate_lines(p._h, None, raw, len(raw), 0, 0, 1, mid, out.data_ptr(),
                                                                  out.numel(), C.byref(n), C.byref(nl))), len(raw))}
    for k, x in inputs.items():
        calls["partial_" + k] = (lambda x=x: check(L.vpt_tokenize_partial_lines(
            p._h, None, x, len(x), 0, 0, 1, out.data_ptr(), out.numel(), C.byref(n), C.byref(nl))), len(x))
        calls["reannotate_" + k] = (lambda x=x: check(L.vpt_reannotate_lines(
            p._h, None, x, len(x), 0, 0, 1, mid, 1, out.data_ptr(), out.numel(), C.byref(n), C.byref(nl))), len(x))
    for fn, _ in calls.values():  # warm-up
        fn()
    times = {k: [] for k in calls}
    for _ in range(args.reps):
        for k, (fn, _) in calls.items():
            t0 = time.perf_counter()
            fn()
            times[k].append(time.perf_counter() - t0)
    for k, ts in times.items():
        res[k + "_s"] = {"median": round(statistics.median(ts), 4), "min": round(min(ts), 4), "max": round(max(ts), 4)}
        res[k + "_input_gb_s"] = round(calls[k][1] / 1e9 / statistics.median(ts), 3)
    for k in inputs:
        t = statistics.median(times["reannotate_" + k])
        res[f"reannotate_{k}_vs_annotate_raw"] = round(t / statistics.median(times["annotate_raw"]), 3)
        res[f"reannotate_{k}_vs_partial_{k}"] = round(t / statistics.median(times["partial_" + k]), 3)

    # the output the timed calls write: the 0 % input is annotate_lines of the raw text
    size = check(L.vpt_annotate_lines(p._h, None, raw, len(raw), 0, 0, 1, mid, out.data_ptr(), out.numel(), C.byref(n),
                                      C.byref(nl)))
    ann = out[:size].numpy().tobytes()
    x = inputs["0pct"]
    size = check(L.vpt_reannotate_lines(p._h, None, x, len(x), 0, 0, 1, mid, 1, out.data_ptr(), out.numel(), C.byref(n),
                                        C.byref(nl)))
    assert out[:size].numpy().tobytes() == ann
    x = inputs["30pct"]
    size = check(L.vpt_reannotate_lines(p._h, None, x, len(x), 0, 0, 1, mid, 1, out.data_ptr(), out.numel(), C.byref(n),
                                        C.byref(nl)))
    res["checks"] = "ok"
    res["open_markers_30pct"] = out[:size].numpy().tobytes().count(b" ")
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
