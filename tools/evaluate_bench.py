#!/usr/bin/env python
"""Throughput of vpt_evaluate_lines next to vpt_tokenize_lines on the same corpus, in one process.

A synthetic model and text (tests/vpt_testlib/synth.py, seeded) are tokenized on the device once; that output is the gold
corpus (at least --mb MB, built by repeating it), and the gold's raw lines are the input of tokenize_lines.  After a
warm-up of both, the two calls alternate for --reps rounds; the script prints the median seconds of each and both
rates in MB of gold text per second, with the card's name and power limit.

    python tools/evaluate_bench.py [--mb 200] [--reps 5] [--predict-tags]
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name, "power_limit": power}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=200.0, help="size of the gold corpus in MB (at least)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--predict-tags", action="store_true", help="both calls with tag prediction (a model with tags)")
    args = ap.parse_args(argv)

    import vaporetto_b200 as vb
    from vpt_testlib import synth
    mb = synth.gen_model_bccwj_shaped(n_patterns=100_000, sample_sentences=200_000,
                                      tag_models=2_000 if args.predict_tags else 0)
    p = vb.Predictor(vb.Model.read(mb), predict_tags=args.predict_tags)
    text, offs, _ = synth.gen_text(100_000, 40, seed=synth.TEXT_SEED + 77)
    raw_block = b"\n".join(text[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)) + b"\n"
    gold_block, _ = p.tokenize_lines(raw_block, predict_tags=args.predict_tags)
    gold_block = gold_block.tobytes()
    reps = max(1, int(args.mb * 1e6 / len(gold_block)) + 1)
    gold, raw = gold_block * reps, raw_block * reps
    flags = dict(predict_tags=args.predict_tags)

    # warm-up, and the check that the gold boundaries are the system's own (with tags, a line whose tokens print fewer
    # than n_tags slots has a narrower gold width, so its tokens count as wrong: main.rs compares the tag vectors)
    ev = p.evaluate_lines(gold, **flags)
    assert ev["fp"] == ev["fn"] == 0 and ev["n_sys"] == ev["n_ref"], ev
    import numpy as np
    out = np.empty(4 * len(raw) + 16, np.uint8)  # allocated (and touched) once: the timing is the call, not the page faults
    out.fill(0)
    p.tokenize_lines(raw, out=out, **flags)
    t_ev, t_tok = [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        p.evaluate_lines(gold, **flags)
        t_ev.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        p.tokenize_lines(raw, out=out, **flags)
        t_tok.append(time.perf_counter() - t0)
    s_ev, s_tok = statistics.median(t_ev), statistics.median(t_tok)
    res = dict(card(), gold_mb=round(len(gold) / 1e6, 1), raw_mb=round(len(raw) / 1e6, 1), lines=ev["n_lines"],
               predict_tags=args.predict_tags, evaluate_s=round(s_ev, 4), tokenize_s=round(s_tok, 4),
               evaluate_gold_mb_s=round(len(gold) / 1e6 / s_ev, 1), tokenize_gold_mb_s=round(len(gold) / 1e6 / s_tok, 1),
               evaluate_s_all=[round(x, 4) for x in t_ev], tokenize_s_all=[round(x, 4) for x in t_tok])
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
