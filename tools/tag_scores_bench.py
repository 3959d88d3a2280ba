#!/usr/bin/env python
"""Cost of the tag candidate scores (vpt_predict_batch_compact_tag_scores, vpt_token_spans_tag_scores).

Workload: config-3-shaped (bench.py's config 3): a 300 000-pattern bccwj-shaped model with 20 000 unidic-shaped tag
models and --sentences sentences of 40 characters of the seeded synthetic text.  Four calls: predict_batch_compact with
tags, with tags and scores, and token_spans the same way.

After a warm-up of each, --reps rounds that alternate the four calls; every call ends in a device synchronisation and is
reported as the median seconds.  Then one call of each under torch.profiler with CUDA activities: the summed device time
of the tag kernels (k_tok_lookup*, k_score_block, k_score_scan, k_tok_score*) per call, and the bytes of scores copied out.
The scores path is checked to leave every other output unchanged.  Prints one JSON line with the card's name and power
limit.

    python tools/tag_scores_bench.py [--sentences 1000000] [--reps 5]
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

KERNELS = ("k_tok_lookup", "k_score_block", "k_score_scan", "k_tok_score")


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().split(", ") + ["", "", ""])[:3]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sentences", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch
    import vaporetto_b200 as vb
    from vpt_testlib import synth

    t0 = time.time()
    mb = synth.gen_model_bccwj_shaped(n_patterns=300_000, sample_sentences=2_000_000, tag_models=20_000)
    text, offs, _ = synth.gen_text(args.sentences, 40, seed=synth.TEXT_SEED + 3)
    print(f"[tag_scores_bench] model and {int(offs[-1])} bytes of text in {time.time() - t0:.0f} s", file=sys.stderr)
    p = vb.Predictor(vb.Model.read(mb), predict_tags=True)

    calls = {
        "compact tags": lambda: p.predict_batch_compact(text, offs, tags=True),
        "compact tags+scores": lambda: p.predict_batch_compact(text, offs, tags=True, tag_scores=True),
        "spans tags": lambda: p.token_spans(text, offs, tags=True),
        "spans tags+scores": lambda: p.token_spans(text, offs, tags=True, tag_scores=True),
    }
    out = {k: f() for k, f in calls.items()}  # warm-up, and the outputs to compare
    for a, b, fields in (("compact tags", "compact tags+scores", ("boundary_bits", "n_tokens", "token_ids", "token_cands")),
                         ("spans tags", "spans tags+scores", ("token_ends", "n_tokens", "token_ids", "token_cands"))):
        for f in fields:
            assert np.array_equal(getattr(out[a], f), getattr(out[b], f)), (a, f)
    secs = {k: [] for k in calls}
    for _ in range(args.reps):
        for k, f in calls.items():
            t = time.perf_counter()
            f()
            secs[k].append(time.perf_counter() - t)

    from torch.profiler import ProfilerActivity, profile
    results = {}
    for k, f in calls.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            r = f()
            torch.cuda.synchronize()
        per = {n: 0.0 for n in KERNELS}
        for ev in prof.events():
            if ev.device_type.name != "CUDA":
                continue
            for n in KERNELS:
                if n in ev.name:
                    per[n] += ev.device_time_total / 1e3
        results[k] = {"seconds_median": round(statistics.median(secs[k]), 4), "seconds_all": [round(s, 4) for s in secs[k]],
                      "kernel_ms": {n: round(v, 3) for n, v in per.items()},
                      "tokens": int(r.token_ids.size), "tokens_with_scores": int((r.token_ids >= 0).sum()),
                      "score_bytes_out": 0 if r.tag_scores is None else int(r.tag_scores.nbytes)}
    print(json.dumps({"bench": "tag_scores", "input_bytes": int(offs[-1]), "sentences": args.sentences, **card(),
                      "results": results}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
