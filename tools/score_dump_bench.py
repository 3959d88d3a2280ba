#!/usr/bin/env python
"""Cost of the predict CLI's score dumps on the line stream (DESIGN §17): 1 M config-2-shaped lines, tokenized alone,
with --scores, with --tag-scores and with both (tags on a config-2-shaped model with 2 000 tag models), each a new stream fed 16 MiB
pieces.  Prints one JSON line per case: wall time (median of --reps alternating calls), GB/s of input and of output,
and the device time of the dump kernels per call from torch.profiler (a separate run).  Needs a GPU."""
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

import vaporetto_b200 as vb  # noqa: E402
from vpt_testlib import synth  # noqa: E402

CASES = [("tokenize", False, False), ("scores", True, False), ("tag_scores", False, True), ("both", True, True)]


def run(p, data, scores, tag_scores, piece=16 << 20):
    n_out = 0
    with p.line_stream(predict_tags=True, scores=scores, tag_scores=tag_scores) as st:
        for lo in range(0, len(data), piece):
            n_out += len(st.feed(data[lo:lo + piece]))
        n_out += len(st.finish()[0])
    return n_out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="device times of the dump kernels (torch.profiler)")
    args = ap.parse_args()
    mb = synth.gen_model_bccwj_shaped(n_patterns=300_000, sample_sentences=50_000, tag_models=2_000)
    p = vb.Predictor(vb.Model.read(mb), predict_tags=True)
    text, offs, _ = synth.gen_text(args.lines, 40, seed=synth.TEXT_SEED + 3)
    data = b"\n".join(text[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)) + b"\n"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    for _, s, t in CASES:
        run(p, data, s, t)  # warm-up
    times = {c[0]: [] for c in CASES}
    outs = {}
    for _ in range(args.reps):
        for name, s, t in CASES:
            t0 = time.perf_counter()
            outs[name] = run(p, data, s, t)
            times[name].append(time.perf_counter() - t0)
    kern = {}
    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        for name, s, t in CASES:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run(p, data, s, t)
                torch.cuda.synchronize()
            kern[name] = {e.key: round(e.device_time_total / 1000.0, 3) for e in prof.key_averages()
                          if "k_dump" in e.key or "k_tok_" in e.key or "k_score_" in e.key}
    for name, _, _ in CASES:
        m = statistics.median(times[name])
        print(json.dumps(dict(case=name, gpu=gpu, lines=args.lines, in_bytes=len(data), out_bytes=outs[name],
                              seconds=round(m, 4), in_gbps=round(len(data) / m / 1e9, 3),
                              out_gbps=round(outs[name] / m / 1e9, 3), kernel_ms=kern.get(name))))
    return 0


if __name__ == "__main__":
    sys.exit(main())
