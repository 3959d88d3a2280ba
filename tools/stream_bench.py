#!/usr/bin/env python
"""Throughput of the line stream (Predictor.line_stream, vpt_line_stream_*) next to the whole-buffer calls it restates
(vpt_tokenize_lines, vpt_evaluate_lines), in one process.

The input is config-2-shaped text (tests/vpt_testlib/synth.py, seeded): --lines lines of 40 characters (1 M lines, about
116 MB), on a 300 000-pattern bccwj-shaped model; for evaluate, the same lines tokenized by the library (the gold text).
Each round times, in this order: the whole-buffer call from a pageable `bytes` object, the whole-buffer call from a
pinned buffer (output pinned as well), and the stream fed in 64 KiB, 1 MiB and 16 MiB pieces through the Python API
(every call's output as `bytes`, as tools/predict_cli.py receives and writes it; a new stream each time).  Every call ends in a device
synchronisation.  After a warm-up round, --reps rounds; the script prints the median seconds and MB/s of input for each,
with the card's name and power limit, as one JSON line.  Every stream output is checked against the whole-buffer one.

    python tools/stream_bench.py [--lines 1000000] [--reps 5] [--predict-tags]
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

PIECES = {"64KiB": 64 << 10, "1MiB": 1 << 20, "16MiB": 16 << 20}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name, "power_limit": power}


def run_stream(p, data: bytes, piece: int, kind: str, flags: dict):
    parts = []
    mv = memoryview(data)
    with p.line_stream(kind, **flags) as s:
        for i in range(0, len(data), piece):
            parts.append(s.feed(mv[i:i + piece]))
        r = s.finish()
    return r if kind == "evaluate" else parts + [r[0]]  # (output pieces, as a CLI writes them)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--predict-tags", action="store_true", help="with tag prediction (a model with 2 000 tag models)")
    args = ap.parse_args(argv)

    import numpy as np
    import torch
    import vaporetto_b200 as vb
    from vpt_testlib import synth
    mb = synth.gen_model_bccwj_shaped(n_patterns=300_000, sample_sentences=200_000,
                                      tag_models=2_000 if args.predict_tags else 0)
    p = vb.Predictor(vb.Model.read(mb), predict_tags=args.predict_tags)
    text, offs, _ = synth.gen_text(args.lines, 40, seed=synth.TEXT_SEED + 7)
    raw = b"\n".join(text[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)) + b"\n"
    del text, offs
    flags = dict(predict_tags=args.predict_tags)
    gold = p.tokenize_lines(raw, **flags)[0].tobytes()

    def pinned(n):
        return torch.empty(n, dtype=torch.uint8).pin_memory().numpy()

    out_cap = (19 if args.predict_tags else 3) * len(raw) + raw.count(b"\n") + 16
    out_pageable = np.zeros(out_cap, np.uint8)  # allocated and touched once: the timing is the call, not page faults
    out_pinned = pinned(out_cap)
    raw_pinned = pinned(len(raw))
    raw_pinned[:] = np.frombuffer(raw, np.uint8)
    gold_pinned = pinned(len(gold))
    gold_pinned[:] = np.frombuffer(gold, np.uint8)
    want_tok = gold
    want_ev = p.evaluate_lines(gold, **flags)

    calls = {
        "tokenize.whole_pageable": lambda: p.tokenize_lines(raw, out=out_pageable, **flags),
        "tokenize.whole_pinned": lambda: p.tokenize_lines(raw_pinned, out=out_pinned, **flags),
        "evaluate.whole_pageable": lambda: p.evaluate_lines(gold, **flags),
        "evaluate.whole_pinned": lambda: p.evaluate_lines(gold_pinned, **flags),
    }
    for name, piece in PIECES.items():
        calls["tokenize.stream_" + name] = lambda piece=piece: run_stream(p, raw, piece, "tokenize", flags)
        calls["evaluate.stream_" + name] = lambda piece=piece: run_stream(p, gold, piece, "evaluate", flags)
    # warm-up and the equivalence check
    for name, fn in calls.items():
        r = fn()
        if name.startswith("tokenize.stream"):
            assert b"".join(r) == want_tok, name
        elif name.startswith("evaluate"):
            assert r == want_ev, name
    times = {name: [] for name in calls}
    for _ in range(args.reps):
        for name, fn in calls.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
    res = dict(card(), lines=args.lines, raw_mb=round(len(raw) / 1e6, 1), gold_mb=round(len(gold) / 1e6, 1),
               predict_tags=args.predict_tags, reps=args.reps)
    for name, ts in times.items():
        s = statistics.median(ts)
        size = len(raw) if name.startswith("tokenize") else len(gold)
        res[name] = {"s": round(s, 4), "mb_s": round(size / 1e6 / s, 1)}
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
