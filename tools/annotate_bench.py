#!/usr/bin/env python
"""Cost of vpt_annotate_lines next to vpt_tokenize_lines on the same raw text, in one process.

A synthetic model with tag models and text of the benchmark's config-2 shape (tests/vpt_testlib/synth.py, seeded: lines
of 40 characters) give the raw lines (at least --mb MB).  After a warm-up, the calls alternate for --reps rounds:
tokenize_lines, annotate_lines at margin 0 and at a mid margin (the median |score| of a sample: about half of the
boundaries Unknown), each with tags off and on, through the C ABI into one preallocated pinned buffer, so the times
are the device pipelines' (Predictor.annotate_lines also copies its output into a bytes object; its time is reported
apart).  The script prints the median, min and max seconds of each, the rates in GB/s of the raw input, the card's
name, power limit and max SM clock, and checks on the timed output that
tokenize_partial_lines(annotate_lines(x, m)) == tokenize_lines(x) (without tags: the synthetic tag strings hold marker
characters, which the partial-annotation format writes unescaped).

    python tools/annotate_bench.py [--mb 100] [--reps 7]
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
    raw = raw_block * max(1, int(args.mb * 1e6 / len(raw_block)) + 1)
    sample = p.predict_batch(text[: int(offs[2000])], offs[:2001] - offs[0])
    mid = int(np.median(np.abs(sample.scores[: int(sample.bound_offsets[-1])])))

    out = torch.empty(20 * len(raw) + 16, dtype=torch.uint8).pin_memory()
    L, n, nl = vb.lib(), C.c_uint64(), C.c_uint64()

    def check(rc):
        vb._check(rc)
        return n.value

    res = dict(card(), raw_mb=round(len(raw) / 1e6, 1), lines=raw.count(b"\n"), mid_margin=mid)
    calls = {}
    for tags in (False, True):
        sfx = "_tags" if tags else ""
        fn = L.vpt_tokenize_lines_tags if tags else L.vpt_tokenize_lines
        calls["tokenize_lines" + sfx] = lambda fn=fn: check(fn(p._h, raw, len(raw), 0, 0, out.data_ptr(), out.numel(),
                                                              C.byref(n), C.byref(nl)))
        for name, m in (("annotate_m0", 0), ("annotate_mid", mid)):
            calls[name + sfx] = lambda tags=tags, m=m: check(L.vpt_annotate_lines(
                p._h, None, raw, len(raw), 0, 0, int(tags), m, out.data_ptr(), out.numel(), C.byref(n), C.byref(nl)))
    calls["annotate_mid_python_bytes"] = lambda: p.annotate_lines(raw, mid)
    for fn in calls.values():  # warm-up
        fn()
    times = {k: [] for k in calls}
    for _ in range(args.reps):
        for k, fn in calls.items():
            t0 = time.perf_counter()
            fn()
            times[k].append(time.perf_counter() - t0)
    sizes = {k: fn() for k, fn in calls.items() if k != "annotate_mid_python_bytes"}
    for k, ts in times.items():
        if k in sizes:
            res[k + "_out_mb"] = round(sizes[k] / 1e6, 1)
        res[k + "_s"] = {"median": round(statistics.median(ts), 4), "min": round(min(ts), 4), "max": round(max(ts), 4)}
        res[k + "_input_gb_s"] = round(len(raw) / 1e9 / statistics.median(ts), 3)
    for base in ("tokenize_lines", "tokenize_lines_tags"):
        t = statistics.median(times[base])
        for name in ("annotate_m0", "annotate_mid"):
            k = name + base[len("tokenize_lines"):]
            res[k + "_vs_tokenize"] = round(statistics.median(times[k]) / t, 3)

    # the round trip on the output the timed calls write
    plain = p.tokenize_lines(raw)[0].tobytes()
    for m in (0, mid):
        size = check(L.vpt_annotate_lines(p._h, None, raw, len(raw), 0, 0, 0, m, out.data_ptr(), out.numel(), C.byref(n),
                                          C.byref(nl)))
        assert nl.value == res["lines"]
        ann = out[:size].numpy().tobytes()
        assert p.tokenize_partial_lines(ann)[0].tobytes() == plain, m
        res[f"round_trip_m{m}"] = "ok"
        res[f"space_markers_m{m}"] = ann.count(b" ")  # ' ' markers, and the text's own spaces
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
