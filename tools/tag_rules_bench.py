#!/usr/bin/env python
"""Cost of PatternMatchTagger rules in the tagged line path (vpt_tokenize_lines_tags_rules).

Workload: config-3-shaped (bench.py's config 3): a 300 000-pattern bccwj-shaped model with 20 000 unidic-shaped tag
models, --lines lines of 40 characters of the seeded synthetic text, tokenised with --predict-tags.  Rule sets: none,
10^4 and 10^6 rules, each with a hit rate of about 0 % (surfaces the text never produces) and about 20 % of the tokens
(the most frequent surfaces of the output until they cover 20 % of it, the rest misses).  Each rule has two tags.

For every case, after a warm-up call: --reps whole-buffer calls from a pageable buffer into a preallocated output, each
ending in a device synchronisation, reported as the median seconds and GB/s of input; then one call under
torch.profiler with CUDA activities, whose per-chunk kernel times (k_tok_lookup, k_rule_lookup, k_tok_write_tags*)
are reported as the mean per chunk.  Rules that match nothing are checked to leave the output unchanged.  Prints one JSON line with the card's name and power limit.

    python tools/tag_rules_bench.py [--lines 500000] [--reps 5]
"""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KERNELS = ("k_tok_lookup", "k_rule_lookup", "k_tok_write_tags")


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().split(", ") + ["", "", ""])[:3]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_rules(out: bytes, n_rules: int, hit: float, fullwidth) -> dict:
    """n_rules rules: the most frequent output surfaces until they cover `hit` of the tokens, then misses."""
    counts = collections.Counter(tok.split(b"/")[0] for line in out.split(b"\n") for tok in line.split(b" ") if tok)
    total = sum(counts.values())
    rules, covered = {}, 0
    for surf, c in counts.most_common():
        if covered >= hit * total or len(rules) >= n_rules:
            break
        rules[fullwidth(surf.decode())] = ["R", "rr"]
        covered += c
    k = 0
    while len(rules) < n_rules:
        rules["miss%07d" % k] = ["R", "rr"]
        k += 1
    return rules, covered / total


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=500_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rule-counts", default="10000,1000000")
    args = ap.parse_args()

    import numpy as np
    import torch
    import vaporetto_b200 as vb
    from vpt_testlib import synth

    t0 = time.time()
    mb = synth.gen_model_bccwj_shaped(n_patterns=300_000, sample_sentences=2_000_000, tag_models=20_000)
    text, offs, _ = synth.gen_text(args.lines, 40, seed=synth.TEXT_SEED + 3)
    data = b"\n".join(bytes(text[int(offs[i]):int(offs[i + 1])]) for i in range(args.lines)) + b"\n"
    print(f"[tag_rules_bench] model and {len(data)} bytes of text in {time.time() - t0:.0f} s", file=sys.stderr)
    p = vb.Predictor(vb.Model.read(mb), predict_tags=True)
    fullwidth = lambda s: "".join(chr(vb.lib().vpt_kytea_fullwidth(ord(c))) for c in s)  # noqa: E731
    out_buf = np.empty(8 * len(data), np.uint8)
    base, _ = p.tokenize_lines(data, out=out_buf, predict_tags=True)
    base = base.tobytes()

    def timed(tagger):
        p.tokenize_lines(data, out=out_buf, predict_tags=True, tag_rules=tagger)  # warm-up
        secs = []
        for _ in range(args.reps):
            t = time.perf_counter()
            p.tokenize_lines(data, out=out_buf, predict_tags=True, tag_rules=tagger)
            secs.append(time.perf_counter() - t)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            got, _ = p.tokenize_lines(data, out=out_buf, predict_tags=True, tag_rules=tagger)
            torch.cuda.synchronize()
        per = {k: [] for k in KERNELS}
        for ev in prof.events():
            for k in KERNELS:
                if k in ev.name and ev.device_type.name == "CUDA":
                    per[k].append(ev.device_time_total / 1e3)
        n_chunks = max(len(per["k_tok_lookup"]), 1)
        ms = {k: round(sum(v) / n_chunks, 4) if v else "not run" for k, v in per.items()}
        med = statistics.median(secs)
        return got.tobytes(), {"seconds": round(med, 4), "GB_per_s": round(len(data) / med / 1e9, 3), "chunks": n_chunks,
                               "ms_per_chunk": ms}

    results = {}
    _, results["no rules"] = timed(None)
    for n in (int(x) for x in args.rule_counts.split(",")):
        for hit in (0.0, 0.2):
            rules, rate = make_rules(base, n, hit, fullwidth)
            tagger = vb.PatternMatchTagger(p, rules)
            got, r = timed(tagger)
            assert rate > 0.0 or got == base, "rules that match nothing must not change the output"
            r["hit_rate"] = round(rate, 4)
            results[f"{n} rules, {int(hit * 100)}% hits"] = r
            tagger.close()
    print(json.dumps({"bench": "tag_rules", "input_bytes": len(data), "lines": args.lines, **card(), "results": results}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
