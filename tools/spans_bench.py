#!/usr/bin/env python
"""Throughput of token spans (Predictor.token_spans, vpt_token_spans) next to the two ways an indexer could get the same
byte offsets from the calls that existed before it, in one process.

Workloads (config-2-shaped text, tests/vpt_testlib/synth.py, seeded; a 300 000-pattern bccwj-shaped model):
  docs40     --docs documents of 40 characters (1 M, about 116 MB): many short documents
  docs32k    about 4 000 documents of about 32 KB, each the same 40-character sentences joined by '\\n': few long
             documents with a line break every ~40 characters
For each workload three calls, alternating, each ending in a device synchronisation:
  spans      vpt_token_spans (Python API): the token ends come back
  compact    vpt_predict_batch_compact + numpy: the boundary bits become token byte ends on the host (no line-break split
             or pre-filter: bare predict, so only the time is comparable)
  lines      vpt_tokenize_lines on the same bytes (docs40: the documents joined by '\\n'): tokenized text comes back
After a warm-up call each, --reps rounds; the script prints the median seconds and GB/s of input (document bytes) of
each, with the card's name and power limit, as one JSON line.  The spans result is checked against the oracle's
composition on a sample of documents before timing.

    python tools/spans_bench.py [--docs 1000000] [--reps 5]
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


def compact_to_ends(np, p, t, off):
    """vpt_predict_batch_compact, then token byte ends from the boundary bits: a set boundary after character i of a
    document ends a token at the byte position of character i + 1; every document's end closes its last token."""
    c = p.predict_batch_compact(t, off)
    b = c.boundaries()
    char_pos = np.flatnonzero((t & 0xC0) != 0x80)          # byte position of every character (valid, non-empty docs)
    k = np.flatnonzero(b)                                  # set boundaries, batch-global
    doc = np.searchsorted(c.bit_offsets, k, side="right") - 1
    pos = np.concatenate((char_pos[k + doc + 1], off[1:].astype(np.int64)))
    pos.sort()
    return pos - off[np.searchsorted(off, pos, side="left") - 1].astype(np.int64)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args(argv)

    import numpy as np
    import torch
    import vaporetto_b200 as vb
    from vpt_testlib import oracle, synth
    from vpt_testlib import spans_oracle as so
    mb = synth.gen_model_bccwj_shaped(n_patterns=300_000, sample_sentences=200_000)
    p = vb.Predictor(vb.Model.read(mb))
    text, offs, _ = synth.gen_text(args.docs, 40, seed=synth.TEXT_SEED + 11)
    t = np.asarray(text, np.uint8)
    offs = np.asarray(offs, np.uint64)

    # docs40: the sentences as documents; docs32k: groups of sentences joined by '\n' (~32 KB each)
    sents = [t[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(offs.size - 1)]
    per = max(1, round(32_000 / (len(t) / max(len(sents), 1) + 1)))
    big = [b"\n".join(sents[i:i + per]) for i in range(0, len(sents), per)]
    big_t = np.frombuffer(b"".join(big), np.uint8)
    big_off = np.zeros(len(big) + 1, np.uint64)
    np.cumsum([len(x) for x in big], out=big_off[1:])
    workloads = {
        "docs40": (t, offs, b"\n".join(sents) + b"\n"),
        "docs32k": (big_t, big_off, big_t.tobytes()),
    }
    del sents, big

    ora = oracle.OraclePredictor(mb)
    res = dict(card(), docs=args.docs, reps=args.reps)
    for wname, (wt, woff, lines) in workloads.items():
        n = woff.size - 1
        r = p.token_spans(wt, woff)
        for d in range(0, n, max(1, n // 50)):  # the spans result against the oracle's composition
            doc = wt[int(woff[d]):int(woff[d + 1])].tobytes().decode()
            assert r.spans(d)[:, 1].tolist() == so.compose(ora, doc), (wname, d)
        ends = compact_to_ends(np, p, wt, woff)
        assert ends.size >= n and ends.max() <= int(np.diff(woff.astype(np.int64)).max())
        out = np.zeros(3 * len(lines) + lines.count(b"\n") + 16, np.uint8)  # allocated and touched once
        calls = {
            "spans": lambda: p.token_spans(wt, woff),
            "compact": lambda: compact_to_ends(np, p, wt, woff),
            "lines": lambda: p.tokenize_lines(lines, out=out),
        }
        for fn in calls.values():
            fn()
        times = {name: [] for name in calls}
        for _ in range(args.reps):
            for name, fn in calls.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t0)
        size = int(woff[-1] - woff[0])
        res[wname] = {"documents": n, "input_mb": round(size / 1e6, 1), "tokens": int(r.token_ends.size)}
        for name, ts in times.items():
            s = statistics.median(ts)
            res[wname][name] = {"s": round(s, 4), "gb_s": round(size / 1e9 / s, 2)}
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
