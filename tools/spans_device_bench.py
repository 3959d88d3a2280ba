#!/usr/bin/env python
"""Token spans of documents already in GPU memory (Predictor.token_spans_device, vpt_token_spans_dev) next to the host
call (Predictor.token_spans, vpt_token_spans) on the same documents, in one process.

Workloads (DESIGN §14; config-2-shaped text, tests/vpt_testlib/synth.py, seeded; a 300 000-pattern bccwj-shaped model):
  docs40     --docs documents of 40 characters (1 M, about 116 MB): many short documents
  docs32k    about 3 600 documents of about 32 KB, the same sentences joined by '\\n': few long documents
For each workload two calls, alternating:
  device     token_spans_device on a CUDA tensor holding the text and int64 offsets; outputs stay on the device
  host       token_spans on the same text and offsets in pinned host memory; outputs come back to host memory
Each call is timed with CUDA events on the current stream around it, ending in a synchronisation, after one warm-up
call each; --reps rounds, medians.  The device result is checked against the host call before timing.  GB/s is of
document bytes.  Prints one JSON line with the card's name, power limit and max SM clock.

    python tools/spans_device_bench.py [--docs 1000000] [--reps 7]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

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
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args(argv)

    import numpy as np
    import torch
    import vaporetto_b200 as vb
    from vpt_testlib import synth
    mb = synth.gen_model_bccwj_shaped(n_patterns=300_000, sample_sentences=200_000)
    p = vb.Predictor(vb.Model.read(mb))
    text, offs, _ = synth.gen_text(args.docs, 40, seed=synth.TEXT_SEED + 11)
    t = np.asarray(text, np.uint8)
    offs = np.asarray(offs, np.uint64)
    sents = [t[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(offs.size - 1)]
    per = max(1, round(32_000 / (len(t) / max(len(sents), 1) + 1)))
    big = [b"\n".join(sents[i:i + per]) for i in range(0, len(sents), per)]
    big_t = np.frombuffer(b"".join(big), np.uint8)
    big_off = np.zeros(len(big) + 1, np.uint64)
    np.cumsum([len(x) for x in big], out=big_off[1:])
    workloads = {"docs40": (t, offs), "docs32k": (big_t, big_off)}
    del sents, big

    res = dict(card(), docs=args.docs, reps=args.reps)
    for wname, (wt, woff) in workloads.items():
        n = woff.size - 1
        h_text = torch.from_numpy(np.array(wt)).pin_memory()
        h_off = torch.from_numpy(woff.astype(np.int64)).pin_memory()
        ht, hoff = h_text.numpy(), h_off.numpy().view(np.uint64)
        d_text, d_off = h_text.cuda(), h_off.cuda()
        want = p.token_spans(ht, hoff)
        got = p.token_spans_device(d_text, d_off).to_host()
        assert np.array_equal(got.status, want.status) and np.array_equal(got.token_ends, want.token_ends), wname
        calls = {"device": lambda: p.token_spans_device(d_text, d_off), "host": lambda: p.token_spans(ht, hoff)}
        for fn in calls.values():
            fn()
        torch.cuda.synchronize()
        times = {name: [] for name in calls}
        for _ in range(args.reps):
            for name, fn in calls.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                e1.synchronize()
                times[name].append(e0.elapsed_time(e1) / 1e3)
        size = int(woff[-1] - woff[0])
        res[wname] = {"documents": n, "input_mb": round(size / 1e6, 1), "tokens": int(want.token_ends.size)}
        for name, ts in times.items():
            s = statistics.median(ts)
            res[wname][name] = {"ms": round(s * 1e3, 2), "gb_s": round(size / 1e9 / s, 2),
                                "spread_ms": [round(min(ts) * 1e3, 2), round(max(ts) * 1e3, 2)]}
        del d_text, d_off
        torch.cuda.empty_cache()
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
