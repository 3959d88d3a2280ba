#!/usr/bin/env python
"""Tokenized text of documents already in GPU memory (Predictor.tokenize_device, vpt_tokenize_dev) next to the host
line call (Predictor.tokenize_lines, vpt_tokenize_lines) on the same documents, in one process.

Workloads (DESIGN §14; config-2-shaped text, tests/vpt_testlib/synth.py, seeded; a 300 000-pattern bccwj-shaped model):
  docs40     --docs documents of 40 characters (1 M, about 116 MB): many short documents
  docs32k    about 3 600 documents of about 32 KB, the same sentences joined by '。' (no '\\n'): few long documents
For each workload two calls, alternating:
  device     tokenize_device on a CUDA tensor holding the text and int64 offsets; the string column stays on the device
  lines      tokenize_lines on the same documents joined by '\\n' in pinned host memory, into a pinned output buffer
Before timing, the device strings joined by '\\n' are checked against the line output.  Each call is timed with CUDA
events on the current stream around it, ending in a synchronisation, after one warm-up call each; --reps rounds,
medians and min-max.  GB/s is of document bytes.  Prints one JSON line with the card's name, power limit and max SM
clock.

    python tools/tokenize_device_bench.py [--docs 1000000] [--reps 7]
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
    big = ["。".encode().join(sents[i:i + per]) for i in range(0, len(sents), per)]
    workloads = {"docs40": sents, "docs32k": big}

    res = dict(card(), docs=args.docs, reps=args.reps)
    for wname, docs in workloads.items():
        n = len(docs)
        assert not any(b"\n" in d or d.endswith(b"\r") for d in docs)
        off = np.zeros(n + 1, np.int64)
        np.cumsum([len(x) for x in docs], out=off[1:])
        d_text = torch.from_numpy(np.frombuffer(b"".join(docs), np.uint8).copy()).cuda()
        d_off = torch.from_numpy(off).cuda()
        h_lines = torch.from_numpy(np.frombuffer(b"".join(d + b"\n" for d in docs), np.uint8).copy()).pin_memory()
        hl = h_lines.numpy()
        h_out = torch.empty(3 * hl.size + 16, dtype=torch.uint8).pin_memory().numpy()
        want, nl = p.tokenize_lines(hl, out=h_out)
        assert nl == n
        got = p.tokenize_device(d_text, d_off)
        chars, goff, status = got.to_host()
        assert (status == 0).all(), wname
        b = chars.tobytes()
        assert b"".join(b[goff[i]:goff[i + 1]] + b"\n" for i in range(n)) == want.tobytes(), wname
        out_bytes = int(goff[-1])
        del got, chars, b
        calls = {"device": lambda: p.tokenize_device(d_text, d_off), "lines": lambda: p.tokenize_lines(hl, out=h_out)}
        for fn in calls.values():
            fn()
        torch.cuda.synchronize()
        times = {name: [] for name in calls}
        for _ in range(args.reps):
            for name, fn in calls.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                r = fn()
                e1.record()
                e1.synchronize()
                times[name].append(e0.elapsed_time(e1) / 1e3)
                del r
        size = int(off[-1])
        res[wname] = {"documents": n, "input_mb": round(size / 1e6, 1), "output_mb": round(out_bytes / 1e6, 1)}
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
