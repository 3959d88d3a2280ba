"""Node-table slots that k_fused probes on bench.py's config-2 text, in the kernel's order, for the `record_load`
`probe_seq` test of l2_probe_bench.cu.

The probe rule is vpt_testlib/probe_model.py's: the 2-character node of every character (the 1-character node at a
sentence start), then the 3-character node when the 2-character record's child mask has the bit of the character
before, or the 1-character node when the 2-character node does not exist.  Every distinct key gets one slot of a table
of the config-2 size; existing nodes get distinct slots, missing keys a uniformly random one (the perfect hash sends
them onto some record).  What the test needs is the distribution of the probes over the slots: how often the records
of frequent characters and pairs come back.

    python profiles/tools/probe_slots.py build/probe_slots.u32 [--sentences 50000] [--table-mb 17.1]
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--sentences", type=int, default=50_000)
    ap.add_argument("--table-mb", type=float, default=17.1)
    args = ap.parse_args()

    import bench
    from vpt_testlib import probe_model, synth

    model = bench.get_model(300_000, 2_000_000, 2)
    text, offs, _ = synth.gen_text(args.sentences, 40, seed=synth.TEXT_SEED)
    sents = [bytes(text[int(offs[i]):int(offs[i + 1])]).decode() for i in range(args.sentences)]

    nodes = set()
    for p in probe_model.char_patterns(model):
        for i in range(len(p)):
            s = p[i:][-3:] if len(p) - i > 3 else p[i:]
            for k in (1, 2, 3):
                if len(s) >= k:
                    nodes.add(s[-k:])
    masks = {}
    for t in nodes:
        if len(t) == 3:
            masks[t[1:]] = masks.get(t[1:], 0) | (1 << probe_model.child_bit(ord(t[0])))

    nslots = int(args.table_mb * 1048576 / 32)
    rng = np.random.default_rng(0x5107)
    perm = rng.permutation(nslots)
    slot_of = {t: int(perm[i]) for i, t in enumerate(sorted(nodes))}

    def slot(key):
        s = slot_of.get(key)
        if s is None:
            s = slot_of[key] = int(rng.integers(nslots))
        return s

    seq = []
    for s in sents:
        for p in range(len(s)):
            if p == 0:
                seq.append(slot(s[0]))
                continue
            t2 = s[p - 1:p + 1]
            seq.append(slot(t2))
            if t2 in nodes:
                if p >= 2 and (masks.get(t2, 0) >> probe_model.child_bit(ord(s[p - 2]))) & 1:
                    seq.append(slot(s[p - 2:p + 1]))
            else:
                seq.append(slot(s[p]))
    arr = np.asarray(seq, np.uint32)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    arr.tofile(args.out)
    chars = sum(len(s) for s in sents)
    _, counts = np.unique(arr, return_counts=True)
    top = np.sort(counts)[::-1]
    print(f"{len(arr)} probes over {chars} characters ({len(arr) / chars:.3f} per character), {len(counts)} distinct "
          f"slots of {nslots}; hottest 1000 / 10000 slots take {top[:1000].sum() / len(arr):.3f} / "
          f"{top[:10000].sum() / len(arr):.3f} of the probes")


if __name__ == "__main__":
    main()
