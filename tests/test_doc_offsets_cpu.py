"""The document offset check of vpt_token_spans_dev without a device: vaporetto_b200/csrc/doc_offsets.hpp, compiled for
the host (tests/native/doc_offsets_test.cpp), against a Python restatement of the rule, over every combination of small
offsets (decreasing ones, negative ones, ones past n_bytes), lengths at the 1 GiB limit, int32 and int64 widths and every
base alignment 0-15.  The device side is tests/test_gpu_spans_device.py."""
import itertools
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "doc_offsets_test.cpp")
GIB = 1 << 30


def as_width(x, width):
    """x stored in a signed integer of `width` bytes and read back."""
    bits = 8 * width
    x &= (1 << bits) - 1
    return x - (1 << bits) if x >> (bits - 1) else x


def restate(offsets, width, n_bytes, shift):
    """Rebased offsets and bad flags: document d is good when 0 <= o[d] <= o[d+1] <= n_bytes, it is at most 1 GiB long
    and it does not start before an earlier offset; the rebased offsets are shift + the running maximum of the offsets
    that lie in [0, n_bytes] (the others count as 0)."""
    o = [as_width(x, width) for x in offsets]
    clamped = [x if 0 <= x <= n_bytes else 0 for x in o]
    out, bad, m = [], [], 0
    for i, c in enumerate(clamped):
        before = m
        m = max(m, c)
        out.append(shift + m)
        if i + 1 < len(o):
            lo, hi = o[i], o[i + 1]
            ok = 0 <= lo <= hi <= n_bytes and hi - lo <= GIB and lo >= before
            bad.append(0 if ok else 1)
    return out, bad


def cases():
    for width in (4, 8):
        for n_bytes in (0, 1, 3, 4):
            vals = [-1, 0, 1, 2, 3, 4, 5]
            for k in (1, 2, 3, 4):
                for offs in itertools.product(vals, repeat=k):
                    yield width, n_bytes, (len(offs) * 7 + sum(offs)) % 16, offs
        # lengths at the limit, and values that do not fit the width
        big = [0, 1, GIB - 1, GIB, GIB + 1, GIB + 2, 2 * GIB, -(1 << 31), (1 << 31) - 1]
        if width == 8:
            big += [-(1 << 63), (1 << 63) - 1, 1 << 32, (1 << 32) + 1]
        for n_bytes in (GIB, GIB + 1, 2 * GIB):
            for offs in itertools.product(big, repeat=3):
                yield width, n_bytes, 0, offs
    for shift in range(16):
        for width in (4, 8):
            for offs in ((0, 3, 3, 7, 9), (2, 5, 4, 9, 12), (1, 1, 20, 6, 8), (0, -3, 4, 4, 9)):
                yield width, 9, shift, offs


def test_doc_offsets_vs_restatement(tmp_path):
    exe = str(tmp_path / "doc_offsets_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-o", exe, SRC])
    cs = list(cases())
    inp = "".join(f"{w} {nb} {sh} {len(o)} " + " ".join(str(x) for x in o) + "\n" for w, nb, sh, o in cs)
    res = subprocess.run([exe], input=inp, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lines = res.stdout.splitlines()
    assert len(lines) == len(cs)
    n_bad = 0
    for (w, nb, sh, offs), line in zip(cs, lines):
        left, right = line.split("|")
        got = ([int(x) for x in left.split()], [int(x) for x in right.split()])
        want = restate(offs, w, nb, sh)
        assert got == want, (w, nb, sh, offs, got, want)
        # what the rule promises: non-decreasing offsets inside the batch, and every good document keeps its range
        out, bad = want
        assert all(sh <= a <= b <= sh + nb for a, b in zip(out, out[1:] + [sh + nb]))
        o = [as_width(x, w) for x in offs]
        for d, b in enumerate(bad):
            if not b:
                assert (out[d] - sh, out[d + 1] - sh) == (o[d], o[d + 1])
            if not (0 <= o[d] <= o[d + 1] <= nb and o[d + 1] - o[d] <= GIB):
                assert b
        n_bad += sum(bad)
    assert n_bad > 1000  # (the cases reach the flag)
