"""vpt_evaluate_lines with a per-line buffer smaller than the number of lines, called through the C ABI (the Python
wrapper always sizes the buffer to the lines)."""
import ctypes
import os

import numpy as np
import pytest

import vaporetto_b200 as vb

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
MODEL = os.path.join(HERE, "golden", "model.bin")
DOCS = os.path.join(HERE, "golden", "docs.tok")


def test_line_capacity_one_row_short(monkeypatch):
    """A per-line buffer one row short returns InvalidArgument after the totals are filled in; every chunk that fits
    writes its rows as with room for all lines, and the chunk that does not fit writes none."""
    p = vb.Predictor(vb.Model.read(open(MODEL, "rb").read()), predict_tags=True)
    good = open(DOCS, "rb").read().split(b"\n")[:2]
    data = b"\n".join(b"" if i % 7 == 3 else good[i % 2] for i in range(400)) + b"\n"
    monkeypatch.setenv("VPT_CHUNK_BYTES", "1000")  # dozens of chunks
    want, full = p.evaluate_lines(data, per_line=True)
    n = full.shape[0]
    assert n == 400
    unwritten = 0xFFFFFFFF
    lc = np.full((n, 7), unwritten, np.uint32)
    counts = vb._EvalCounts()
    rc = vb.lib().vpt_evaluate_lines(p._h, data, len(data), 0, 0, 0, ctypes.byref(counts), lc.ctypes.data, n - 1)
    assert rc == 2 and b"line_capacity" in vb.lib().vpt_last_error()
    assert {name: int(getattr(counts, name)) for name, _ in vb._EvalCounts._fields_} == want
    written = int(np.count_nonzero((lc != unwritten).any(axis=1)))
    assert n // 2 < written < n  # only the last chunk's rows are missing
    assert np.array_equal(lc[:written], full[:written])
    assert (lc[written:] == unwritten).all()
