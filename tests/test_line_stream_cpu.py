"""The line stream's chunk cutting (vaporetto_b200/csrc/line_feed.hpp) on the host, and the argument checks of the Python
LineStream that need no device.  The GPU side is tests/test_gpu_line_stream.py."""
import os
import subprocess

import pytest

import vaporetto_b200 as vb

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "native", "line_feed_test.cpp")
HDR = os.path.join(ROOT, "vaporetto_b200", "csrc", "line_feed.hpp")


def test_line_feed_cuts(tmp_path):
    """Thousands of random byte strings x feed splits x chunk sizes x flush points: the chunks concatenate to the input,
    every chunk but the last ends in '\\n', a chunk over its nominal size is one line, a flush leaves no complete line
    held, a line over the limit is reported, and no input gives no chunks."""
    exe = str(tmp_path / "line_feed_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-o", exe, SRC])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.startswith("line feed ok")


def test_stream_arguments_without_device():
    """Argument errors are raised before the library is asked for a stream."""
    p = vb.Predictor.__new__(vb.Predictor)  # no device: the checks below come first
    p._h = None
    with pytest.raises(vb.VaporettoError) as e:
        p.line_stream(kind="segment")
    assert e.value.code == 2 and "kind" in str(e.value)
    with pytest.raises(vb.VaporettoError) as e:
        p.line_stream(wsconst="X")
    assert e.value.code == 2 and "wsconst" in str(e.value)


def test_stream_abi_without_device():
    """The C calls reject NULL handles and refuse to stream on a host-only predictor (there is no CPU fallback)."""
    L = vb.lib()
    assert L.vpt_line_stream_feed(None, b"a", 1) == 2
    assert L.vpt_line_stream_flush(None) == 2
    assert L.vpt_line_stream_finish(None, None, None) == 2
    L.vpt_line_stream_free(None)  # a no-op
    model = vb.Model.read(open(os.path.join(HERE, "golden", "model.bin"), "rb").read())
    host_only = vb.Predictor(model, device=-1)
    with pytest.raises(vb.VaporettoError) as e:
        host_only.line_stream()
    assert e.value.kind == "CudaError"
