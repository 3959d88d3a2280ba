"""The evaluate command's pieces that run without a GPU: the tokenized-text parser of the test oracle against the
reference's known answers, the oracle's metric loops on hand-derived cases, and the CLI's output formatting."""
import importlib.util
import math
import os
import subprocess
import sys

import pytest

from golden.tokenized_kat import FIRST_ERROR, KAT
from vpt_testlib import eval_oracle as eo

HERE = os.path.dirname(os.path.abspath(__file__))
CLI = os.path.join(os.path.dirname(HERE), "tools", "evaluate_cli.py")
MODEL = os.path.join(HERE, "golden", "model.bin")

_spec = importlib.util.spec_from_file_location("evaluate_cli", CLI)
cli = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(cli)


@pytest.mark.parametrize("line,want", KAT)
def test_parse_tokenized_kat(line, want):
    if want[0] == "error":
        with pytest.raises(eo.GoldError) as e:
            eo.parse_tokenized(line)
        assert e.value.msg == want[1] and e.value.code == eo.INVALID_ARGUMENT
    else:
        assert eo.parse_tokenized(line) == want


@pytest.mark.parametrize("line,msg", FIRST_ERROR)
def test_parse_tokenized_first_error(line, msg):
    with pytest.raises(eo.GoldError) as e:
        eo.parse_tokenized(line)
    assert e.value.msg == msg


def test_parse_tokenized_tags_unescaped():
    """Tag fields hold the unescaped characters; an escaped ' ' or '/' stays inside the field."""
    raw, b, tags = eo.parse_tokenized("a/x\\ y\\/z/ b\\/c/\\\\")
    assert raw == "ab/c" and b == [1, 0, 0]
    assert tags == [["x y/z", None], [None, None], [None, None], ["\\", None]]


def test_bufread_lines():
    assert eo.bufread_lines(b"") == []
    assert eo.bufread_lines(b"a\r\n\nb\r") == [b"a", b"", b"b\r"]
    assert eo.bufread_lines(b"a\n\r\n") == [b"a", b""]


def test_metrics_hand_derived():
    """gold "a b c" against system "ab c": TP 1, FN 1; word metric n_sys 2, n_ref 3, n_cor 1."""
    _, ref_b, ref_t = eo.parse_tokenized("a b c")
    _, sys_b, sys_t = eo.parse_tokenized("ab c")
    res = [(ref_b, ref_t, sys_b, sys_t)]
    c = eo.char_metric(res)
    assert c == {"tp": 1, "tn": 0, "fp": 0, "fn": 1}
    w = eo.word_metric(res)
    assert w == {"n_sys": 2, "n_ref": 3, "n_cor": 1}
    assert cli.report(c, "char") == "Precision: 1\nRecall: 0.5\nF1: 0.6666666666666666\nTP: 1, TN: 0, FP: 0, FN: 1\n"
    assert cli.report(w, "word") == ("Precision: 0.5\nRecall: 0.3333333333333333\nF1: 0.4\n")


def test_word_metric_tags_and_matched():
    """A token counts only when no boundary disagreed since the last shared one, and its tags are equal."""
    _, rb, rt = eo.parse_tokenized("ab/X c/Y d")
    _, sb, st = eo.parse_tokenized("ab/X c/Z d")
    assert eo.word_metric([(rb, rt, sb, st)]) == {"n_sys": 3, "n_ref": 3, "n_cor": 2}
    _, sb2, st2 = eo.parse_tokenized("a b/X c/Y d")
    assert eo.word_metric([(rb, rt, sb2, st2)]) == {"n_sys": 4, "n_ref": 3, "n_cor": 2}


def test_rust_f64_display():
    cases = [(1.0, "1"), (0.5, "0.5"), (0.000005, "0.000005"), (1e-7, "0.0000001"), (math.nan, "NaN"),
             (2 / 3, "0.6666666666666666"), (0.0, "0"), (1e16, "10000000000000000"), (123.25, "123.25"),
             (0.1 + 0.2, "0.30000000000000004"), (math.inf, "inf"), (-0.0, "-0")]
    for x, want in cases:
        assert cli.rust_f64(x) == want, x


def test_report_empty_is_nan():
    zero = dict.fromkeys(("tp", "tn", "fp", "fn", "n_sys", "n_ref", "n_cor"), 0)
    assert cli.report(zero, "char") == "Precision: NaN\nRecall: NaN\nF1: NaN\nTP: 0, TN: 0, FP: 0, FN: 0\n"
    assert cli.report(zero, "word") == "Precision: NaN\nRecall: NaN\nF1: NaN\n"
    # all tokens wrong: precision and recall 0, F1 0 / 0
    assert cli.report({"n_sys": 2, "n_ref": 2, "n_cor": 0}, "word") == "Precision: 0\nRecall: 0\nF1: NaN\n"


def test_cli_rejects_unknown_options():
    out = subprocess.run([sys.executable, CLI, "--model", MODEL, "--metric", "chars"], input=b"", capture_output=True)
    assert out.returncode != 0 and b"invalid choice" in out.stderr
