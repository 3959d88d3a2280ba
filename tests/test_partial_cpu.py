"""Partially annotated lines on the host: the oracle's restatement of Sentence::from_partial_annotation against the
reference's own tests and doc examples (tests/golden/partial_annotation_kat.json), and the byte automaton of
k_part_parse (partial_parse.hpp) against that restatement over every short string of the format's symbols."""
import ctypes as C
import json
import os

import pytest

from vpt_testlib import oracle
from vpt_testlib import partial_oracle as po

KAT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "partial_annotation_kat.json"), encoding="utf-8"))


@pytest.mark.parametrize("case", KAT["errors"], ids=lambda c: c["name"])
def test_kat_errors(case):
    with pytest.raises(oracle.OracleError) as e:
        po.parse(case["input"].encode())
    assert e.value.message == case["error"]


@pytest.mark.parametrize("case", KAT["parses"], ids=lambda c: c["name"])
def test_kat_parses(case):
    text, given = po.parse(case["input"].encode())
    assert text.decode() == case["raw_text"]
    assert given == case["boundaries"]
    pos = [0]
    for ch in case["raw_text"]:
        pos.append(pos[-1] + len(ch.encode()))
    assert pos == case["char_to_str_pos"]


@pytest.mark.parametrize("case", KAT["tokenized"], ids=range(len(KAT["tokenized"])))
def test_kat_tokenized(case):
    assert po.write(case["input"].encode()) == case["output"]


def test_automaton_every_string_up_to_7_symbols():
    msg = C.create_string_buffer(1024)
    n = po.parse_test_lib().pp_check_all(7, msg, 1024)
    assert n == sum(10 ** k for k in range(1, 8)), msg.value.decode()
