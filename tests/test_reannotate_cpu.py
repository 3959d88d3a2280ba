"""Re-annotation on the host: the input tag regions of k_part_tags (partial_parse.hpp) against the reference loop's tag
handling over every short string of the format's symbols, and the oracle's vpt_reannotate_lines chain on hand-written
lines whose output the definitions of the C header fix."""
import ctypes as C
import os

import pytest

from vpt_testlib import oracle
from vpt_testlib import partial_oracle as po
from vpt_testlib.reannotate_oracle import ReannotateOracle, tags_test_lib

HERE = os.path.dirname(os.path.abspath(__file__))
MAXM = 2**31 - 1


def test_tag_regions_every_string_up_to_7_symbols():
    msg = C.create_string_buffer(1024)
    n = tags_test_lib().rt_check_all(7, msg, 1024)
    assert n == sum(10 ** k for k in range(1, 8)), msg.value.decode()


@pytest.fixture(scope="module")
def ora():
    return ReannotateOracle(open(os.path.join(HERE, "golden", "model.bin"), "rb").read(), predict_tags=True)


def run(o, line: str, **kw) -> str:
    out, nl = o.lines((line + "\n").encode(), **kw)
    assert nl == 1
    return out.decode()[:-1]


# (input, keyword arguments, output): every marker given, so the model decides nothing but the tags
CASES = [
    ("escaped_slash_and_backslash", "猫/a\\/b/c\\\\d|だ", {}, "猫/a/b/c\\d|だ"),
    ("escaped_marker_in_tag", "猫/x\\|y\\ z\\-w|だ", {}, "猫/x|y z-w|だ"),
    ("empty_and_trailing_empty_fields", "猫//x//|だ/|は", {}, "猫//x|だ|は"),
    ("only_empty_fields_carry_none", "猫/|だ//", {}, "猫|だ"),
    ("mid_token_character", "火/名詞-星|猫", {}, "火/名詞-星|猫"),
    ("last_character", "火-星/名詞/カセー", {}, "火-星/名詞/カセー"),
    ("dropped", "火/名詞-星/x|猫", {"keep_tags": False}, "火-星|猫"),
    ("wsconst_k_keeps_given_word_boundary", "火|星", {"wsconst": "K", "margin": MAXM}, "火|星"),
    ("wsconst_k_clears_open_boundary", "火 星", {"wsconst": "K", "margin": MAXM}, "火-星"),
    ("tags_next_to_open_boundary", "火/X 星/Y", {"margin": MAXM}, "火/X 星/Y"),
]


@pytest.mark.parametrize("line,kw,want", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_hand_written(ora, line, kw, want):
    assert run(ora, line, **kw) == want


def test_predicted_tags_and_kept_tags(ora):
    """The model's tags on every token end that carries no input tags; the input's where it does."""
    line = "ま-ぁ|社-長|は|火-星|猫/X|だ"
    assert run(ora, line, predict_tags=True) == "ま-ぁ/名詞/マー|社-長/名詞/シャチョー|は/助詞/ワ|火-星/名詞/カセー|猫/X|だ/助動詞/ダ"
    assert run(ora, line, predict_tags=True, keep_tags=False) == \
        "ま-ぁ/名詞/マー|社-長/名詞/シャチョー|は/助詞/ワ|火-星/名詞/カセー|猫/名詞/ネコ|だ/助動詞/ダ"
    # open boundaries: the tokens next to them get no model tags, the input tags stay
    got = run(ora, "ま ぁ/X 社", predict_tags=True, margin=MAXM)
    assert got == "ま ぁ/X 社"


def test_margin_zero_decides_every_open_boundary(ora):
    got = run(ora, "ま ぁ 社 長 は 火 星 猫 だ")
    assert " " not in got and got.replace("|", "").replace("-", "") == "まぁ社長は火星猫だ"
    # given markers are written as given, even against the model
    assert run(ora, "ま|ぁ-社 長") .startswith("ま|ぁ-社")


def test_empty_lines_and_errors(ora):
    out, nl = ora.lines(b"\n\r\n")
    assert out == b"\n\n" and nl == 2
    for bad, code in ((b"a|b\n\xe7\x8c|\xff\n", 5), (b"a|b\n\xe7\x8c\xab?b\n", 2), (b"a|b\nab|\n", 2)):
        with pytest.raises(oracle.OracleError) as e:
            ora.lines(bad)
        want = po.PartialOracle(open(os.path.join(HERE, "golden", "model.bin"), "rb").read()).lines(bad)
        assert want[2] == (code, e.value.message) and e.value.message.endswith(" (line 1)")
        assert e.value.output == b"a|b\n"
