"""Partially annotated output on the host: the oracle's restatement of Sentence::write_partial_annotation_text and the
host Sentence.write_partial_annotation_text against the reference's doc examples (sentence.rs:209-212, 895-905,
1024-1030), and the oracle's vpt_annotate_lines chain at margin 0 read back by the oracle's partial parser."""
import os
import random

import pytest

import vaporetto_b200 as vb
from vpt_testlib import partial_oracle as po
from vpt_testlib.annotate_oracle import AnnotateOracle, write
from vpt_testlib.oracle import OraclePredictor

HERE = os.path.dirname(os.path.abspath(__file__))
TEXT = "まぁ良いだろう"
TOKENIZED = [0, 1, 0, 1, 0, 0]  # Sentence::from_tokenized("まぁ 良い だろう")


def from_partial(line: str):
    """Sentence::from_partial_annotation through the oracle's parser: (text, boundaries)."""
    text, given = po.parse(line.encode())
    return text.decode(), given


def test_doc_from_raw():
    assert write(TEXT, [2] * 6) == "ま ぁ 良 い だ ろ う"
    assert vb.Sentence.from_raw(TEXT).write_partial_annotation_text() == "ま ぁ 良 い だ ろ う"


def test_doc_tokenized():
    assert write(TEXT, TOKENIZED) == "ま-ぁ|良-い|だ-ろ-う"
    s = vb.Sentence.from_raw(TEXT)
    s.boundaries_mut()[:] = TOKENIZED
    assert s.write_partial_annotation_text() == "ま-ぁ|良-い|だ-ろ-う"
    # from_tokenized("まぁ/副詞/マー 良い/形容詞/ヨイ だろう/助動詞/ダロー"): the tags sit on each token's last character
    tags = [[None, None] for _ in TEXT]
    tags[1], tags[3], tags[6] = ["副詞", "マー"], ["形容詞", "ヨイ"], ["助動詞", "ダロー"]
    assert write(TEXT, TOKENIZED, tags) == "ま-ぁ/副詞/マー|良-い/形容詞/ヨイ|だ-ろ-う/助動詞/ダロー"


def test_doc_boundaries_mut():
    text, bnd = from_partial("火-星|に|行-き|ま-し た")
    bnd[6] = 1
    assert write(text, bnd) == "火-星|に|行-き|ま-し|た"
    s = vb.Sentence.from_raw(text)
    s.boundaries_mut()[:] = bnd
    assert s.write_partial_annotation_text() == "火-星|に|行-き|ま-し|た"


def test_tags_unescaped_and_trailing_none():
    """Tags are written as they are; slots after the last tag are left out, None slots before it are empty fields."""
    tags = [[None, None, None], ["a b", None, "-|/\\"], [None, None, None]]
    assert write("猫がい", [1, 2], tags) == "猫|が/a b//-|/\\ い"


@pytest.mark.parametrize("tags", [False, True])
def test_margin_zero_reads_back_as_tokenize_lines(tags):
    """margin 0: every line of the oracle's output, read by from_partial_annotation and written by
    write_tokenized_text, is the oracle's tokenize_lines line (the model's tag strings hold no marker characters)."""
    mb = open(os.path.join(HERE, "golden", "model.bin"), "rb").read()
    o, ap = OraclePredictor(mb, predict_tags=True), AnnotateOracle(mb, predict_tags=True)
    rng = random.Random(5)
    sents = ["まぁ社長は火星猫だ", "まぁ良いだろう", "火星", "社長は社長だ" * 9, "Vaporetto 1.5 と猫", "東京特許許可局",
             "ＡＢＣ１２３漢字かなカナ"]
    lines = [rng.choice(sents) for _ in range(60)] + ["", "a\0b"]
    data = "\n".join(lines).encode() + b"\n"
    got, nl = ap.lines(data, 0, predict_tags=tags)
    want, wl = o.tokenize_lines(data, predict_tags=tags)
    assert nl == wl == len(lines)
    out = [po.write(line.encode()) if line else "" for line in got.decode().split("\n")[:-1]]
    assert "\n".join(out) + "\n" == want.decode()


def test_margin_edges_in_the_oracle():
    """A score of exactly +-margin is known; margin 1 leaves only the scores 0 Unknown."""
    mb = open(os.path.join(HERE, "golden", "model.bin"), "rb").read()
    o, ap = OraclePredictor(mb), AnnotateOracle(mb)
    line = "まぁ社長は火星猫だ"
    sc, _ = o.predict(line)
    for m in sorted({abs(int(x)) for x in sc} | {1}):
        got, _ = ap.lines(line.encode() + b"\n", m, no_norm=True)
        marks = got.decode()[1:-1:2]
        assert [c == " " for c in marks] == [-m < int(x) < m for x in sc]
