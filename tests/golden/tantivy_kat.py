"""Known answers of vaporetto_tantivy's token stream and of SplitLinebreaksFilter, transcribed from the reference's tests.

TANTIVY_TOKEN_STREAMS: vaporetto_tantivy/src/lib.rs:256-491 (test_tokenize_empty, test_tokenizer_tokyo,
test_tokenizer_no_wsconst, test_tokenize_wsconst_d, test_tokenizer_wsconst_g, test_tokenize_wsconst_dg) with
test_model/model.zst (tests/golden/tantivy_model.bin): (text, wsconst, [(text, offset_from, offset_to, position,
position_length), ...]).

SPLIT_LINEBREAKS: vaporetto_rules/src/sentence_filters/split_linebreaks.rs:43-78 (test_split_lf, test_split_cr,
test_split_crlf): (raw text, tokens after the filter).  The sentences come from `Sentence::from_tokenized` of the raw
text, i.e. every boundary starts as NotWordBoundary, so the tokens are the line breaks and the runs between them.
"""


def _tokens(pairs):
    n = len(pairs)
    return [(t, a, b, i, n) for i, (t, a, b) in enumerate(pairs)]


TANTIVY_TOKEN_STREAMS = [
    ("", "", []),
    ("東京特許許可局", "", _tokens([("東京", 0, 6), ("特許", 6, 12), ("許可", 12, 18), ("局", 18, 21)])),
    ("123456円🤌🏿", "", _tokens([("1", 0, 1), ("2", 1, 2), ("3", 2, 3), ("4", 3, 4), ("5", 4, 5), ("6", 5, 6),
                                  ("円", 6, 9), ("🤌", 9, 13), ("🏿", 13, 17)])),
    ("123456円🤌🏿", "D", _tokens([("123456", 0, 6), ("円", 6, 9), ("🤌", 9, 13), ("🏿", 13, 17)])),
    ("123456円🤌🏿", "G", _tokens([("1", 0, 1), ("2", 1, 2), ("3", 2, 3), ("4", 3, 4), ("5", 4, 5), ("6", 5, 6),
                                   ("円", 6, 9), ("🤌🏿", 9, 17)])),
    ("123456円🤌🏿", "DG", _tokens([("123456", 0, 6), ("円", 6, 9), ("🤌🏿", 9, 17)])),
]

SPLIT_LINEBREAKS = [
    ("前の行\n次の行", ["前の行", "\n", "次の行"]),
    ("前の行\r次の行", ["前の行", "\r", "次の行"]),
    ("前の行\r\n次の行", ["前の行", "\r", "\n", "次の行"]),
]
