"""Known answers of `Sentence::from_tokenized`, restated as data from the reference's tests
(vaporetto/src/sentence.rs, tests at the cited lines), plus the first-error rules of its character loop
(sentence.rs:285-406) on lines with two violations.

Each case: (input, expected) where expected is either ("error", message) or (raw text, boundaries (1 = WordBoundary)
between characters, tags per character (n_tags entries each, None for an empty / missing field)).
"""

E = "InvalidArgumentError: tokenized_text: "
_B = [0, 0, 0, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 1, 1]  # "Rust で 良い プログラミング 体験 を ！"
_RAW = "Rustで良いプログラミング体験を！"


def _tags(n, at):
    out = [[None] * n for _ in range(len(_RAW))]
    for i, t in at.items():
        out[i] = list(t)
    return out


KAT = [
    # sentence.rs:1480 test_sentence_from_tokenized_empty
    ("", ("error", E + "must contain at least one character")),
    # sentence.rs:1508 test_sentence_from_tokenized_null
    ("A1あ\0ア亜", ("error", E + "must not contain NULL")),
    # sentence.rs:1536 test_sentence_from_tokenized_start_with_space
    (" Rust で 良い プログラミング 体験 を ！", ("error", E + "must not start with a whitespace")),
    # sentence.rs:1564 test_sentence_from_tokenized_end_with_space
    ("Rust で 良い プログラミング 体験 を ！ ", ("error", E + "must not end with a whitespace")),
    # sentence.rs:1592 test_sentence_from_tokenized_two_spaces
    ("Rust で 良い  プログラミング 体験 を ！", ("error", E + "must not contain consecutive whitespaces")),
    # sentence.rs:1620 test_sentence_from_tokenized_one
    ("あ", ("あ", [], [[]])),
    # sentence.rs:1645 test_sentence_from_tokenized
    ("Rust で 良い プログラミング 体験 を ！", (_RAW, _B, [[] for _ in _RAW])),
    # sentence.rs:1775 test_sentence_from_tokenized_with_tags
    ("Rust/名詞 で 良い/形容詞 プログラミング 体験 を ！/補助記号",
     (_RAW, _B, _tags(1, {3: ["名詞"], 6: ["形容詞"], 17: ["補助記号"]}))),
    # sentence.rs:1953 test_sentence_from_tokenized_with_tags_two_slashes
    ("Rust/名詞 で 良い/形容詞/イイ プログラミング 体験 を ！/補助記号",
     (_RAW, _B, _tags(2, {3: ["名詞", None], 6: ["形容詞", "イイ"], 17: ["補助記号", None]}))),
    # sentence.rs:2168 test_sentence_from_tokenized_with_tags_empty_slashes
    ("Rust//ラスト で 良い/形容詞/イイ プログラミング 体験 を ！//ビックリ",
     (_RAW, _B, _tags(2, {3: [None, "ラスト"], 6: ["形容詞", "イイ"], 17: [None, "ビックリ"]}))),
    # sentence.rs:2383 test_sentence_from_tokenized_with_escape_whitespace
    ("火星 猫 の 生態 ( M \\  et\\ al. )",
     ("火星猫の生態(M et al.)", [0, 1, 1, 1, 0, 1, 1, 1, 1, 0, 0, 0, 0, 0, 1], [[] for _ in range(16)])),
    # sentence.rs:2505 test_sentence_from_tokenized_with_escape_backslash
    ("改行 に \\\\n を 用い る", ("改行に\\nを用いる", [0, 1, 1, 0, 1, 1, 0, 1], [[] for _ in range(9)])),
    # sentence.rs:2586 test_sentence_from_tokenized_escape_slash
    ("品詞 に \\/ を 用い る", ("品詞に/を用いる", [0, 1, 1, 1, 1, 0, 1], [[] for _ in range(8)])),
]

# The first violation the character loop meets decides the error (sentence.rs:285-406); the trailing-whitespace check
# runs after the loop.  Derived from the loop, not from the reference's tests.
FIRST_ERROR = [
    (" a  b", E + "must not start with a whitespace"),
    ("a  b ", E + "must not contain consecutive whitespaces"),
    ("a \0 b  ", E + "must not contain NULL"),
    ("/a\0", E + "a slash must follow a character"),
    ("a /b  c", E + "a slash must follow a character"),
    ("a/b\0 c  d", E + "must not contain NULL"),
    ("a\\\0", E + "must not contain NULL"),
    ("a/x\\ y  z", E + "must not contain consecutive whitespaces"),
    ("ab /", E + "a slash must follow a character"),
    ("ab ", E + "must not end with a whitespace"),
    # a lone '\' has no character: the reference divides by zero (sentence.rs:450); here it is this error
    ("\\", E + "must contain at least one character"),
]
