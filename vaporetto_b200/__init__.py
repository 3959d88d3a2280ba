"""vaporetto_b200 — Python mirror of the reference's `Model` / `Predictor` / `Sentence` API
(vaporetto/src/lib.rs:82-91) over the C ABI of libvaporetto_b200.so (include/vaporetto_b200.h).

The compute path is the CUDA library; there is no CPU fallback.  Importing this package works without a GPU
(so the ABI can be inspected), creating a `Predictor` does not.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import numpy as np

__all__ = ["Model", "Predictor", "Sentence", "VaporettoError", "CharacterBoundary", "CharacterType", "lib", "build",
           "BatchResult", "build_blob", "shard_by_bytes", "LineStream", "SpansResult", "SpanToken", "Tokenizer",
           "PatternMatchTagger", "DeviceSpans", "DeviceText"]

_PKG = os.path.dirname(os.path.abspath(__file__))
_SO = os.environ.get("VPT_B200_LIBRARY") or os.path.join(_PKG, "libvaporetto_b200.so")  # (override: A/B builds)


def build(force: bool = False) -> str:
    """Compile the CUDA extension in-tree with nvcc for sm_90a (see csrc/Makefile)."""
    import subprocess
    csrc = os.path.join(_PKG, "csrc")
    if force and os.path.exists(_SO):
        os.remove(_SO)
    subprocess.check_call(["make", "-C", csrc, "-s"])
    return _SO


class VaporettoError(Exception):
    """Mirror of `VaporettoError` (vaporetto/src/errors.rs:15-38)."""

    KIND = {1: "InvalidModel", 2: "InvalidArgument", 3: "InvalidSentence", 4: "DecodeError", 5: "IOError",
            16: "CudaError", 17: "Unsupported", 18: "Internal"}

    def __init__(self, code: int, msg: str):
        super().__init__(msg)
        self.code = code
        self.kind = self.KIND.get(code, "Unknown")


class CharacterBoundary:  # sentence.rs:70-82
    NotWordBoundary = 0
    WordBoundary = 1
    Unknown = 2


class CharacterType:  # sentence.rs:9-29
    Digit, Roman, Hiragana, Katakana, Kanji, Other = 1, 2, 3, 4, 5, 6


class _Info(C.Structure):
    _fields_ = [("device", C.c_int32), ("predict_tags", C.c_int32), ("n_tags", C.c_int32), ("char_scorer", C.c_int32),
                ("type_scorer", C.c_int32), ("fast_path", C.c_int32), ("bias", C.c_int32), ("char_window", C.c_int32),
                ("type_window", C.c_int32), ("n_char_patterns", C.c_uint32), ("n_type_patterns", C.c_uint32),
                ("n_char_nodes", C.c_uint32), ("n_type_nodes", C.c_uint32), ("max_char_pattern_len", C.c_uint32),
                ("blob_bytes", C.c_uint64), ("kernel_launches_per_batch", C.c_int32)]


class _KernelPlan(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("kernel", "seeds_smem", "common_shape", "deep", "states", "r0_fixed", "general",
                                         "split3", "overflow", "text_cap", "slot_cap", "gap", "lag", "sub_blocks", "group")]


KERNEL_NAMES = {1: "k_fused", 2: "k_tile_fast", 3: "k_score_fast", 4: "k_score_general"}


# every symbol include/vaporetto_b200.h declares: (name, restype, argtypes)
_P = C.c_void_p
ABI = [
    ("vpt_last_error", C.c_char_p, []),
    ("vpt_version", C.c_char_p, []),
    ("vpt_model_read", C.c_int, [C.c_char_p, C.c_size_t, C.POINTER(_P), C.POINTER(C.c_size_t)]),
    ("vpt_model_free", None, [_P]),
    ("vpt_model_read_kytea", C.c_int, [C.c_char_p, C.c_size_t, C.POINTER(_P)]),
    ("vpt_concat_grapheme_clusters", C.c_int, [C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    ("vpt_split_linebreaks", C.c_int, [C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    ("vpt_model_read_zstd", C.c_int, [C.c_char_p, C.c_size_t, C.POINTER(_P)]),
    ("vpt_model_to_vec", C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_uint64)]),
    ("vpt_model_dictionary_len", C.c_uint64, [_P]),
    ("vpt_model_dictionary_get", C.c_int, [_P, C.c_uint64, C.POINTER(C.c_char_p), C.POINTER(_P), C.POINTER(C.c_uint64),
                                          C.POINTER(C.c_char_p)]),
    ("vpt_model_replace_dictionary", C.c_int, [_P, _P, _P, _P, _P, C.c_uint64]),
    ("vpt_predictor_new", C.c_int, [_P, C.c_int, C.c_int, C.POINTER(_P)]),
    ("vpt_predictor_free", None, [_P]),
    ("vpt_predictor_get_info", C.c_int, [_P, C.POINTER(_Info)]),
    ("vpt_predictor_kernel_plan", C.c_int, [_P, C.c_int, C.POINTER(_KernelPlan)]),
    ("vpt_blob_build", C.c_int, [_P, C.c_int, C.POINTER(_P), C.POINTER(C.c_uint64)]),
    ("vpt_blob_free", None, [_P]),
    ("vpt_predictor_blob_size", C.c_uint64, [_P]),
    ("vpt_predictor_blob_export", C.c_int, [_P, _P, C.c_uint64]),
    ("vpt_predictor_from_blob", C.c_int, [_P, C.c_uint64, C.c_int, C.POINTER(_P)]),
    ("vpt_predict_batch", C.c_int, [_P, _P, _P, C.c_size_t, _P, _P, C.c_size_t, _P, _P, _P, _P, C.c_size_t, _P,
                                    C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    ("vpt_workspace_size", C.c_uint64, [C.c_size_t]),
    ("vpt_predict_batch_dev", C.c_int, [_P, _P, _P, C.c_size_t, _P, C.c_uint64, _P, _P, _P, _P, _P, _P, _P, _P]),
    ("vpt_predict_batch_dev_profiled", C.c_int, [_P, _P, _P, C.c_size_t, _P, C.c_uint64, _P, _P, _P, _P, _P, _P, _P, _P,
                                                 _P]),
    ("vpt_predict", C.c_int, [_P, C.c_char_p, C.c_size_t, _P, _P, C.c_size_t, _P, _P, C.c_size_t, C.POINTER(C.c_uint64)]),
    ("vpt_fill_tags", C.c_int, [_P, C.c_char_p, C.c_size_t, _P, _P, _P, _P, _P, _P, C.c_size_t]),
    ("vpt_tag_string", C.c_char_p, [_P, C.c_uint32, C.c_uint32, C.c_uint32]),
    ("vpt_tag_n_candidates", C.c_uint32, [_P, C.c_uint32, C.c_uint32]),
    ("vpt_tag_score_len", C.c_uint32, [_P, C.c_uint32]),
    ("vpt_tag_n_tokens", C.c_uint32, [_P]),
    ("vpt_char_types", C.c_int, [C.c_char_p, C.c_size_t, _P, C.c_size_t, C.POINTER(C.c_uint64)]),
    ("vpt_write_tokenized_text", C.c_int, [_P, C.c_char_p, C.c_size_t, _P, _P, _P, _P, C.c_size_t,
                                           C.POINTER(C.c_uint64)]),
    ("vpt_tokenize_lines", C.c_int, [_P, _P, C.c_size_t, C.c_int, C.c_uint32, _P, C.c_size_t, C.POINTER(C.c_uint64),
                                     C.POINTER(C.c_uint64)]),
    ("vpt_kytea_fullwidth", C.c_uint32, [C.c_uint32]),
    ("vpt_device_pci_bus_id", C.c_int, [C.c_int, C.c_char_p, C.c_size_t]),
    ("vpt_predict_tags_batch_dev", C.c_int, [_P, _P, _P, C.c_size_t, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    ("vpt_predict_batch_tags", C.c_int, [_P, _P, _P, C.c_size_t, _P, _P, C.c_size_t, _P, _P, _P, _P, C.c_size_t, _P,
                                         C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    ("vpt_predict_batch_compact", C.c_int, [_P, _P, _P, C.c_size_t, _P, C.c_size_t, _P, _P, _P, _P, _P, C.c_size_t,
                                            C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    ("vpt_unpack_boundaries", C.c_int, [_P, C.c_uint64, C.c_uint64, _P]),
    ("vpt_tokenize_lines_tags", C.c_int, [_P, _P, C.c_size_t, C.c_int, C.c_uint32, _P, C.c_size_t,
                                          C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    ("vpt_evaluate_lines", C.c_int, [_P, _P, C.c_size_t, C.c_int, C.c_uint32, C.c_int, _P, _P, C.c_uint64]),
    ("vpt_line_stream_new", C.c_int, [_P, C.c_int, C.c_int, C.c_uint32, C.c_int, _P, _P, C.POINTER(_P)]),
    ("vpt_line_stream_feed", C.c_int, [_P, _P, C.c_size_t]),
    ("vpt_line_stream_flush", C.c_int, [_P]),
    ("vpt_line_stream_finish", C.c_int, [_P, C.POINTER(C.c_uint64), _P]),
    ("vpt_line_stream_free", None, [_P]),
    ("vpt_tag_rules_new", C.c_int, [_P, C.c_uint64, _P, _P, _P, _P, _P, C.c_uint64, C.POINTER(_P)]),
    ("vpt_tag_rules_free", None, [_P]),
    ("vpt_tag_rules_max_output", C.c_uint64, [_P]),
    ("vpt_tokenize_lines_tags_rules", C.c_int, [_P, _P, _P, C.c_size_t, C.c_int, C.c_uint32, _P, C.c_size_t,
                                                C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    ("vpt_line_stream_new_rules", C.c_int, [_P, _P, C.c_int, C.c_int, C.c_uint32, C.c_int, _P, _P, C.POINTER(_P)]),
    ("vpt_line_stream_new_scores", C.c_int, [_P, _P, C.c_int, C.c_uint32, C.c_int, C.c_uint32, _P, _P, C.POINTER(_P)]),
    ("vpt_tokenize_partial_lines", C.c_int, [_P, _P, _P, C.c_size_t, C.c_int, C.c_uint32, C.c_int, _P, C.c_size_t,
                                             C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    ("vpt_line_stream_new_partial", C.c_int, [_P, _P, C.c_int, C.c_uint32, C.c_int, _P, _P, C.POINTER(_P)]),
    ("vpt_annotate_lines", C.c_int, [_P, _P, _P, C.c_size_t, C.c_int, C.c_uint32, C.c_int, C.c_int32, _P, C.c_size_t,
                                     C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    ("vpt_line_stream_new_annotate", C.c_int, [_P, _P, C.c_int, C.c_uint32, C.c_int, C.c_int32, _P, _P, C.POINTER(_P)]),
    ("vpt_reannotate_lines", C.c_int, [_P, _P, _P, C.c_size_t, C.c_int, C.c_uint32, C.c_int, C.c_int32, C.c_int, _P,
                                       C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    ("vpt_line_stream_new_reannotate", C.c_int, [_P, _P, C.c_int, C.c_uint32, C.c_int, C.c_int32, C.c_int, _P, _P,
                                                 C.POINTER(_P)]),
    ("vpt_write_partial_annotation_text", C.c_int, [_P, _P, C.c_size_t, _P, _P, _P, _P, C.c_size_t, C.POINTER(C.c_uint64)]),
    ("vpt_token_spans", C.c_int, [_P, _P, _P, C.c_size_t, C.c_int, C.c_uint32, _P, _P, _P, _P, _P, C.c_size_t,
                                  C.POINTER(C.c_uint64)]),
    ("vpt_tag_n_slots", C.c_uint32, [_P, C.c_uint32]),
    ("vpt_predict_batch_compact_tag_scores", C.c_int, [_P, _P, _P, C.c_size_t, _P, C.c_size_t, _P, _P, _P, _P, _P,
                                                       C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                                       C.POINTER(C.c_uint64), _P, C.c_size_t, C.POINTER(C.c_uint64)]),
    ("vpt_token_spans_tag_scores", C.c_int, [_P, _P, _P, C.c_size_t, C.c_int, C.c_uint32, _P, _P, _P, _P, _P, C.c_size_t,
                                             C.POINTER(C.c_uint64), _P, C.c_size_t, C.POINTER(C.c_uint64)]),
    ("vpt_token_spans_dev_workspace_size", C.c_uint64, [_P, C.c_size_t, C.c_uint64, C.c_int]),
    ("vpt_token_spans_dev", C.c_int, [_P, _P, C.c_uint64, _P, C.c_int, C.c_size_t, C.c_int, C.c_uint32, _P, _P, _P, _P, _P,
                                      _P, _P, C.c_uint64, _P]),
    ("vpt_tokenize_dev_workspace_size", C.c_uint64, [_P, _P, C.c_size_t, C.c_uint64, C.c_int]),
    ("vpt_tokenize_dev_out_bound", C.c_uint64, [_P, _P, C.c_size_t, C.c_uint64, C.c_int]),
    ("vpt_tokenize_dev", C.c_int, [_P, _P, _P, C.c_uint64, _P, C.c_int, C.c_size_t, C.c_int, C.c_uint32, C.c_int, _P, _P,
                                   C.c_uint64, _P, _P, C.c_uint64, _P]),
]

# vpt_stream_write_fn: int (*)(void* ctx, const uint8_t* bytes, size_t n)
STREAM_WRITE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t)
STREAM_KINDS = {"tokenize": 0, "evaluate": 1}
DUMP_SCORES, DUMP_TAG_SCORES = 1, 2  # VPT_DUMP_SCORES, VPT_DUMP_TAG_SCORES

_lib = None


def lib():
    """Loads libvaporetto_b200.so; fails loudly if the extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            raise ImportError(f"{_SO} is missing: the CUDA extension must be built first "
                              f"(python -c 'import __graft_entry__ as g; g.build()'); there is no CPU fallback")
        L = C.CDLL(_SO)
        for name, res, args in ABI:
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def _check(rc: int):
    if rc != 0:
        raise VaporettoError(rc, lib().vpt_last_error().decode("utf-8", "replace"))


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data


class Model:
    """`vaporetto::Model` (model.rs:58-168): an on-disk model image."""

    def __init__(self, handle, consumed: int):
        self._h = handle
        self.consumed = consumed

    @classmethod
    def read(cls, src) -> "Model":
        """`Model::read` (model.rs:142-153): file-like object or bytes with the raw (un-zstd'd) model."""
        data = src if isinstance(src, (bytes, bytearray, memoryview)) else src.read()
        return cls.read_slice(bytes(data))[0]

    @classmethod
    def read_slice(cls, data: bytes):
        """`Model::read_slice` (model.rs:127-134): returns (model, remaining bytes)."""
        h = _P()
        used = C.c_size_t()
        _check(lib().vpt_model_read(data, len(data), C.byref(h), C.byref(used)))
        return cls(h, used.value), data[used.value:]

    @classmethod
    def read_zstd(cls, src) -> "Model":
        """`Model::read(&mut zstd::Decoder::new(file)?)` (predict/src/main.rs:110-111): a *.model.zst image, decoded by
        the library (libzstd.so.1); a raw model image is accepted as well."""
        data = src if isinstance(src, (bytes, bytearray, memoryview)) else src.read()
        data = bytes(data)
        h = _P()
        _check(lib().vpt_model_read_zstd(data, len(data), C.byref(h)))
        return cls(h, len(data))

    @classmethod
    def read_kytea(cls, src) -> "Model":
        """`KyteaModel::read` + `Model::try_from` (kytea_model.rs:423-550): converts a KyTea binary model."""
        data = src if isinstance(src, (bytes, bytearray, memoryview)) else src.read()
        data = bytes(data)
        h = _P()
        _check(lib().vpt_model_read_kytea(data, len(data), C.byref(h)))
        return cls(h, len(data))

    def to_vec(self) -> bytes:
        """`Model::to_vec` (model.rs:99-104): the model file image."""
        if self._h is None:
            raise VaporettoError(2, "InvalidArgumentError: model: already consumed by Predictor::new")
        out = _P()
        n = C.c_uint64()
        _check(lib().vpt_model_to_vec(self._h, C.byref(out), C.byref(n)))
        try:
            return C.string_at(out, n.value)
        finally:
            lib().vpt_blob_free(out)

    def dictionary(self):
        """`Model::dictionary` (model.rs:155-158): [(word, weights, comment)]."""
        out = []
        for i in range(lib().vpt_model_dictionary_len(self._h)):
            w, c = C.c_char_p(), C.c_char_p()
            p, n = _P(), C.c_uint64()
            _check(lib().vpt_model_dictionary_get(self._h, i, C.byref(w), C.byref(p), C.byref(n), C.byref(c)))
            weights = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_int32)), shape=(n.value,)).tolist() if n.value else []
            out.append((w.value.decode("utf-8"), weights, c.value.decode("utf-8")))
        return out

    def replace_dictionary(self, records) -> None:
        """`Model::replace_dictionary` (model.rs:160-163); records: [(word, weights, comment)] checked like
        `WordWeightRecord::new` (dict_model.rs:39-50)."""
        n = len(records)
        words = (C.c_char_p * max(n, 1))(*[r[0].encode("utf-8") for r in records])
        comments = (C.c_char_p * max(n, 1))(*[r[2].encode("utf-8") for r in records])
        arrays = [np.ascontiguousarray(r[1], np.int32) for r in records]
        wptr = (_P * max(n, 1))(*[a.ctypes.data for a in arrays])
        lens = (C.c_uint64 * max(n, 1))(*[a.size for a in arrays])
        _check(lib().vpt_model_replace_dictionary(self._h, words, wptr, lens, comments, n))

    def _take(self):
        h, self._h = self._h, None
        if h is None:
            raise VaporettoError(2, "InvalidArgumentError: model: already consumed by Predictor::new")
        return h

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h and _lib is not None:  # (module globals are already gone when the interpreter shuts down)
            _lib.vpt_model_free(h)


def build_blob(model: Model, predict_tags: bool = False) -> np.ndarray:
    """Host-only build of the flat device model (vpt_blob_build); consumes `model`.  The blob can be broadcast
    as bytes and turned into a predictor on every rank with Predictor.from_blob."""
    out = _P()
    n = C.c_uint64()
    _check(lib().vpt_blob_build(model._take(), int(predict_tags), C.byref(out), C.byref(n)))
    try:
        return np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_uint8)), shape=(n.value,)).copy()
    finally:
        lib().vpt_blob_free(out)


def shard_by_bytes(offsets, rank: int, world: int):
    """Contiguous sentence range [lo, hi) of `rank` when a batch is split over `world` ranks balanced by bytes
    (SURVEY.md §8e).  Every sentence belongs to exactly one rank."""
    off = np.asarray(offsets, np.uint64)
    n = off.size - 1
    total = int(off[-1] - off[0])
    cuts = [int(np.searchsorted(off, int(off[0]) + total * r // world, side="left")) for r in range(world + 1)]
    cuts[0], cuts[-1] = 0, n
    cuts = [min(max(c, 0), n) for c in cuts]
    for i in range(1, world + 1):
        cuts[i] = max(cuts[i], cuts[i - 1])
    return cuts[rank], cuts[rank + 1]


def shard_lines(data, rank: int, world: int):
    """Byte range [lo, hi) of `rank` when a buffer of lines (the input of Predictor.tokenize_lines) is split over
    `world` ranks: cuts are placed after the first '\n' at or after every r/world-th byte, so every line belongs to
    exactly one rank and the concatenation of the ranks' outputs equals the single-process output."""
    t = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else np.ascontiguousarray(data, np.uint8)
    n = t.size
    cuts = [0]
    for r in range(1, world):
        p = max(n * r // world, cuts[-1])
        nl = np.flatnonzero(t[p:] == 10)
        cuts.append(p + int(nl[0]) + 1 if p < n and nl.size else n)
    cuts.append(n)
    return cuts[rank], cuts[rank + 1]


class BatchResult:
    """Outputs of a batched predict: flat arrays + per-sentence offsets."""

    def __init__(self, scores, boundaries, bound_offsets, status, char_states=None, type_states=None,
                 char_offsets=None):
        self.scores = scores
        self.boundaries = boundaries
        self.bound_offsets = bound_offsets
        self.status = status
        self.char_states = char_states
        self.type_states = type_states
        self.char_offsets = char_offsets

    def sentence_scores(self, i: int) -> np.ndarray:
        return self.scores[int(self.bound_offsets[i]):int(self.bound_offsets[i + 1])]

    def sentence_boundaries(self, i: int) -> np.ndarray:
        return self.boundaries[int(self.bound_offsets[i]):int(self.bound_offsets[i + 1])]


class Predictor:
    """`vaporetto::Predictor` (predictor.rs:434-665) resident on one CUDA device."""

    def __init__(self, model: Model, predict_tags: bool = False, device: int = 0):
        """`Predictor::new(model, predict_tags)` — consumes `model` (predictor.rs:450)."""
        h = _P()
        _check(lib().vpt_predictor_new(model._take(), int(predict_tags), device, C.byref(h)))
        self._h = h
        self._load_info()

    @classmethod
    def from_blob(cls, blob, device: int = 0) -> "Predictor":
        self = cls.__new__(cls)
        b = np.ascontiguousarray(np.frombuffer(blob, dtype=np.uint8))
        h = _P()
        _check(lib().vpt_predictor_from_blob(b.ctypes.data, b.size, device, C.byref(h)))
        self._h = h
        self._load_info()
        return self

    def _load_info(self):
        info = _Info()
        _check(lib().vpt_predictor_get_info(self._h, C.byref(info)))
        self.info = {k: getattr(info, k) for k, _ in _Info._fields_}
        self.n_tags = info.n_tags
        self.predict_tags = bool(info.predict_tags)
        self._store_tag_scores = False
        self._score_len_table = None

    def store_tag_scores(self, flag: bool) -> None:
        """`Predictor::store_tag_scores(flag)` (predictor.rs:511-514): Sentence.fill_tags keeps every known token's score
        vector, for Token.tag_candidates."""
        self._store_tag_scores = bool(flag)

    def _score_lens(self) -> np.ndarray:
        """vpt_tag_score_len of every token id (int64), built once per predictor."""
        if self._score_len_table is None:
            L = lib()
            n = L.vpt_tag_n_tokens(self._h)
            self._score_len_table = np.array([L.vpt_tag_score_len(self._h, t) for t in range(n)], np.int64)
        return self._score_len_table

    def tag_candidates(self, token_id: int, scores) -> list:
        """`Token::tag_candidates` (sentence.rs:1219-1250) of a token with id `token_id` (-1: none) and score vector
        `scores`: one list of (tag, score) per tag slot of the token's own model; a slot with one candidate gives
        (tag, 0), an empty slot gives []."""
        return _tag_candidates(self, token_id, scores)

    def kernel_plan(self, states: bool = False) -> dict:
        """The scoring kernel a batch runs (`kernel`: k_fused, k_tile_fast, k_score_fast or k_score_general), its
        template switches and its tile geometry (vpt_predictor_kernel_plan); `states`: a batch that asks for
        pattern-id states."""
        pl = _KernelPlan()
        _check(lib().vpt_predictor_kernel_plan(self._h, int(states), C.byref(pl)))
        out = {k: getattr(pl, k) for k, _ in _KernelPlan._fields_}
        out["kernel"] = KERNEL_NAMES[pl.kernel]
        return out

    def export_blob(self) -> np.ndarray:
        n = lib().vpt_predictor_blob_size(self._h)
        out = np.empty(n, np.uint8)
        _check(lib().vpt_predictor_blob_export(self._h, out.ctypes.data, n))
        return out

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h and _lib is not None:  # (module globals are already gone when the interpreter shuts down)
            _lib.vpt_predictor_free(h)

    # -- predict ------------------------------------------------------------------------------------
    def predict(self, sentence: "Sentence") -> None:
        """`Predictor::predict(&self, &mut Sentence)` (predictor.rs:518-543)."""
        b = sentence._bytes
        n = sentence._n
        scores = np.zeros(max(n - 1, 1), np.int32)
        bounds = np.zeros(max(n - 1, 1), np.uint8)
        want = self.info["char_scorer"] == 2 or self.info["type_scorer"] == 3
        cs = np.full(n, 0xFFFFFFFF, np.uint32) if want else None
        ts = np.full(n, 0xFFFFFFFF, np.uint32) if want else None
        nch = C.c_uint64()
        _check(lib().vpt_predict(self._h, b, len(b), scores.ctypes.data, bounds.ctypes.data, max(n - 1, 1), _ptr(cs),
                                 _ptr(ts), n, C.byref(nch)))
        assert nch.value == n
        sentence._scores = scores[: n - 1]
        sentence._boundaries = bounds[: n - 1].copy()
        sentence._char_states = cs
        sentence._type_states = ts
        sentence._predictor = self
        sentence._tags = None
        sentence._tag_scores = None

    def predict_batch(self, text, offsets, want_scores: bool = True, want_states: bool = False,
                      out: Optional[BatchResult] = None) -> BatchResult:
        """Batched predict over host buffers (vpt_predict_batch).  text: uint8 array / bytes,
        offsets: uint64 [n+1].  Outputs are sized from the text length unless `out` supplies buffers."""
        t = np.frombuffer(text, np.uint8) if isinstance(text, (bytes, bytearray)) else np.ascontiguousarray(text, np.uint8)
        off = np.ascontiguousarray(offsets, np.uint64)
        n = off.size - 1
        nbytes = int(off[-1] - off[0]) if n > 0 else 0
        if out is None:
            cap = max(nbytes, 1)
            out = BatchResult(np.empty(cap, np.int32) if want_scores else None, np.empty(cap, np.uint8),
                              np.empty(n + 1, np.uint64), np.empty(max(n, 1), np.int32),
                              np.empty(cap, np.uint32) if want_states else None,
                              np.empty(cap, np.uint32) if want_states else None,
                              np.empty(n + 1, np.uint64))
        nb = C.c_uint64()
        nc = C.c_uint64()
        _check(lib().vpt_predict_batch(self._h, t.ctypes.data, off.ctypes.data, n, _ptr(out.scores),
                                       out.boundaries.ctypes.data, out.boundaries.size, out.bound_offsets.ctypes.data,
                                       _ptr(out.status), _ptr(out.char_states), _ptr(out.type_states),
                                       0 if out.char_states is None else out.char_states.size,
                                       _ptr(out.char_offsets), C.byref(nb), C.byref(nc)))
        res = BatchResult(None if out.scores is None else out.scores[: nb.value], out.boundaries[: nb.value],
                          out.bound_offsets, out.status[:n],
                          None if out.char_states is None else out.char_states[: nc.value],
                          None if out.type_states is None else out.type_states[: nc.value], out.char_offsets)
        res.n_boundaries = nb.value
        res.n_chars = nc.value
        return res

    def predict_batch_tags(self, text, offsets, want_scores: bool = True):
        """predict + predict_tags for a batch with tag prediction on the device (vpt_predict_batch_tags).  Returns
        (BatchResult, tag_token [chars] int32, tag_cand [chars, n_tags] int32, n_unserved): the arrays `fill_tags`
        computes per sentence, indexed by BatchResult.char_offsets."""
        t = np.frombuffer(text, np.uint8) if isinstance(text, (bytes, bytearray)) else np.ascontiguousarray(text, np.uint8)
        off = np.ascontiguousarray(offsets, np.uint64)
        n = off.size - 1
        cap = max(int(off[-1] - off[0]) if n > 0 else 0, 1)
        nt = max(self.n_tags, 1)
        scores = np.empty(cap, np.int32) if want_scores else None
        bounds = np.empty(cap, np.uint8)
        boff = np.empty(n + 1, np.uint64)
        coff = np.empty(n + 1, np.uint64)
        status = np.empty(max(n, 1), np.int32)
        tok = np.empty(cap, np.int32)
        cand = np.empty(cap * nt, np.int32)
        nb, nc, nu = C.c_uint64(), C.c_uint64(), C.c_uint64()
        _check(lib().vpt_predict_batch_tags(self._h, t.ctypes.data, off.ctypes.data, n, _ptr(scores), bounds.ctypes.data, cap,
                                            boff.ctypes.data, status.ctypes.data, tok.ctypes.data, cand.ctypes.data, cap,
                                            coff.ctypes.data, C.byref(nb), C.byref(nc), C.byref(nu)))
        res = BatchResult(None if scores is None else scores[: nb.value], bounds[: nb.value], boff, status[:n], None, None, coff)
        return res, tok[: nc.value], cand[: nc.value * nt].reshape(-1, nt), int(nu.value)

    def tag_string(self, token_id: int, slot: int, cand: int) -> Optional[str]:
        """Tag string of (token id, tag slot, candidate) as the token records of predict_batch_compact name it."""
        v = lib().vpt_tag_string(self._h, int(token_id), int(slot), int(cand))
        return None if v is None else v.decode("utf-8")

    def predict_batch_compact(self, text, offsets, tags: bool = False, tag_scores: bool = False) -> "CompactResult":
        """predict (+ predict_tags) for a batch with compact results (vpt_predict_batch_compact): one bit per boundary, one
        record per token; see CompactResult.  `tag_scores` (with tags): the tag candidate scores of every token record too
        (vpt_predict_batch_compact_tag_scores; CompactResult.tag_candidates)."""
        if tag_scores and not tags:
            raise VaporettoError(2, "InvalidArgumentError: tag_scores: needs tags=True")
        t = np.frombuffer(text, np.uint8) if isinstance(text, (bytes, bytearray)) else np.ascontiguousarray(text, np.uint8)
        off = np.ascontiguousarray(offsets, np.uint64)
        n = off.size - 1
        cap = max(int(off[-1] - off[0]) if n > 0 else 0, 1)
        nt = self.n_tags if tags else 0
        bits = np.zeros((cap + 31) // 32 + 1, np.uint32)
        n_chars = np.zeros(max(n, 1), np.uint32)
        status = np.zeros(max(n, 1), np.uint8)
        n_tokens = np.zeros(max(n, 1), np.uint32)
        tok = np.empty(cap, np.int32) if tags else None
        cand = np.empty(cap * max(nt, 1), np.uint8) if tags else None
        nb, ntok, nu = C.c_uint64(), C.c_uint64(), C.c_uint64()
        sc, nsc = self._score_buffer(cap) if tag_scores else None, C.c_uint64()
        _check(lib().vpt_predict_batch_compact_tag_scores(
            self._h, t.ctypes.data, off.ctypes.data, n, bits.ctypes.data, bits.size, n_chars.ctypes.data, status.ctypes.data,
            n_tokens.ctypes.data, _ptr(tok), _ptr(cand), cap if tags else 0, C.byref(nb), C.byref(ntok), C.byref(nu), _ptr(sc),
            0 if sc is None else sc.size, C.byref(nsc)))
        r = CompactResult(bits[: (nb.value + 31) // 32], int(nb.value), n_chars[:n], status[:n], n_tokens[:n],
                          None if tok is None else tok[: ntok.value],
                          None if cand is None else cand[: ntok.value * max(nt, 1)].reshape(-1, max(nt, 1)), int(nu.value))
        if tag_scores:
            _attach_scores(r, self, sc[: nsc.value])
        return r

    def _score_buffer(self, max_tokens: int) -> np.ndarray:
        """int32 buffer for the tag scores of at most `max_tokens` token records (each gets at most the longest vector)."""
        lens = self._score_lens()
        return np.empty(max(max_tokens * int(lens.max(initial=0)), 1), np.int32)

    def tokenize_lines(self, data, out: Optional[np.ndarray] = None, no_norm: bool = False, wsconst: str = "",
                       predict_tags: bool = False, tag_rules: Optional["PatternMatchTagger"] = None):
        """The reference CLI's `predict` loop (predict/src/main.rs:126-181) over a whole buffer of raw bytes
        (vpt_tokenize_lines): lines are split, scored (on KyteaFullwidthFilter(line) unless no_norm) and written
        out as space-separated tokens on the device; `wsconst`: letters of the CLI's --wsconst options ("D", "DR", ...:
        KyteaWsConstFilter; "G": ConcatGraphemeClustersFilter); `predict_tags`: the CLI's --predict-tags
        (vpt_tokenize_lines_tags); `tag_rules`: a PatternMatchTagger made for this predictor, run after the tag
        prediction (vpt_tokenize_lines_tags_rules; only with predict_tags).  Returns (uint8 view of the output lines,
        number of lines)."""
        mask = _wsconst_mask(wsconst)
        t = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else np.ascontiguousarray(data, np.uint8)
        if out is None:
            out = np.empty((3 + (16 if predict_tags else 0)) * t.size + int(np.count_nonzero(t == 10)) + 16, np.uint8)
        n = C.c_uint64()
        nl = C.c_uint64()
        fn = lib().vpt_tokenize_lines_tags if predict_tags else lib().vpt_tokenize_lines
        if tag_rules is not None and predict_tags:
            def fn(h, *args, _rules=tag_rules._handle()):
                return lib().vpt_tokenize_lines_tags_rules(h, _rules, *args)
        for _ in range(2):
            rc = fn(self._h, t.ctypes.data, t.size, int(no_norm), mask, out.ctypes.data, out.size, C.byref(n), C.byref(nl))
            if rc == 2 and predict_tags and n.value > out.size:
                out = np.empty(n.value + 16, np.uint8)   # long tag strings: the call reported the size it needs
                continue
            break
        _check(rc)
        return out[: n.value], int(nl.value)

    def tokenize_partial_lines(self, data, out: Optional[np.ndarray] = None, no_norm: bool = False, wsconst: str = "",
                               predict_tags: bool = False, tag_rules: Optional["PatternMatchTagger"] = None):
        """tokenize_lines for partially annotated lines (vpt_tokenize_partial_lines): every line is in the format of
        the reference's Sentence::from_partial_annotation ('|' boundary, '-' no boundary, ' ' unknown after every
        character but the last; tag fields after '/' are checked and dropped).  The model predicts the raw text, the
        `wsconst` post-filters run, then every '|' / '-' of the line overrides the boundary it marks; with
        `predict_tags` the tags (and `tag_rules`) follow.  An empty line gives an empty output line; a malformed line
        raises VaporettoError (InvalidArgument, or IOError for invalid UTF-8) naming the first such line.  Returns
        (uint8 view of the output lines, number of lines)."""
        mask = _wsconst_mask(wsconst)
        t = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else np.ascontiguousarray(data, np.uint8)
        if out is None:
            out = np.empty((3 + (16 if predict_tags else 0)) * t.size + int(np.count_nonzero(t == 10)) + 16, np.uint8)
        n = C.c_uint64()
        nl = C.c_uint64()
        rules = tag_rules._handle() if tag_rules is not None else None
        for _ in range(2):
            rc = lib().vpt_tokenize_partial_lines(self._h, rules, t.ctypes.data, t.size, int(no_norm), mask,
                                                  int(predict_tags), out.ctypes.data, out.size, C.byref(n), C.byref(nl))
            if rc == 2 and predict_tags and n.value > out.size:
                out = np.empty(n.value + 16, np.uint8)   # long tag strings: the call reported the size it needs
                continue
            break
        _check(rc)
        return out[: n.value], int(nl.value)

    def annotate_lines(self, data, margin: int = 0, no_norm: bool = False, wsconst: str = "", predict_tags: bool = False,
                       tag_rules: Optional["PatternMatchTagger"] = None, out: Optional[np.ndarray] = None):
        """tokenize_lines in the partial-annotation format (vpt_annotate_lines, the reference's
        Sentence::write_partial_annotation_text): '|' boundary, '-' no boundary, ' ' Unknown between every two
        characters.  A boundary whose score lies strictly between -margin and margin is left Unknown, unless a `wsconst`
        post-filter clears it; tokens next to an Unknown boundary get no tags (`predict_tags`, `tag_rules`).  Tags are
        written unescaped, as the reference writes them.  margin=0 leaves nothing Unknown.  A line the reference cannot
        read gives an empty line.  Returns (bytes of the output lines, number of lines)."""
        mask = _wsconst_mask(wsconst)
        t = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else np.ascontiguousarray(data, np.uint8)
        if out is None:
            out = np.empty((2 + (16 if predict_tags else 0)) * t.size + int(np.count_nonzero(t == 10)) + 16, np.uint8)
        n = C.c_uint64()
        nl = C.c_uint64()
        rules = tag_rules._handle() if tag_rules is not None else None
        for _ in range(2):
            rc = lib().vpt_annotate_lines(self._h, rules, t.ctypes.data, t.size, int(no_norm), mask, int(predict_tags),
                                          int(margin), out.ctypes.data, out.size, C.byref(n), C.byref(nl))
            if rc == 2 and n.value > out.size:
                out = np.empty(n.value + 16, np.uint8)   # long tag strings: the call reported the size it needs
                continue
            break
        _check(rc)
        return out[: n.value].tobytes(), int(nl.value)

    def reannotate_lines(self, data, margin: int = 0, keep_tags: bool = True, no_norm: bool = False, wsconst: str = "",
                         predict_tags: bool = False, tag_rules: Optional["PatternMatchTagger"] = None,
                         out: Optional[np.ndarray] = None):
        """Partially annotated lines in, partially annotated lines out (vpt_reannotate_lines): every line is read as
        tokenize_partial_lines reads it, and written as annotate_lines writes its lines.  The caller's '|' and '-' are
        written as given; a ' ' becomes '|' or '-' where the model is sure (its score lies outside (-margin, margin), or
        a `wsconst` post-filter decides it) and stays ' ' otherwise.  With `keep_tags`, every character whose tag fields
        are not all empty gets exactly its input tags back (unescaped), in place of the model's and the rules' tags;
        otherwise the input tags are dropped.  An empty line gives an empty output line; a malformed line raises
        tokenize_partial_lines' VaporettoError.  Returns (bytes of the output lines, number of lines)."""
        mask = _wsconst_mask(wsconst)
        t = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else np.ascontiguousarray(data, np.uint8)
        if out is None:
            out = np.empty((2 + (16 if predict_tags else 0)) * t.size + int(np.count_nonzero(t == 10)) + 16, np.uint8)
        n = C.c_uint64()
        nl = C.c_uint64()
        rules = tag_rules._handle() if tag_rules is not None else None
        for _ in range(2):
            rc = lib().vpt_reannotate_lines(self._h, rules, t.ctypes.data, t.size, int(no_norm), mask, int(predict_tags),
                                            int(margin), int(keep_tags), out.ctypes.data, out.size, C.byref(n),
                                            C.byref(nl))
            if rc == 2 and n.value > out.size:
                out = np.empty(n.value + 16, np.uint8)   # long tag strings: the call reported the size it needs
                continue
            break
        _check(rc)
        return out[: n.value].tobytes(), int(nl.value)

    def evaluate_lines(self, data, no_norm: bool = False, wsconst: str = "", predict_tags: bool = False,
                       per_line: bool = False):
        """The reference's `evaluate` command (evaluate/src/main.rs:69-195, vpt_evaluate_lines) over a buffer holding a
        gold corpus in the tokenized format: every non-empty line is parsed (Sentence::from_tokenized), predicted as
        tokenize_lines predicts it (same `no_norm`, `wsconst`, `predict_tags`) and compared with its gold boundaries
        and tags, all on the device.  Returns a dict of the counts (n_lines, n_sentences, tp, tn, fp, fn for
        --metric char; n_sys, n_ref, n_cor for --metric word) and, with `per_line`, also a uint32 array
        (n_lines, 7) of tp, tn, fp, fn, n_sys, n_ref, n_cor per input line.  A bad gold line raises VaporettoError
        (InvalidArgument, or IOError for invalid UTF-8) naming the first such line."""
        mask = _wsconst_mask(wsconst)
        t = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else np.ascontiguousarray(data, np.uint8)
        counts = _EvalCounts()
        lc = None
        if per_line:
            n_lines = int(np.count_nonzero(t == 10)) + (1 if t.size and t[-1] != 10 else 0)
            lc = np.zeros((n_lines, 7), np.uint32)
        _check(lib().vpt_evaluate_lines(self._h, t.ctypes.data, t.size, int(no_norm), mask, int(predict_tags),
                                        C.byref(counts), _ptr(lc), 0 if lc is None else lc.shape[0]))
        out = {name: int(getattr(counts, name)) for name, _ in _EvalCounts._fields_}
        return (out, lc) if per_line else out

    def token_spans(self, text, offsets, no_norm: bool = False, wsconst: str = "", tags: bool = False,
                    tag_scores: bool = False) -> "SpansResult":
        """vaporetto_tantivy's token_stream (lib.rs:157-229) for a batch of documents on the device (vpt_token_spans):
        document d is text[offsets[d]:offsets[d + 1]] (bytes or uint8 array, UTF-8); it is pre-filtered (unless
        `no_norm`), predicted, split on both sides of every '\r' / '\n' and post-filtered by the `wsconst` letters
        (D, R, H, T, K, O, G).  `tags`: the tag records of every token (needs predict_tags).  `tag_scores` (with tags):
        their tag candidate scores too (vpt_token_spans_tag_scores; SpansResult.tag_candidates).  See SpansResult."""
        if tag_scores and not tags:
            raise VaporettoError(2, "InvalidArgumentError: tag_scores: needs tags=True")
        mask = _wsconst_mask(wsconst)
        t = np.frombuffer(text, np.uint8) if isinstance(text, (bytes, bytearray)) else np.ascontiguousarray(text, np.uint8)
        off = np.ascontiguousarray(offsets, np.uint64)
        n = off.size - 1
        cap = max(int(off[-1] - off[0]) if n > 0 else 0, 1)  # a token has at least one byte
        nt = self.n_tags if tags else 0
        n_tokens = np.zeros(max(n, 1), np.uint32)
        status = np.zeros(max(n, 1), np.uint8)
        ends = np.empty(cap, np.uint32)
        tok = np.empty(cap, np.int32) if tags else None
        cand = np.empty(cap * max(nt, 1), np.uint8) if tags else None
        total = C.c_uint64()
        sc, nsc = self._score_buffer(cap) if tag_scores else None, C.c_uint64()
        _check(lib().vpt_token_spans_tag_scores(self._h, t.ctypes.data, off.ctypes.data, max(n, 0), int(no_norm), mask,
                                                n_tokens.ctypes.data, status.ctypes.data, ends.ctypes.data, _ptr(tok),
                                                _ptr(cand), cap, C.byref(total), _ptr(sc), 0 if sc is None else sc.size,
                                                C.byref(nsc)))
        k = int(total.value)
        r = SpansResult(n_tokens[:max(n, 0)], status[:max(n, 0)], ends[:k], None if tok is None else tok[:k],
                        None if cand is None else cand[: k * max(nt, 1)].reshape(-1, max(nt, 1))[:, :nt])
        if tag_scores:
            _attach_scores(r, self, sc[: nsc.value])
        return r

    def token_spans_device(self, text, offsets, no_norm: bool = False, wsconst: str = "", tags: bool = False,
                           stream=None) -> "DeviceSpans":
        """token_spans for documents already in GPU memory (vpt_token_spans_dev): `text` is a 1-D torch.uint8 CUDA
        tensor (any view of a larger buffer), `offsets` its n_docs + 1 int32 or int64 Arrow-style offsets on the same
        device; document d is text[offsets[d]:offsets[d + 1]].  A cuDF / Arrow string column or a CuPy array comes in
        without a copy through torch.as_tensor (the column's chars and offsets buffers).  The call is queued on `stream`
        (default: torch.cuda.current_stream()), its workspace and outputs come from torch's caching allocator on that
        stream, and it neither synchronises nor reads anything back: it is stream-ordered and can be captured in a CUDA
        graph.  A document whose offsets are not a range inside the text has status 4 (VPT_SENT_BAD_RANGE) and no
        tokens.  See DeviceSpans; DeviceSpans.to_host() gives what token_spans returns."""
        import torch
        if not isinstance(text, torch.Tensor) or text.dtype != torch.uint8 or text.dim() != 1 or not text.is_cuda:
            raise VaporettoError(2, "InvalidArgumentError: text: must be a 1-D torch.uint8 CUDA tensor")
        if (not isinstance(offsets, torch.Tensor) or offsets.dtype not in (torch.int32, torch.int64) or offsets.dim() != 1
                or offsets.numel() < 1):
            raise VaporettoError(2, "InvalidArgumentError: offsets: must be a 1-D int32 or int64 tensor of n_docs + 1")
        if text.device != offsets.device or text.device.index != self.info["device"]:
            raise VaporettoError(2, f"InvalidArgumentError: text/offsets: must be on the predictor's device "
                                    f"cuda:{self.info['device']}")
        mask = _wsconst_mask(wsconst)
        dev = text.device
        st = torch.cuda.current_stream(dev) if stream is None else stream
        n, nb = offsets.numel() - 1, text.numel()
        nt = self.n_tags if tags else 0
        L = lib()
        with torch.cuda.stream(st):
            text, offsets = text.contiguous(), offsets.contiguous()
            ws_bytes = L.vpt_token_spans_dev_workspace_size(self._h, n, nb, int(tags))
            ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
            tok_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
            n_tokens = torch.empty(max(n, 1), dtype=torch.int32, device=dev)[:n]  # (an empty tensor has no pointer)
            status = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)[:n]
            ends = torch.empty(max(nb, 1), dtype=torch.int32, device=dev)  # a token has at least one byte
            ids = torch.empty(max(nb, 1), dtype=torch.int32, device=dev) if tags else None
            cands = torch.empty((max(nb, 1), nt), dtype=torch.uint8, device=dev) if tags else None
            dp = lambda t: None if t is None else t.data_ptr()
            _check(L.vpt_token_spans_dev(self._h, dp(text) if nb else None, nb, dp(offsets), offsets.element_size(), n,
                                         int(no_norm), mask, dp(tok_off), dp(n_tokens), dp(status), dp(ends), dp(ids),
                                         dp(cands) if nt else None, dp(ws), ws_bytes, st.cuda_stream))
        return DeviceSpans(tok_off, n_tokens, status, ends, ids, cands, st, ws)

    def tokenize_device(self, text, offsets, no_norm: bool = False, wsconst: str = "", predict_tags: bool = False,
                        tag_rules: Optional["PatternMatchTagger"] = None, out_capacity: Optional[int] = None,
                        stream=None) -> "DeviceText":
        """The tokenized text of documents already in GPU memory (vpt_tokenize_dev), as a device string column: one
        string per document, what tokenize_lines writes for it as one line without the '\n' ('\r' and '\n' inside a
        document are ordinary characters).  `text` and `offsets` are as in token_spans_device; `wsconst`, `predict_tags`
        and `tag_rules` as in tokenize_lines (tag_rules needs predict_tags).  `out_capacity`: bytes of the output buffer
        (None: vpt_tokenize_dev_out_bound, with which every document is written; 0: offsets only).  The call is queued
        on `stream` (default: torch.cuda.current_stream()), its workspace and outputs come from torch's caching
        allocator on that stream, and it neither synchronises nor reads anything back: it is stream-ordered and can be
        captured in a CUDA graph.  A rejected document has a non-zero status (4: offsets out of range) and an empty
        string.  See DeviceText."""
        import torch
        if not isinstance(text, torch.Tensor) or text.dtype != torch.uint8 or text.dim() != 1 or not text.is_cuda:
            raise VaporettoError(2, "InvalidArgumentError: text: must be a 1-D torch.uint8 CUDA tensor")
        if (not isinstance(offsets, torch.Tensor) or offsets.dtype not in (torch.int32, torch.int64) or offsets.dim() != 1
                or offsets.numel() < 1):
            raise VaporettoError(2, "InvalidArgumentError: offsets: must be a 1-D int32 or int64 tensor of n_docs + 1")
        if text.device != offsets.device or text.device.index != self.info["device"]:
            raise VaporettoError(2, f"InvalidArgumentError: text/offsets: must be on the predictor's device "
                                    f"cuda:{self.info['device']}")
        if out_capacity is not None and int(out_capacity) < 0:
            raise VaporettoError(2, "InvalidArgumentError: out_capacity: must not be negative")
        mask = _wsconst_mask(wsconst)
        dev = text.device
        st = torch.cuda.current_stream(dev) if stream is None else stream
        n, nb = offsets.numel() - 1, text.numel()
        rules = None if tag_rules is None else tag_rules._handle()
        L = lib()
        cap = L.vpt_tokenize_dev_out_bound(self._h, rules, n, nb, int(predict_tags)) if out_capacity is None \
            else int(out_capacity)
        with torch.cuda.stream(st):
            text, offsets = text.contiguous(), offsets.contiguous()
            ws_bytes = L.vpt_tokenize_dev_workspace_size(self._h, rules, n, nb, int(predict_tags))
            ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
            out_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
            chars = torch.empty(cap, dtype=torch.uint8, device=dev)
            status = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)[:n]  # (an empty tensor has no pointer)
            _check(L.vpt_tokenize_dev(self._h, rules, text.data_ptr() if nb else None, nb, offsets.data_ptr(),
                                      offsets.element_size(), n, int(no_norm), mask, int(predict_tags), out_off.data_ptr(),
                                      chars.data_ptr() if cap else None, cap, status.data_ptr(), ws.data_ptr(), ws_bytes,
                                      st.cuda_stream))
            complete = out_off[-1] <= cap
        return DeviceText(out_off, chars, status, complete, st, (ws, text, offsets, tag_rules))

    def line_stream(self, kind: str = "tokenize", no_norm: bool = False, wsconst: str = "",
                    predict_tags: bool = False, tag_rules: Optional["PatternMatchTagger"] = None,
                    scores: bool = False, tag_scores: bool = False, margin: int = 0,
                    keep_tags: bool = True) -> "LineStream":
        """tokenize_lines (kind="tokenize"), evaluate_lines (kind="evaluate"), tokenize_partial_lines
        (kind="partial"), annotate_lines (kind="annotate", with `margin`) or reannotate_lines (kind="reannotate",
        with `margin` and `keep_tags`) on input fed in pieces of any size,
        with host memory bounded by the pipeline, not by the input (vpt_line_stream_*): see LineStream.  `tag_rules`
        as in tokenize_lines.  `scores` / `tag_scores` (tokenize only; `tag_scores` needs predict_tags and a model with
        tag slots) add the predict CLI's --scores / --tag-scores dumps behind every token line
        (vpt_line_stream_new_scores)."""
        return LineStream(self, kind, no_norm, wsconst, predict_tags, tag_rules, scores, tag_scores, margin, keep_tags)


class LineStream:
    """A line stream (vpt_line_stream_new): the loop of tokenize_lines or evaluate_lines over input fed in pieces, split
    at any byte.  feed(data) and flush() return the output delivered during the call (bytes; b"" for evaluate);
    finish() returns (the rest of the output, number of lines) for tokenize and the dict of evaluate_lines for
    evaluate.  The concatenated output equals the whole-buffer call's on the concatenated input.  flush() delivers the
    output of every complete line fed so far.  After an error every call raises it again.  Use as a context manager, or
    call close()."""

    def __init__(self, predictor: "Predictor", kind: str, no_norm: bool, wsconst: str, predict_tags: bool,
                 tag_rules: Optional["PatternMatchTagger"] = None, scores: bool = False, tag_scores: bool = False,
                 margin: int = 0, keep_tags: bool = True):
        if kind not in STREAM_KINDS and kind not in ("partial", "annotate", "reannotate"):
            raise VaporettoError(2, "InvalidArgumentError: kind: 'tokenize', 'evaluate', 'partial', 'annotate' or "
                                    "'reannotate'")
        dumps = (DUMP_SCORES if scores else 0) | (DUMP_TAG_SCORES if tag_scores else 0)
        if dumps and kind != "tokenize":
            raise VaporettoError(2, "InvalidArgumentError: scores, tag_scores: kind='tokenize' only")
        mask = _wsconst_mask(wsconst)
        self._predictor = predictor  # (the stream uses the predictor until it is closed)
        self._tag_rules = tag_rules  # (and the rules)
        self._kind = kind
        self._parts: List[bytes] = []
        self._exc: Optional[BaseException] = None
        self._write = STREAM_WRITE_FN(self._sink)  # (kept alive as long as the stream)
        h = _P()
        rules = tag_rules._handle() if tag_rules is not None else None
        if kind == "partial":
            _check(lib().vpt_line_stream_new_partial(predictor._h, rules, int(no_norm), mask, int(predict_tags),
                                                     C.cast(self._write, _P), None, C.byref(h)))
        elif kind == "annotate":
            _check(lib().vpt_line_stream_new_annotate(predictor._h, rules, int(no_norm), mask, int(predict_tags),
                                                      int(margin), C.cast(self._write, _P), None, C.byref(h)))
        elif kind == "reannotate":
            _check(lib().vpt_line_stream_new_reannotate(predictor._h, rules, int(no_norm), mask, int(predict_tags),
                                                        int(margin), int(keep_tags), C.cast(self._write, _P), None,
                                                        C.byref(h)))
        elif dumps:
            _check(lib().vpt_line_stream_new_scores(predictor._h, rules, int(no_norm), mask, int(predict_tags), dumps,
                                                    C.cast(self._write, _P), None, C.byref(h)))
        else:
            _check(lib().vpt_line_stream_new_rules(predictor._h, rules, STREAM_KINDS[kind], int(no_norm), mask,
                                                   int(predict_tags), C.cast(self._write, _P), None, C.byref(h)))
        self._h = h

    def _sink(self, ctx, data, n):
        try:
            self._parts.append(C.string_at(data, n))
            return 0
        except BaseException as e:  # re-raised by the call that delivered the output
            self._exc = e
            return 1

    def _run(self, fn, *args) -> bytes:
        if self._h is None:
            raise VaporettoError(2, "InvalidArgumentError: stream: closed")
        try:
            rc = fn(self._h, *args)
            if self._exc is not None:
                raise self._exc
            _check(rc)
            return b"".join(self._parts)
        finally:
            self._parts.clear()
            self._exc = None

    def feed(self, data) -> bytes:
        t = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else np.ascontiguousarray(data, np.uint8)
        return self._run(lib().vpt_line_stream_feed, t.ctypes.data, t.size)

    def flush(self) -> bytes:
        return self._run(lib().vpt_line_stream_flush)

    def finish(self):
        n = C.c_uint64()
        counts = _EvalCounts()
        out = self._run(lib().vpt_line_stream_finish, C.byref(n), C.byref(counts))
        if self._kind == "evaluate":
            return {name: int(getattr(counts, name)) for name, _ in _EvalCounts._fields_}
        return out, int(n.value)

    def close(self) -> None:
        h, self._h = getattr(self, "_h", None), None
        if h and _lib is not None:  # (module globals are already gone when the interpreter shuts down)
            _lib.vpt_line_stream_free(h)

    def __enter__(self) -> "LineStream":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def __del__(self):
        self.close()


class PatternMatchTagger:
    """`vaporetto_rules::sentence_filters::PatternMatchTagger::new(rules)` (pattern_match_tagger.rs:21-41) for the tagged
    line path (vpt_tag_rules_new): `rules` maps a token surface to its tags, one entry per tag slot, None for a slot the
    rule leaves alone.  Passed as `tag_rules=` to Predictor.tokenize_lines / line_stream with predict_tags, it fills
    every tag slot the model left None for a token whose surface is a key; predicted tags are never overwritten.  Unless
    no_norm, tokens are matched by their KyteaFullwidthFilter image and keys are not normalised: write full-width keys
    ("ＡＢＣ") for the default, half-width ones match only with no_norm.  Bound to `predictor` (its device and n_tags)."""

    def __init__(self, predictor: "Predictor", rules: dict):
        surf, soff, qoff, slots, tags = bytearray(), [0], [0], [], bytearray()
        for key, vals in rules.items():
            surf += key.encode("utf-8")
            soff.append(len(surf))
            for v in vals:
                if v is None:
                    slots += [0xFFFFFFFF, 0]
                else:
                    b = v.encode("utf-8")
                    slots += [len(tags), len(b)]
                    tags += b
            qoff.append(len(slots) // 2)
        a = (np.frombuffer(bytes(surf) or b"\0", np.uint8), np.array(soff, np.uint64), np.array(qoff, np.uint64),
             np.array(slots or [0], np.uint32), np.frombuffer(bytes(tags) or b"\0", np.uint8))  # (copied by the call)
        self._predictor = predictor  # (the rules are bound to the predictor and must not outlive it)
        self._h = None
        h = _P()
        _check(lib().vpt_tag_rules_new(predictor._h, len(rules), a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data,
                                       a[3].ctypes.data, a[4].ctypes.data, len(tags), C.byref(h)))
        self._h = h

    def _handle(self):
        if self._h is None:
            raise VaporettoError(2, "InvalidArgumentError: rules: closed")
        return self._h

    def max_output(self) -> int:
        """The largest device output buffer a chunk of a call with these rules has used (vpt_tag_rules_max_output)."""
        return int(lib().vpt_tag_rules_max_output(self._h)) if self._h else 0

    def close(self) -> None:
        h, self._h = getattr(self, "_h", None), None
        if h and _lib is not None:
            _lib.vpt_tag_rules_free(h)

    def __del__(self):
        self.close()


class _EvalCounts(C.Structure):
    _fields_ = [(name, C.c_uint64) for name in ("n_lines", "n_sentences", "tp", "tn", "fp", "fn", "n_sys", "n_ref",
                                                "n_cor")]


def _wsconst_mask(wsconst: str) -> int:
    """The CLI's --wsconst letters as the C ABI's bit set (VPT_WSCONST_*)."""
    mask = 0
    for ch in wsconst:
        if ch not in "DRHTKOG":
            raise VaporettoError(2, "InvalidArgumentError: wsconst: one of D, R, H, T, K, O, G")
        mask |= 1 << ("DRHTKOG".index(ch) + 1)
    return mask


def _tag_candidates(p: "Predictor", token_id: int, scores) -> list:
    """Token::tag_candidates (sentence.rs:1219-1250) over the predictor's tag strings."""
    if token_id < 0:
        return []
    L = lib()
    out, i = [], 0
    for k in range(L.vpt_tag_n_slots(p._h, token_id)):
        nc = L.vpt_tag_n_candidates(p._h, token_id, k)
        tag = lambda c: L.vpt_tag_string(p._h, token_id, k, c).decode("utf-8")
        if nc == 1:
            out.append([(tag(0), 0)])
        else:
            out.append([(tag(c), int(scores[i + c])) for c in range(nc)])
            i += nc
    return out


def _attach_scores(r, p: "Predictor", scores: np.ndarray) -> None:
    """tag_scores, score_offsets and the predictor behind tag_candidates of a CompactResult / SpansResult."""
    ids = r.token_ids
    lens = np.append(p._score_lens(), 0)[ids]  # (id -1: the appended 0)
    r.tag_scores = scores
    r.score_offsets = np.concatenate(([0], np.cumsum(lens))).astype(np.uint64)
    r._predictor = p


class _ScoredRecords:
    """tag_candidates of the token records of a result with tag scores."""
    tag_scores = None       # int32: the score vectors of the records with a token id >= 0, in record order
    score_offsets = None    # uint64 [tokens + 1]: record r's vector is tag_scores[score_offsets[r]:score_offsets[r + 1]]

    def tag_candidates(self, r: int) -> list:
        """`Token::tag_candidates` of token record r: [[(tag, score), ...] per tag slot]; a one-candidate slot gives
        (tag, 0), an empty slot [], a record with id -1 []."""
        if self.tag_scores is None:
            raise VaporettoError(2, "InvalidArgumentError: tag_candidates: the call was made without tag_scores=True")
        lo, hi = int(self.score_offsets[r]), int(self.score_offsets[r + 1])
        return _tag_candidates(self._predictor, int(self.token_ids[r]), self.tag_scores[lo:hi])


class CompactResult(_ScoredRecords):
    """Result of Predictor.predict_batch_compact: `boundary_bits` (uint32 words of the batch's boundary bit stream),
    `n_chars` / `status` / `n_tokens` per sentence, `token_ids` [tokens] and `token_cands` [tokens, n_tags] (uint8, 255 =
    none) when tags were requested.  Sentence s owns the bits [bit_offsets[s], bit_offsets[s + 1]) and the token records
    [token_offsets[s], token_offsets[s + 1])."""

    def __init__(self, bits, n_boundaries, n_chars, status, n_tokens, token_ids, token_cands, n_unserved):
        self.boundary_bits, self.n_boundaries = bits, n_boundaries
        self.n_chars, self.status, self.n_tokens = n_chars, status, n_tokens
        self.token_ids, self.token_cands, self.n_unserved = token_ids, token_cands, n_unserved
        nb = np.where(n_chars > 0, n_chars.astype(np.int64) - 1, 0)
        self.bit_offsets = np.concatenate(([0], np.cumsum(nb))).astype(np.uint64)
        self.token_offsets = np.concatenate(([0], np.cumsum(n_tokens.astype(np.int64)))).astype(np.uint64)

    def boundaries(self, s: Optional[int] = None) -> np.ndarray:
        """Boundaries as bytes (0 / 1): of sentence `s`, or of the whole batch (vpt_unpack_boundaries)."""
        lo, hi = (0, self.n_boundaries) if s is None else (int(self.bit_offsets[s]), int(self.bit_offsets[s + 1]))
        out = np.empty(hi - lo, np.uint8)
        _check(lib().vpt_unpack_boundaries(self.boundary_bits.ctypes.data, lo, hi - lo, out.ctypes.data))
        return out


class SpansResult(_ScoredRecords):
    """Result of Predictor.token_spans: `n_tokens` and `status` (VPT_SENT_*: 0 ok, 1 empty, 2 NUL, 3 invalid UTF-8) per
    document, `token_base` (n_docs + 1, uint64) the first token record of every document, `token_ends` (uint32) the byte
    offset of every token's exclusive end from its document's start, and with tags `token_ids` (int32, -1: no tag model)
    and `token_cands` (uint8 [tokens, n_tags], 255: none)."""

    def __init__(self, n_tokens, status, token_ends, token_ids, token_cands):
        self.n_tokens, self.status, self.token_ends = n_tokens, status, token_ends
        self.token_ids, self.token_cands = token_ids, token_cands
        self.token_base = np.concatenate(([0], np.cumsum(n_tokens.astype(np.uint64)))).astype(np.uint64)

    def spans(self, d: int) -> np.ndarray:
        """[from, to) byte offsets of the tokens of document d, as a (k, 2) uint32 array."""
        ends = self.token_ends[int(self.token_base[d]): int(self.token_base[d + 1])]
        out = np.empty((ends.size, 2), np.uint32)
        out[:, 1] = ends
        out[:1, 0] = 0
        out[1:, 0] = ends[:-1]
        return out


class DeviceSpans:
    """Result of Predictor.token_spans_device, torch tensors on the device, valid once the call's stream reaches them:
    `token_offsets` (int64, n_docs + 1: the first token record of every document, the total last), `n_tokens` (int32) and
    `status` (uint8, VPT_SENT_*; 4 = offsets out of range) per document, `token_ends` (int32, sized by the text's bytes:
    its first token_offsets[-1] entries are the token ends), and with tags `token_ids` (int32) and `token_cands` (uint8
    [bytes, n_tags]), sized like token_ends."""

    def __init__(self, token_offsets, n_tokens, status, token_ends, token_ids, token_cands, stream, workspace):
        self.token_offsets, self.n_tokens, self.status = token_offsets, n_tokens, status
        self.token_ends, self.token_ids, self.token_cands = token_ends, token_ids, token_cands
        self.stream = stream
        self._workspace = workspace  # (kept with the outputs: the queued kernels use it)

    def to_host(self) -> "SpansResult":
        """Synchronises the stream and returns the SpansResult token_spans gives for the same documents."""
        self.stream.synchronize()
        k = int(self.token_offsets[-1].item())
        host = lambda t, dt: t.cpu().numpy().view(dt)
        return SpansResult(host(self.n_tokens, np.uint32), host(self.status, np.uint8),
                           host(self.token_ends[:k], np.uint32),
                           None if self.token_ids is None else host(self.token_ids[:k], np.int32),
                           None if self.token_cands is None else host(self.token_cands[:k], np.uint8))


class DeviceText:
    """Result of Predictor.tokenize_device, torch tensors on the device, valid once the call's stream reaches them: a
    string column with `offsets` (int64, n_docs + 1: document d's string is chars[offsets[d]:offsets[d + 1]], the total
    last), `chars` (uint8, the output capacity), `status` (uint8 per document, VPT_SENT_*; 4 = offsets out of range) and
    `complete`, a 0-d bool tensor: whether every document was written (offsets[-1] <= capacity).  A document is written
    in full or not at all; with complete False the offsets are still exact, so they size a second call."""

    def __init__(self, offsets, chars, status, complete, stream, keep):
        self.offsets, self.chars, self.status, self.complete = offsets, chars, status, complete
        self.stream = stream
        self._keep = keep  # (the workspace and the inputs stay alive with the outputs: the queued kernels use them)

    def to_host(self):
        """Synchronises the stream and returns (chars[:total] as a numpy uint8 array, offsets as int64, status as
        uint8); raises VaporettoError when the output is incomplete."""
        self.stream.synchronize()
        off = self.offsets.cpu().numpy()
        total = int(off[-1])
        if total > self.chars.numel():
            raise VaporettoError(2, f"InvalidArgumentError: out_capacity: {self.chars.numel()} bytes, the tokenized text "
                                    f"needs {total}")
        return self.chars[:total].cpu().numpy(), off, self.status.cpu().numpy()

    def strings(self) -> List[str]:
        """Every document's tokenized text (to_host, decoded)."""
        chars, off, _ = self.to_host()
        b = chars.tobytes()
        return [b[off[d]:off[d + 1]].decode() for d in range(off.size - 1)]


class SpanToken:
    """`tantivy::tokenizer::Token` as vaporetto_tantivy's token stream fills it (lib.rs:207-219): the token's text, its
    byte offsets [offset_from, offset_to) in the document, its position, and position_length = the document's number of
    tokens."""
    __slots__ = ("text", "offset_from", "offset_to", "position", "position_length")

    def __init__(self, text: str, offset_from: int, offset_to: int, position: int, position_length: int):
        self.text, self.offset_from, self.offset_to = text, offset_from, offset_to
        self.position, self.position_length = position, position_length

    def _key(self):
        return (self.text, self.offset_from, self.offset_to, self.position, self.position_length)

    def __eq__(self, other):
        return isinstance(other, SpanToken) and self._key() == other._key()

    def __repr__(self):
        return "SpanToken(text=%r, offset_from=%d, offset_to=%d, position=%d, position_length=%d)" % self._key()


_SENT_MESSAGES = {1: "InvalidArgumentError: text: must contain at least one character",
                  2: "InvalidArgumentError: text: must not contain NULL",
                  3: "InvalidArgumentError: text: must be valid UTF-8"}


class Tokenizer:
    """`vaporetto_tantivy::VaporettoTokenizer` (lib.rs:54-155) over a device predictor: the full-width pre-filter,
    predict, SplitLinebreaksFilter and the `wsconst` post-filters (letters D, R, H, T, K, O, G; another letter raises
    "Could not parse a wsconst value", lib.rs:69-85).  token_stream(text) returns the adapter's tokens; token_streams(texts)
    those of many documents from one device call (Predictor.token_spans)."""

    def __init__(self, predictor: "Predictor", wsconst: str = ""):
        if any(ch not in "DRHTKOG" for ch in wsconst):
            raise VaporettoError(2, "Could not parse a wsconst value")
        self.predictor, self.wsconst = predictor, wsconst

    def token_stream(self, text: str) -> List[SpanToken]:
        return self.token_streams([text])[0]

    def token_streams(self, texts: Sequence[str]) -> List[List[SpanToken]]:
        enc = [t.encode("utf-8") for t in texts]
        off = np.zeros(len(enc) + 1, np.uint64)
        np.cumsum([len(e) for e in enc], out=off[1:])
        r = self.predictor.token_spans(b"".join(enc), off, wsconst=self.wsconst)
        out = []
        for d, e in enumerate(enc):
            st = int(r.status[d])
            if st >= 2:  # (the adapter panics on NUL; a str cannot hold invalid UTF-8)
                raise VaporettoError(2, f"{_SENT_MESSAGES[st]} (document {d})")
            sp = r.spans(d).tolist()
            out.append([SpanToken(e[a:b].decode("utf-8"), a, b, k, len(sp)) for k, (a, b) in enumerate(sp)])
        return out


class Token:
    """`vaporetto::Token` (sentence.rs:1195-1258)."""

    def __init__(self, sentence: "Sentence", start: int, end: int):
        self._s, self._start, self._end = sentence, start, end

    def surface(self) -> str:
        p = self._s._pos
        return self._s._bytes[p[self._start]:p[self._end]].decode("utf-8")

    def start(self) -> int:
        return self._start

    def end(self) -> int:
        return self._end

    def tags(self) -> List[Optional[str]]:
        k = self._s.n_tags()
        return self._s.tags()[(self._end - 1) * k:self._end * k]

    def tag_candidates(self):
        """`Token::tag_candidates` (sentence.rs:1219-1250): [[(tag, score), ...] per tag slot of the token's model]; []
        for a token without a tag model.  Needs Predictor.store_tag_scores(True) before fill_tags (the reference
        panics without it)."""
        s = self._s
        if s._tag_scores is None:
            raise RuntimeError("Predictor::store_tag_scores() must be set to true to use this function.")
        i = self._end - 1
        return _tag_candidates(s._predictor, int(s._tag_token[i]), s._tag_scores[i])


class Sentence:
    """`vaporetto::Sentence` (sentence.rs:85-1193), raw-text subset used around `predict`."""

    def __init__(self, text: str):
        self._set(text)

    @classmethod
    def from_raw(cls, text: str) -> "Sentence":
        """`Sentence::from_raw` (sentence.rs:217-247)."""
        return cls(text)

    def update_raw(self, text: str) -> None:
        """`Sentence::update_raw` (sentence.rs:264-283); on error the sentence becomes " "."""
        try:
            self._set(text)
        except VaporettoError:
            self._set(" ")
            raise

    def _set(self, text: str):
        b = text.encode("utf-8") if isinstance(text, str) else bytes(text)
        types = np.zeros(max(len(b), 1), np.uint8)
        n = C.c_uint64()
        _check(lib().vpt_char_types(b, len(b), types.ctypes.data, types.size, C.byref(n)))
        self._bytes = b
        self._n = n.value
        self._types = types[: self._n].copy()
        starts = [i for i, c in enumerate(b) if (c & 0xC0) != 0x80]
        self._pos = starts + [len(b)]
        self._boundaries = np.full(self._n - 1, CharacterBoundary.Unknown, np.uint8)
        self._scores = np.zeros(0, np.int32)
        self._char_states = None
        self._type_states = None
        self._predictor = None
        self._tags = None
        self._tag_token = None
        self._tag_cand = None
        self._tag_scores = None

    def as_raw_text(self) -> str:
        return self._bytes.decode("utf-8")

    def char_types(self) -> np.ndarray:
        return self._types

    def boundaries(self) -> np.ndarray:
        return self._boundaries

    def boundaries_mut(self) -> np.ndarray:
        return self._boundaries

    def split_linebreaks(self) -> None:
        """`SplitLinebreaksFilter::filter(&mut sentence)` (vaporetto_rules, split_linebreaks.rs:9-37)."""
        b = self.as_raw_text().encode("utf-8")
        bd = np.ascontiguousarray(self._boundaries, np.uint8)
        _check(lib().vpt_split_linebreaks(b, len(b), bd.ctypes.data, bd.size))
        self._boundaries[:] = bd

    def concat_grapheme_clusters(self) -> None:
        """`ConcatGraphemeClustersFilter::filter(&mut sentence)` (vaporetto_rules, concat_grapheme_clusters.rs:10-35)."""
        b = self.as_raw_text().encode("utf-8")
        bd = np.ascontiguousarray(self._boundaries, np.uint8)
        _check(lib().vpt_concat_grapheme_clusters(b, len(b), bd.ctypes.data, bd.size))
        self._boundaries[:] = bd

    def boundary_scores(self) -> np.ndarray:
        """`Sentence::boundary_scores` (sentence.rs:1040-1046)."""
        return self._scores

    def n_tags(self) -> int:
        return 0 if self._tags is None else self._predictor.n_tags

    def fill_tags(self) -> None:
        """`Sentence::fill_tags` (sentence.rs:1144-1148) -> `Predictor::predict_tags` (predictor.rs:546-637)."""
        p = self._predictor
        if p is None:
            return
        k = p.n_tags
        tt = np.full(self._n, -1, np.int32)
        tc = np.full(max(self._n * k, 1), -1, np.int32)
        ts = None
        if p._store_tag_scores:
            stride = max(int(p._score_lens().max(initial=0)), 1)
            ts = np.zeros((self._n, stride), np.int32)
        _check(lib().vpt_fill_tags(p._h, self._bytes, len(self._bytes), self._boundaries.ctypes.data,
                                   _ptr(self._char_states), _ptr(self._type_states), tt.ctypes.data, tc.ctypes.data,
                                   _ptr(ts), 0 if ts is None else ts.shape[1]))
        self._tag_token, self._tag_cand = tt, tc
        self._tag_scores = None if ts is None else [ts[i, : p._score_lens()[t]] if t >= 0 else ts[i, :0] for i, t in enumerate(tt)]
        tags: List[Optional[str]] = []
        for i in range(self._n):
            for s in range(k):
                c = tc[i * k + s]
                if tt[i] < 0 or c < 0:
                    tags.append(None)
                else:
                    tags.append(lib().vpt_tag_string(p._h, int(tt[i]), s, int(c)).decode("utf-8"))
        self._tags = tags

    def tags(self) -> List[Optional[str]]:
        return [] if self._tags is None else self._tags

    def iter_tokens(self):
        """`Sentence::iter_tokens` (sentence.rs:819; TokenIterator :1273-1299)."""
        start, skip = 0, False
        for i, b in enumerate(self._boundaries):
            if b == CharacterBoundary.WordBoundary:
                if not skip:
                    yield Token(self, start, i + 1)
                skip = False
                start = i + 1
            elif b == CharacterBoundary.Unknown:
                skip = True
        if not skip:
            yield Token(self, start, self._n)

    def write_tokenized_text(self) -> str:
        """`Sentence::write_tokenized_text` (sentence.rs:850-886)."""
        p = self._predictor
        cap = 2 * len(self._bytes) + 64
        ln = C.c_uint64()
        have = self._tags is not None
        for _ in range(2):
            # the call reports the full length even when it truncated: retry once with the exact size
            buf = C.create_string_buffer(cap)
            _check(lib().vpt_write_tokenized_text(p._h if p else None, self._bytes, len(self._bytes),
                                                  self._boundaries.ctypes.data,
                                                  self._tag_token.ctypes.data if have else None,
                                                  self._tag_cand.ctypes.data if have else None, buf, cap, C.byref(ln)))
            if ln.value < cap:
                break
            cap = ln.value + 1
        if ln.value >= cap:
            raise VaporettoError(18, "write_tokenized_text: length changed between calls")
        return buf.raw[: ln.value].decode("utf-8")

    def write_partial_annotation_text(self) -> str:
        """`Sentence::write_partial_annotation_text` (sentence.rs:907-944): tags unescaped."""
        p = self._predictor
        cap = 2 * len(self._bytes) + 64
        ln = C.c_uint64()
        have = self._tags is not None
        bd = np.ascontiguousarray(self._boundaries, np.uint8)
        for _ in range(2):
            buf = C.create_string_buffer(cap)
            _check(lib().vpt_write_partial_annotation_text(p._h if p else None, self._bytes, len(self._bytes),
                                                           bd.ctypes.data, self._tag_token.ctypes.data if have else None,
                                                           self._tag_cand.ctypes.data if have else None, buf, cap,
                                                           C.byref(ln)))
            if ln.value < cap:
                break
            cap = ln.value + 1
        if ln.value >= cap:
            raise VaporettoError(18, "write_partial_annotation_text: length changed between calls")
        return buf.raw[: ln.value].decode("utf-8")
