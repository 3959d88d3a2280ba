// Per-offset arithmetic of the document offset kernels (doc_offsets.cu): the caller's int32 or int64 Arrow-style offsets
// of vpt_token_spans_dev become the u64 offsets the scoring and span kernels read.  Compiled for the device by
// doc_offsets.cu and for the host by tests/native/doc_offsets_test.cpp, which runs it over small offset arrays against a
// Python restatement (tests/test_doc_offsets_cpu.py).
//
//   rebased offset i = shift + max(key(o[0]), ..., key(o[i])),   key(o) = o inside [0, n_bytes], else 0
//
// shift is d_utf8's address mod 16: the kernels read the text from d_utf8 rounded down to 16 bytes, so every 16-byte
// block they touch holds a byte of [d_utf8, d_utf8 + n_bytes).  The prefix maximum keeps the offsets non-decreasing and
// inside [shift, shift + n_bytes] whatever the caller passed, so no kernel reads outside the batch; an offset outside
// [0, n_bytes] does not raise it, so it spoils only the two documents it bounds.  A document whose
// range is not in the batch, or that starts before an earlier offset (its rebased start would not be its own), is
// flagged and reported as VPT_SENT_BAD_RANGE with no tokens; every other document keeps its exact range.
#pragma once
#include <cstdint>

#include "common.hpp"

namespace vpt {

constexpr uint64_t kMaxDocBytes = uint64_t(1) << 30;  // a document's length limit (as vpt_token_spans)

// what offset `o` adds to the prefix maximum: itself inside [0, n_bytes], else nothing
VPT_HD uint64_t doc_key(int64_t o, uint64_t n_bytes) { return o >= 0 && uint64_t(o) <= n_bytes ? uint64_t(o) : 0u; }

// 0 <= lo <= hi <= n_bytes and hi - lo <= 1 GiB
VPT_HD bool doc_range_ok(int64_t lo, int64_t hi, uint64_t n_bytes) {
    return lo >= 0 && lo <= hi && uint64_t(hi) <= n_bytes && uint64_t(hi - lo) <= kMaxDocBytes;
}

// document [lo, hi) given the largest key of the offsets before lo in the array (0 for the first document)
VPT_HD bool doc_bad(int64_t lo, int64_t hi, uint64_t n_bytes, uint64_t max_before) {
    return !doc_range_ok(lo, hi, n_bytes) || uint64_t(lo) < max_before;
}

}  // namespace vpt
