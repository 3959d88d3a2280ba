// CPU oracle of vpt_predict_tags_batch_dev: `Predictor::predict_tags` (reference predictor.rs:546-637) on boundaries the
// caller gives, over the oracle's Sentence / Predictor (oracle/vaporetto_oracle.cpp, compiled into this library
// unchanged).  Per sentence: parse_raw, predict (for the pattern-id states), the caller's 0 / 1 boundaries over the
// predicted ones, fill_tags.  Test infrastructure only: tests/vpt_testlib/tags_given_oracle.py builds and loads it.
#include "../../oracle/vaporetto_oracle.cpp"

extern "C" {

// A batch in the layout of vpt_predict_tags_batch_dev: sentence i is utf8[byte_offsets[i], byte_offsets[i + 1]), its
// boundaries are boundaries[bound_offsets[i] ..] (NULL: keep the predicted ones), its characters tag_token /
// tag_cand [char_offsets[i] ..) (n_tags candidates per character).  A sentence the reference rejects (empty, NUL,
// invalid UTF-8) gets -1 over its characters.  Returns 0, or 2 with ora_last_error() naming the sentence whose
// offsets or boundaries do not fit it.
int ora_tags_given(const void* p, const char* utf8, const uint64_t* byte_offsets, size_t n_sent,
                   const uint64_t* bound_offsets, const uint8_t* boundaries, const uint64_t* char_offsets,
                   int32_t* tag_token, int32_t* tag_cand) {
    ORA_TRY
    auto* pr = static_cast<const Predictor*>(p);
    const size_t nt = pr->n_tags;
    Sentence s;
    vector<int32_t> tt, ti;
    for (size_t i = 0; i < n_sent; ++i) {
        const size_t c0 = size_t(char_offsets[i]), nc = size_t(char_offsets[i + 1] - char_offsets[i]);
        try {
            s.parse_raw(utf8 + byte_offsets[i], size_t(byte_offsets[i + 1] - byte_offsets[i]));
            pr->predict(s);
        } catch (const Error&) {
            for (size_t k = 0; k < nc; ++k) tag_token[c0 + k] = -1;
            for (size_t k = 0; k < nc * nt; ++k) tag_cand[c0 * nt + k] = -1;
            continue;
        }
        const string at = " (sentence " + std::to_string(i) + ")";
        if (nc != s.len()) throw Error(INVALID_ARGUMENT, "char_offsets: do not fit the sentence" + at);
        if (boundaries) {
            if (bound_offsets[i + 1] - bound_offsets[i] != s.boundaries.size())
                throw Error(INVALID_ARGUMENT, "bound_offsets: do not fit the sentence" + at);
            for (size_t k = 0; k < s.boundaries.size(); ++k) {
                const uint8_t b = boundaries[bound_offsets[i] + k];
                if (b > 1) throw Error(INVALID_ARGUMENT, "boundaries: must be 0 or 1" + at);
                s.boundaries[k] = b;
            }
        }
        pr->fill_tags(s, tt, ti, nullptr);
        memcpy(tag_token + c0, tt.data(), nc * 4);
        if (nt) memcpy(tag_cand + c0 * nt, ti.data(), nc * nt * 4);
    }
    return 0;
    ORA_CATCH(idret)
}

}  // extern "C"
