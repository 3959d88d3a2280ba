// Host run of the document offset arithmetic of vpt_token_spans_dev (vaporetto_b200/csrc/doc_offsets.hpp), composed as
// k_doc_max / k_doc_scan / k_doc_offsets compose it: the rebased offset i is shift + the prefix maximum of the keys of the
// offsets, document d is flagged by doc_bad with the maximum before it.  tests/test_doc_offsets_cpu.py feeds cases on
// stdin, one per line: "width n_bytes shift k o[0] .. o[k-1]" (width 4: the offsets are stored as int32 and read back
// sign-extended, as the kernels read them), and compares each output line "v[0] .. v[k-1] | bad[0] .. bad[k-2]" with a
// Python restatement.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../vaporetto_b200/csrc/doc_offsets.hpp"

using namespace vpt;

int main() {
    int width;
    unsigned long long n_bytes;
    unsigned shift;
    size_t k;
    while (scanf("%d %llu %u %zu", &width, &n_bytes, &shift, &k) == 4) {
        std::vector<int64_t> o(k);
        for (size_t i = 0; i < k; ++i) {
            long long x;
            if (scanf("%lld", &x) != 1) return 2;
            o[i] = width == 4 ? int64_t(int32_t(uint32_t(uint64_t(x)))) : int64_t(x);
        }
        std::vector<uint64_t> before(k);  // largest key in front of i
        uint64_t m = 0;
        for (size_t i = 0; i < k; ++i) {
            before[i] = m;
            m = std::max(m, doc_key(o[i], n_bytes));
        }
        for (size_t i = 0; i < k; ++i) printf("%llu ", (unsigned long long)(std::max(before[i], doc_key(o[i], n_bytes)) + shift));
        printf("|");
        for (size_t d = 0; d + 1 < k; ++d) printf(" %d", doc_bad(o[d], o[d + 1], n_bytes, before[d]) ? 1 : 0);
        printf("\n");
    }
    return 0;
}
