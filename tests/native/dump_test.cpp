// Host build of the dump kernels' arithmetic (vaporetto_b200/csrc/dump.hpp): the digit counts and decimal writer against
// snprintf("%d") / ("%llu") on every digit-count edge of i32 and u64, and the UTF-8 length and encoding of the
// full-width image of every BMP code point against the oracle's encoder (append_utf8, kytea_fullwidth_cp).  Prints
// "ok" and exits 0 when everything matches.
#include "../../oracle/vaporetto_oracle.cpp"
#include "../../vaporetto_b200/csrc/dump.hpp"

#include <cstdio>
#include <vector>

static int fails = 0;
static void expect(bool c, const char* what, long long v) {
    if (!c && fails++ < 20) std::printf("FAIL %s %lld\n", what, v);
}

int main() {
    std::vector<long long> vals = {INT32_MIN, INT32_MIN + 1, -1, 0, 1, INT32_MAX, INT32_MAX - 1};
    for (long long p = 1; p <= 1000000000LL; p *= 10)
        for (long long v : {p, p - 1, p + 1, -p, -(p - 1), -(p + 1)})
            if (v >= INT32_MIN && v <= INT32_MAX) vals.push_back(v);
    for (long long v : vals) {
        char want[32];
        const int n = std::snprintf(want, sizeof want, "%d", int32_t(v));
        expect(vpt::dec_len(int32_t(v)) == uint32_t(n), "dec_len", v);
        uint8_t got[32];
        vpt::DumpWrite w{got};
        w.i32(int32_t(v));
        expect(w.p - got == n && std::memcmp(got, want, size_t(n)) == 0, "i32", v);
        vpt::DumpCount c;
        c.i32(int32_t(v));
        expect(c.n == uint64_t(n), "count i32", v);
    }
    for (unsigned long long p = 1; p <= 10000000000000000000ULL; p *= 10) {
        for (unsigned long long v : {p, p - 1, p + 1}) {
            char want[32];
            const int n = std::snprintf(want, sizeof want, "%llu", v);
            uint8_t got[32];
            vpt::DumpWrite w{got};
            w.u64(v);
            expect(vpt::dec_len_u64(v) == uint32_t(n) && w.p - got == n && std::memcmp(got, want, size_t(n)) == 0, "u64",
                   (long long)v);
        }
        if (p == 10000000000000000000ULL) break;
    }
    for (uint32_t c = 0; c < 0x10000; ++c) {
        if (c >= 0xD800 && c < 0xE000) continue;  // not characters
        for (int norm = 0; norm < 2; ++norm) {
            const uint32_t m = norm ? vpt::kytea_fullwidth(c) : c;
            expect(m == (norm ? kytea_fullwidth_cp(c) : c), "fullwidth", c);
            std::string want;
            append_utf8(want, m);
            uint8_t got[8];
            vpt::DumpWrite w{got};
            w.cp(m);
            vpt::DumpCount k;
            k.cp(m);
            expect(vpt::utf8_len(m) == want.size() && k.n == want.size(), "utf8_len", c);
            expect(size_t(w.p - got) == want.size() && std::memcmp(got, want.data(), want.size()) == 0, "utf8", c);
            const uint8_t* q = got;
            expect(vpt::dump_next_cp(q) == m && q == w.p, "decode", c);
        }
    }
    if (fails) return 1;
    std::printf("ok\n");
    return 0;
}
