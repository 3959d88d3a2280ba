// The partial-annotation output of include/vaporetto_b200.hpp: Sentence::write_partial_annotation_text on the reference's
// doc example (host), and with `gpu`, Predictor::annotate_lines and LineStream(AnnotateLines) on the lines of <input>:
// both outputs must agree, and the whole-buffer one goes to stdout for the caller to compare.  Each line's
// predict + fill_tags + write_partial_annotation_text at margin 0 must equal annotate_lines' line.
// usage: annotate_cpp_test <model.bin> [gpu <input> <margin>]
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>

#include "../../include/vaporetto_b200.hpp"

using namespace vaporetto;

#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "CHECK failed at line %d: %s\n", __LINE__, #c); return 1; } } while (0)

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    std::string buf;
    Sentence::from_raw("まぁ良いだろう").write_partial_annotation_text(buf);
    CHECK(buf == "ま ぁ 良 い だ ろ う");
    if (argc < 5) {
        std::printf("annotate cpp (host) ok\n");
        return 0;
    }
    std::ifstream f(argv[1], std::ios::binary), in(argv[3], std::ios::binary);
    const std::vector<uint8_t> bytes((std::istreambuf_iterator<char>(f)), {});
    const std::string text((std::istreambuf_iterator<char>(in)), {});
    const int32_t margin = int32_t(std::atol(argv[4]));
    Predictor p(Model::read(bytes), true);
    const std::string whole = p.annotate_lines(text, margin, false, 0, true);
    std::string streamed;
    {
        LineStream st(p, LineStream::AnnotateLines{margin},
                      [&](const uint8_t* b, size_t n) { streamed.append(reinterpret_cast<const char*>(b), n); }, false, 0,
                      true);
        for (size_t i = 0; i < text.size(); i += 777) st.feed(text.substr(i, 777));
        st.finish();
    }
    CHECK(streamed == whole);
    // the host Sentence path at margin 0: every line as annotate_lines writes it
    const std::string zero = p.annotate_lines(text, 0, true, 0, true);
    size_t lo = 0, zlo = 0;
    while (lo < text.size()) {
        size_t end = text.find('\n', lo), zend = zero.find('\n', zlo);
        if (end == std::string::npos) end = text.size();
        const std::string line = text.substr(lo, end - lo), want = zero.substr(zlo, zend - zlo);
        if (!line.empty()) {
            Sentence s = Sentence::from_raw(line);
            p.predict(s);
            s.fill_tags();
            s.write_partial_annotation_text(buf);
            CHECK(buf == want);
        }
        lo = end + 1;
        zlo = zend + 1;
    }
    std::fwrite(whole.data(), 1, whole.size(), stdout);
    return 0;
}
