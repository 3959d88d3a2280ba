// Re-annotation through include/vaporetto_b200.hpp: Predictor::reannotate_lines and LineStream(ReannotateLines) on the
// partially annotated lines of <input>, with the input tags kept and dropped.  The whole-buffer and streamed outputs
// must agree; the kept one goes to stdout, then the dropped one, for the caller to compare.
// usage: reannotate_cpp_test <model.bin> <input> <margin>
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
    if (argc < 4) return 2;
    std::ifstream f(argv[1], std::ios::binary), in(argv[2], std::ios::binary);
    const std::vector<uint8_t> bytes((std::istreambuf_iterator<char>(f)), {});
    const std::string text((std::istreambuf_iterator<char>(in)), {});
    const int32_t margin = int32_t(std::atol(argv[3]));
    Predictor p(Model::read(bytes), true);
    std::string out;
    for (bool keep : {true, false}) {
        const std::string whole = p.reannotate_lines(text, margin, keep, false, 0, true);
        std::string streamed;
        {
            LineStream st(p, LineStream::ReannotateLines{margin, keep},
                          [&](const uint8_t* b, size_t n) { streamed.append(reinterpret_cast<const char*>(b), n); },
                          false, 0, true);
            for (size_t i = 0; i < text.size(); i += 777) st.feed(text.substr(i, 777));
            st.finish();
        }
        CHECK(streamed == whole);
        out += whole;
    }
    // a malformed line throws, naming it
    bool threw = false;
    try {
        p.reannotate_lines("猫|だ\n猫?だ\n", margin);
    } catch (const VaporettoError& e) {
        threw = std::string(e.what()).find("(line 1)") != std::string::npos;
    }
    CHECK(threw);
    std::fwrite(out.data(), 1, out.size(), stdout);
    return 0;
}
