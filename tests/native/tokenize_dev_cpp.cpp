// One call of vaporetto::Predictor::tokenize_dev (include/vaporetto_b200.hpp) on documents copied to the device, with
// int32 offsets and a sizing pass first.  usage: tokenize_dev_cpp <model.bin> <predict_tags 0|1> <doc>...
// Prints every document's tokenized text on its own line.
#include <cuda_runtime.h>

#include <cstdio>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>

#include "../../include/vaporetto_b200.hpp"

#define CK(x) do { if ((x) != cudaSuccess) { std::fprintf(stderr, "%s failed\n", #x); return 1; } } while (0)

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    std::ifstream f(argv[1], std::ios::binary);
    std::vector<uint8_t> bytes((std::istreambuf_iterator<char>(f)), {});
    const bool tags = std::string(argv[2]) == "1";
    vaporetto::Predictor p(vaporetto::Model::read(bytes), tags, 0);
    std::string text;
    std::vector<int32_t> off{0};
    for (int i = 3; i < argc; ++i) {
        text += argv[i];
        off.push_back(int32_t(text.size()));
    }
    const size_t n = off.size() - 1;
    uint8_t *d_text = nullptr, *d_status = nullptr, *d_chars = nullptr;
    int32_t* d_off = nullptr;
    int64_t* d_out_off = nullptr;
    void* d_ws = nullptr;
    CK(cudaMalloc(&d_text, text.size() + 1));
    CK(cudaMalloc(&d_off, 4 * off.size()));
    CK(cudaMalloc(&d_out_off, 8 * (n + 1)));
    CK(cudaMalloc(&d_status, n + 1));
    CK(cudaMemcpy(d_text, text.data(), text.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_off, off.data(), 4 * off.size(), cudaMemcpyHostToDevice));
    vaporetto::Predictor::DeviceText out;
    out.workspace_bytes = p.tokenize_dev_workspace_size(n, text.size(), tags);
    CK(cudaMalloc(&d_ws, out.workspace_bytes));
    out.workspace = d_ws;
    out.offsets = d_out_off;
    out.status = d_status;
    try {
        // the offsets-only pass sizes the output exactly
        p.tokenize_dev(d_text, text.size(), d_off, 4, n, out, false, 0, tags);
        std::vector<int64_t> h_off(n + 1);
        CK(cudaMemcpy(h_off.data(), d_out_off, 8 * (n + 1), cudaMemcpyDeviceToHost));
        if (uint64_t(h_off[n]) > p.tokenize_dev_out_bound(n, text.size(), tags)) return 3;
        CK(cudaMalloc(&d_chars, h_off[n] + 1));
        out.chars = d_chars;
        out.capacity = uint64_t(h_off[n]);
        p.tokenize_dev(d_text, text.size(), d_off, 4, n, out, false, 0, tags);
        std::string chars(static_cast<size_t>(h_off[n]), '\0');
        CK(cudaMemcpy(&chars[0], d_chars, chars.size(), cudaMemcpyDeviceToHost));
        for (size_t d = 0; d < n; ++d) std::printf("%s\n", chars.substr(size_t(h_off[d]), size_t(h_off[d + 1] - h_off[d])).c_str());
    } catch (const vaporetto::VaporettoError& e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    cudaFree(d_text); cudaFree(d_off); cudaFree(d_out_off); cudaFree(d_status); cudaFree(d_ws); cudaFree(d_chars);
    return 0;
}
