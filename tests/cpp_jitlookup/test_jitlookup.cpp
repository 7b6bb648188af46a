// TEST INFRASTRUCTURE ONLY.  Generates the lookup-check kernels of a lowered lookup program with jit::generate
// (miden-vm_b200/csrc/jit.hpp, MODE_LOOKUP_CHECK) and compiles them with NVRTC for sm_90a; no device is needed.
//   test_jitlookup <program.bin> <mode> <out prefix>
// program.bin: the op-list words (u32, little-endian); mode: lookup-check | constraints | lookup | check, the last three
// for comparing the other modes' generated source.  The lookup program's column count is the largest interaction column
// plus one.  Writes <prefix>.cu (the generated source) and, unless mode is given with a "-source" suffix,
// <prefix>.cubin.  Prints one line:
//   JITLOOKUP chunks=<n> spill_base=<n> spill_ext=<n> cols=<n> source_bytes=<n> cubin_bytes=<n> compile_ms=<t>
#include "jit.hpp"

#include <chrono>
#include <cstring>
#include <fstream>
#include <iterator>

int main(int argc, char** argv) {
    if (argc != 4) { fprintf(stderr, "usage: %s program.bin lookup-check|constraints|lookup|check[-source] out_prefix\n", argv[0]); return 2; }
    std::ifstream in(argv[1], std::ios::binary);
    std::vector<char> bytes((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
    if (!in.good() && !in.eof()) { fprintf(stderr, "cannot read %s\n", argv[1]); return 2; }
    std::vector<uint32_t> w(bytes.size() / 4);
    memcpy(w.data(), bytes.data(), w.size() * 4);
    std::string mode_s = argv[2];
    const bool source_only = mode_s.size() > 7 && mode_s.substr(mode_s.size() - 7) == "-source";
    if (source_only) mode_s.resize(mode_s.size() - 7);
    const jit::Mode mode = mode_s == "lookup-check" ? jit::MODE_LOOKUP_CHECK : mode_s == "lookup" ? jit::MODE_LOOKUP
                         : mode_s == "check" ? jit::MODE_CHECK : jit::MODE_CONSTRAINTS;
    uint32_t n_cols = 0;
    if (mode == jit::MODE_LOOKUP || mode == jit::MODE_LOOKUP_CHECK)
        for (uint32_t q = 0; q < w[3]; q++) n_cols = std::max(n_cols, w[5 + 3 * (size_t)w[2] + 4 * (size_t)q] + 1);
    jit::GenInfo gi;
    const std::string src = jit::generate(w.data(), &gi, mode, n_cols);
    const std::string prefix = argv[3];
    { std::ofstream o(prefix + ".cu"); o << src; }
    size_t cubin_bytes = 0;
    double ms = 0;
    if (!source_only) {
        auto t0 = std::chrono::steady_clock::now();
        std::vector<char> cubin;
        try { cubin = jit::compile(src); }
        catch (const std::exception& e) { printf("JITLOOKUP_ERROR %s\n", e.what()); return 1; }
        ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        std::ofstream o(prefix + ".cubin", std::ios::binary);
        o.write(cubin.data(), (std::streamsize)cubin.size());
        cubin_bytes = cubin.size();
    }
    printf("JITLOOKUP chunks=%u spill_base=%u spill_ext=%u cols=%u source_bytes=%zu cubin_bytes=%zu compile_ms=%.0f\n",
           gi.n_chunks, gi.spill_base, gi.spill_ext, n_cols, src.size(), cubin_bytes, ms);
    return 0;
}
