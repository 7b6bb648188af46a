// Host-side construction of the NTT tables (tiny: O(N1 + N2 + sqrt N) words per plan).  Shared by
// session.cu, which uploads them, and tests/cpp/test_ntt_v2.cpp, which runs the block functions of
// ntt2.cuh on the CPU with exactly these tables.
#pragma once
#include "gl.cuh"
#include "kernels.cuh"
#include <vector>

namespace ntt_tables {
using gl::u64;
using gl::u32;

// N = N1 * N2: one contiguous pass up to 2^11, otherwise a strided pass of N1 and a contiguous pass of N2
inline void split_n(u32 n, u32& n1, u32& n2) {
    if (n <= 11) { n1 = 0; n2 = n; }
    else { n1 = n / 2; n2 = n - n1; }
}
inline std::vector<u64> powers(u64 base, size_t count) {
    std::vector<u64> v(count);
    u64 x = 1;
    for (size_t i = 0; i < count; i++) { v[i] = x; x = gl::mul(x, base); }
    return v;
}

struct NttHost {
    u32 n, n1, n2, lo_bits;
    std::vector<u64> data;
    size_t o_tw1, o_twi1, o_twi2, o_lo, o_hi, o_ilo, o_ihi;
    mk::NttTables view(const u64* b) const {
        return mk::NttTables{n, n1, n2, lo_bits, b + o_tw1, b + o_twi1, b + o_twi2, b + o_lo, b + o_hi, b + o_ilo, b + o_ihi};
    }
};
inline NttHost build_ntt(u32 n) {
    NttHost h;
    h.n = n; split_n(n, h.n1, h.n2);
    h.lo_bits = (n + 1) / 2;
    u32 n1 = h.n1, n2 = h.n2, lo_bits = h.lo_bits;
    u64 w = gl::two_adic_generator(n), wi = gl::inv(w);
    auto push = [&](const std::vector<u64>& v) {   // every table starts on a 16-byte boundary: it may be the source of a bulk copy (tma.cuh)
        if (h.data.size() & 1) h.data.push_back(0);
        size_t off = h.data.size(); h.data.insert(h.data.end(), v.begin(), v.end()); return off;
    };
    u64 w1 = gl::two_adic_generator(n1), w2 = gl::two_adic_generator(n2);
    h.o_tw1 = push(powers(w1, n1 ? (size_t)1 << (n1 - 1) : 1));
    h.o_twi1 = push(powers(gl::inv(w1), n1 ? (size_t)1 << (n1 - 1) : 1));
    h.o_twi2 = push(powers(gl::inv(w2), n2 ? (size_t)1 << (n2 - 1) : 1));
    h.o_lo = push(powers(w, (size_t)1 << lo_bits));
    h.o_hi = push(powers(gl::exp_pow2(w, lo_bits), (size_t)1 << (n - lo_bits)));
    h.o_ilo = push(powers(wi, (size_t)1 << lo_bits));
    h.o_ihi = push(powers(gl::exp_pow2(wi, lo_bits), (size_t)1 << (n - lo_bits)));
    return h;
}

// Per coset base g of a size-2^n forward transform:
//   tab_b[j1] = g^j1 / N
//   tab_c[(1 << s) - 1 + j] = (g^N1)^(N2 / 2^(s+1)) * w_{2^(s+1)}^j,  s < n2, j < 2^s   (staged twiddles, ntt2.cuh)
// A base's tab_c block is the source of a bulk copy (table_load, ntt2.cuh) when it is 16-byte aligned: the blocks start at
// nb * N1 + b * N2 words, even unless N1 = 1 and nb is odd (then table_load falls back to a plain copy).
struct PremulHost {
    u32 n_bases;
    std::vector<u64> data;
    size_t o_b, o_c;
    mk::PremulTables view(const u64* b) const { return mk::PremulTables{b + o_b, b + o_c}; }
};
inline PremulHost build_premul(const std::vector<u64>& bases, u32 n) {
    u32 n1, n2; split_n(n, n1, n2);
    size_t N1 = (size_t)1 << n1, N2 = (size_t)1 << n2, nb = bases.size();
    u64 n_inv = gl::inv((u64)1 << n);
    PremulHost h;
    h.n_bases = (u32)nb;
    h.o_b = 0; h.o_c = nb * N1;
    h.data.assign(nb * (N1 + N2), 0);
    for (size_t b = 0; b < nb; b++) {
        u64 g = bases[b], gN1 = gl::exp_pow2(g, n1);
        u64 x = n_inv;
        for (size_t j1 = 0; j1 < N1; j1++) { h.data[h.o_b + b * N1 + j1] = x; x = gl::mul(x, g); }
        u64* tc = &h.data[h.o_c + b * N2];
        for (u32 s = 0; s < n2; s++) {
            u64 shift = gl::exp_pow2(gN1, n2 - 1 - s), ws = gl::two_adic_generator(s + 1);
            u64 y = shift;
            for (size_t j = 0; j < ((size_t)1 << s); j++) { tc[(((size_t)1 << s) - 1) + j] = y; y = gl::mul(y, ws); }
        }
    }
    return h;
}

}  // namespace ntt_tables
