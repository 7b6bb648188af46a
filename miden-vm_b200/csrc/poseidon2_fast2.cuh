// Lazy-reduction Goldilocks arithmetic + Poseidon2 (width 12) for the sm_90a integer pipes: the field
// arithmetic of the hash and NTT kernels.  Same permutation as the canonical p2::permute (poseidon2.cuh) up to the
// choice of representatives; reference: crates/crypto/src/hash/algebraic_sponge/poseidon2/mod.rs:226-319 (layer structure),
// constants.rs:18-31 (internal diagonal).
//
// What keeps the SASS instruction count per permutation down:
//   * the 128-bit product comes from ONE unsigned __int128 multiplication (4 IMAD.WIDE + 3) instead
//     of a separate mul.lo / mul.hi pair (11);
//   * every "fold the carry back" adds a 0 / 2^32 - 1 mask on the ALU pipe (fold);
//   * the 4x4 MDS uses the 8-addition evaluation order (t01, t23, t0123, t01123, t01233);
//   * negative diagonal entries subtract from (sum + 8p) instead of adding (8p - x);
//   * x/4 and x/8 are one exact division by 2^k: (x + n p) >> k with n = -x mod 2^k;
//   * the internal rounds reduce lanes 1..11 once every 8 rounds only (internal_rounds_lazy).
//
// Every function is __host__ __device__: the device side uses the carry flag through PTX idioms
// (add.cc/addc, sub.cc/subc inside ONE asm statement), the host side restates each
// primitive with unsigned __int128, so that tests/cpp/test_arith_v2.cpp runs THIS source on the CPU
// against the canonical p2::permute and the reference's KAT.  Elements travel as arbitrary u64
// representatives (value mod p, not necessarily < p); callers canonicalise what they store.
#pragma once
#include "gl.cuh"
#include "poseidon2.cuh"

namespace glf {
using gl::u64;
using gl::u32;
typedef unsigned __int128 u128;

struct W { u64 lo; u32 hi; };   // lo + hi * 2^64, hi stays small (< 2^8 in every use)

static constexpr u64 EPS = 0xFFFFFFFFull;            // 2^64 mod p

// ---- carry primitives ----------------------------------------------------------------------------
// r = a + b mod 2^64, c = carry (0 / 1)
GL_HD void addc64(u64 a, u64 b, u64& r, u32& c) {
#ifdef __CUDA_ARCH__
    asm("add.cc.u64 %0, %2, %3;\n\taddc.u32 %1, 0, 0;" : "=l"(r), "=r"(c) : "l"(a), "l"(b));
#else
    u128 s = (u128)a + b; r = (u64)s; c = (u32)(s >> 64);
#endif
}
// r = a - b mod 2^64, m = 0xFFFFFFFF if the subtraction borrowed, else 0
GL_HD void subb64(u64 a, u64 b, u64& r, u32& m) {
#ifdef __CUDA_ARCH__
    asm("sub.cc.u64 %0, %2, %3;\n\tsubc.u32 %1, 0, 0;" : "=l"(r), "=r"(m) : "l"(a), "l"(b));
#else
    r = a - b; m = a < b ? 0xFFFFFFFFu : 0u;
#endif
}
// a * (2^32 - 1) as a 64-bit product.  The explicit mul.wide keeps ptxas fusing it with the following add.cc
// into one IMAD.WIDE.U32 with carry-out (a plain C product of a limb of the 128-bit multiply does not fuse).
GL_HD u64 mul_eps(u32 a) {
#if defined(__CUDA_ARCH__)
    u64 m;
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(m) : "r"(a), "r"(0xFFFFFFFFu));
    return m;
#else
    return (u64)a * 0xFFFFFFFFull;
#endif
}
// c * (2^32 - 1) + r for c in {0, 1}.  Callers guarantee no overflow.  Added as the mask 0 / 2^32 - 1 on the ALU pipe:
// the hash kernels are bound by the FMA-heavy pipe, where the IMAD.WIDE form of this fold costs four cycles per warp
// (~1.6 plain IMADs), and the ALU pipe has slack.
GL_HD u64 fold(u32 c, u64 r) { return r + (u64)(0u - c); }

GL_HD u64 canon(u64 x) { return x >= gl::P ? x - gl::P : x; }

// 128-bit (hi:lo) -> u64 representative.  2^64 = 2^32 - 1, 2^96 = -1 (mod p).
GL_HD u64 red128(u64 lo, u64 hi) {
    u32 x2 = (u32)hi, x3 = (u32)(hi >> 32);
    u64 t, r; u32 m, c;
    subb64(lo, (u64)x3, t, m);
    t -= (u64)m;                     // borrowed: the wrap added 2^64 = 2^32 - 1, take it back (t >= 2^64 - 2^32 then)
    addc64(t, mul_eps(x2), r, c);       // x2 * (2^32 - 1) <= 2^64 - 2^33 + 1
    return fold(c, r);               // carried: r < 2^64 - 2^33 + 1, so r + 2^32 - 1 fits
}
GL_HD u64 mul(u64 a, u64 b) {
    u128 q = (u128)a * b;
    return red128((u64)q, (u64)(q >> 64));
}
// a^2.  (Three partial products, a0^2 + a0 a1 2^33 + a1^2 2^64, save an IMAD.WIDE but add shifts and a longer carry chain.)
GL_HD u64 sqr(u64 a) { return mul(a, a); }

// x + k for a canonical constant k (< p): a carry leaves r < k < p, so the fold fits.
GL_HD u64 add_const(u64 x, u64 k) {
    u64 r; u32 c;
    addc64(x, k, r, c);
    return fold(c, r);
}

// ---- 96-bit accumulators -------------------------------------------------------------------------
GL_HD W wide(u64 x) { W w; w.lo = x; w.hi = 0; return w; }
GL_HD void wadd(W& w, u64 x) {
#ifdef __CUDA_ARCH__
    asm("add.cc.u64 %0, %0, %2;\n\taddc.u32 %1, %1, 0;" : "+l"(w.lo), "+r"(w.hi) : "l"(x));
#else
    u128 s = (u128)w.lo + x; w.lo = (u64)s; w.hi += (u32)(s >> 64);
#endif
}
GL_HD void wadd(W& w, W x) {
#ifdef __CUDA_ARCH__
    asm("add.cc.u64 %0, %0, %2;\n\taddc.u32 %1, %1, %3;" : "+l"(w.lo), "+r"(w.hi) : "l"(x.lo), "r"(x.hi));
#else
    u128 s = (u128)w.lo + x.lo; w.lo = (u64)s; w.hi += x.hi + (u32)(s >> 64);
#endif
}
// a + b of two representatives as a wide value
GL_HD W wsum(u64 a, u64 b) {
    W w;
    addc64(a, b, w.lo, w.hi);
    return w;
}
// w - x for wide w >= x (the caller adds a multiple of p to w beforehand)
GL_HD void wsub(W& w, W x) {
#ifdef __CUDA_ARCH__
    u64 lo; u32 hi;
    asm("sub.cc.u64 %0, %2, %3;\n\tsubc.u32 %1, %4, %5;" : "=l"(lo), "=r"(hi) : "l"(w.lo), "l"(x.lo), "r"(w.hi), "r"(x.hi));
    w.lo = lo; w.hi = hi;
#else
    u32 b = w.lo < x.lo ? 1u : 0u; w.lo -= x.lo; w.hi = w.hi - x.hi - b;
#endif
}
GL_HD W wshl(u64 x, int k) { W w; w.lo = x << k; w.hi = (u32)(x >> (64 - k)); return w; }
GL_HD W wtriple(u64 x) { W w = wshl(x, 1); wadd(w, x); return w; }
// wide (hi < 2^32) -> u64 representative: lo + hi * (2^32 - 1), one carry fold.
GL_HD u64 wred(W w) {
    u64 r; u32 c;
    addc64(w.lo, mul_eps(w.hi), r, c);
    return fold(c, r);
}
static constexpr u64 P8_LO = 0xFFFFFFF800000008ull;   // 8p = 2^67 - 2^35 + 8
static constexpr u32 P8_HI = 7u;

// ---- canonical (< p) arithmetic for the NTT butterflies ------------------------------------------
GL_HD u64 canon_cc(u64 r) {      // r in [0, 2^64) -> r mod p
    u64 t; u32 m;
    subb64(r, gl::P, t, m);
    return t - (u64)m;           // borrowed (r < p): add p back == subtract 2^32 - 1 from the wrapped value
}
GL_HD u64 csub(u64 a, u64 b) {   // a, b < p
    u64 d; u32 m;
    subb64(a, b, d, m);
    return d - (u64)m;
}
GL_HD u64 cadd(u64 a, u64 b) { return csub(a, gl::P - b); }   // a - (p - b)
GL_HD u64 cmul(u64 a, u64 b) { return canon_cc(mul(a, b)); }

// x / 2 for any representative; result < 2^64.  (p + 1) / 2 = 2^63 - 2^31 + 1.
GL_HD u64 half(u64 x) { return (x >> 1) + (u64)((u32)x & 1u) * 0x7FFFFFFF80000001ull; }
// x / 2^k (k = 2, 3) for any representative: (x + n p) / 2^k with n = -x mod 2^k, which is
// ceil(x / 2^k) + n * (p - 1) / 2^k, and (p - 1) / 2^k = 2^(32-k) * (2^32 - 1).  Result < 2^64.
template <int K>
GL_HD u64 div2k(u64 x) {
    u32 n = (0u - (u32)x) & ((1u << K) - 1u);
    u64 q = (x >> K) + (n ? 1ull : 0ull);
    return (u64)(n << (32 - K)) * EPS + q;
}

// ---- 96-bit values as operands (the lazy internal rounds keep lanes 1..11 unreduced) -----------------
// w << k for a wide w (k = 1, 2); the caller's bound keeps the result below 2^96
GL_HD W wshl96(W w, int k) { W r; r.lo = w.lo << k; r.hi = (w.hi << k) | (u32)(w.lo >> (64 - k)); return r; }
GL_HD W wshr96(W w, int k) { W r; r.lo = (w.lo >> k) | ((u64)w.hi << (64 - k)); r.hi = w.hi >> k; return r; }
// w / 2 exactly: (w + (w odd) * p) >> 1
GL_HD W whalf(W w) {
    wadd(w, gl::P & (0ull - (w.lo & 1ull)));
    return wshr96(w, 1);
}
// w / 2^K exactly (K = 2, 3): (w + n p) >> K with n = -w mod 2^K (p = 1 mod 2^32), n p = n 2^64 - n (2^32 - 1)
template <int K>
GL_HD W wdiv2k(W w) {
    u32 n = (0u - (u32)w.lo) & ((1u << K) - 1u);
    w.hi += n;
    wsub(w, wide((u64)n * EPS));          // n > 0 put n 2^64 on top first, so the difference stays non-negative ((n << 32) - n on the ALU pipe: no difference)
    return wshr96(w, K);
}

}  // namespace glf

namespace p2f {
using gl::u64;
using gl::u32;
using glf::W;

#if !defined(__CUDA_ARCH__) && defined(P2F_TRACK_BOUNDS)
static u32 p2f_max_hi = 0;      // host test instrumentation: largest high word a lazy lane ever held
#endif

GL_HD u64 sbox(u64 x) {
    u64 x2 = glf::sqr(x), x3 = glf::mul(x2, x), x4 = glf::sqr(x2);
    return glf::mul(x3, x4);
}

// M4 = [[2,3,1,1],[1,2,3,1],[1,1,2,3],[3,1,1,2]] on each chunk (8 additions + 2 doublings), then every
// chunk receives the column sums (block-circulant [2M, M, M]).
GL_HD void external_layer(u64* s) {
    W y[12];
#pragma unroll
    for (int c = 0; c < 12; c += 4) {
        W t01 = glf::wsum(s[c], s[c + 1]), t23 = glf::wsum(s[c + 2], s[c + 3]);
        W t0123 = t01; glf::wadd(t0123, t23);
        W t01123 = t0123; glf::wadd(t01123, s[c + 1]);
        W t01233 = t0123; glf::wadd(t01233, s[c + 3]);
        W y3 = t01233; glf::wadd(y3, glf::wshl(s[c], 1));
        W y1 = t01123; glf::wadd(y1, glf::wshl(s[c + 2], 1));
        glf::wadd(t01123, t01);
        glf::wadd(t01233, t23);
        y[c] = t01123; y[c + 1] = y1; y[c + 2] = t01233; y[c + 3] = y3;
    }
#pragma unroll
    for (int l = 0; l < 4; l++) {
        W col = y[l];
        glf::wadd(col, y[4 + l]); glf::wadd(col, y[8 + l]);
#pragma unroll
        for (int c = 0; c < 12; c += 4) {
            W o = y[c + l];
            glf::wadd(o, col);
            s[c + l] = glf::wred(o);
        }
    }
}

// The 22 internal rounds with lanes 1..11 kept as UNREDUCED 96-bit values (VERDICT r1 #7): only lane 0 enters an S-box, so only
// lane 0 is reduced every round; the other lanes are reduced after every block of 8 rounds (8 + 8 + 6).  Bounds, with M_j the
// bound of the lanes entering round j of a block (M_0 = 2^64): sum_j < 2^64 + 11 M_j, the subtracting lanes use
// sum_j + OFF_j with OFF_j = ceil(4 M_j / p) p >= |d| lane, and M_(j+1) = sum_j + max(4 M_j, OFF_j) -- 2^68.1, 2^72.0, 2^75.9, 2^79.8,
// 2^83.7, 2^87.6, 2^91.5, 2^95.5 < 2^96 (tests/cpp/test_arith_v2.cpp recomputes the table and tracks the largest value seen).
// Per round this removes 11 of the 12 reductions (one IMAD.WIDE + five ALU instructions each) for one extra register per lane:
// fewer SASS instructions and IMAD.WIDE per round (the FMA-heavy pipe is the binding one).
#define P2F_OFF_LO {0xfffffffb00000005ull, 0xffffffbb00000045ull, 0xfffffbfb00000405ull, 0xffffc3bb00003c45ull, \
                    0xfffc77fb00038805ull, 0xffcb07bb0034f845ull, 0xfce573fb031a8c05ull, 0xd171cbbb2e8e3445ull}
#define P2F_OFF_HI {0x4u, 0x44u, 0x404u, 0x3c44u, 0x38804u, 0x34f844u, 0x31a8c04u, 0x2e8e3444u}
static const u64 H_OFF_LO[8] = P2F_OFF_LO;
static const u32 H_OFF_HI[8] = P2F_OFF_HI;
#ifdef __CUDACC__
__constant__ u64 D_OFF_LO[8] = P2F_OFF_LO;
__constant__ u32 D_OFF_HI[8] = P2F_OFF_HI;
#endif

GL_HD void internal_rounds_lazy(u64* s, const u64* rc) {
#ifdef __CUDA_ARCH__
    const u64* off_lo = D_OFF_LO; const u32* off_hi = D_OFF_HI;
#else
    const u64* off_lo = H_OFF_LO; const u32* off_hi = H_OFF_HI;
#endif
    W L[11];
#pragma unroll
    for (int i = 0; i < 11; i++) L[i] = glf::wide(s[i + 1]);
    u64 s0 = s[0];
    int r = 0;
#pragma unroll 1
    for (int blk = 0; blk < 3; blk++) {
        const int n = blk < 2 ? 8 : 6;
#pragma unroll 1
        for (int j = 0; j < n; j++, r++) {
            s0 = sbox(glf::add_const(s0, rc[r]));
            W sum = glf::wide(s0);
#pragma unroll
            for (int i = 0; i < 11; i++) glf::wadd(sum, L[i]);
            W sump = sum;
            { W off; off.lo = off_lo[j]; off.hi = off_hi[j]; glf::wadd(sump, off); }
            W t;
            t = sump; glf::wsub(t, glf::wshl(s0, 1)); s0 = glf::wred(t);                              // d0 = -2
            glf::wadd(L[0], sum);                                                                     // 1
            L[1] = glf::wshl96(L[1], 1); glf::wadd(L[1], sum);                                        // 2
            L[2] = glf::whalf(L[2]); glf::wadd(L[2], sum);                                            // 1/2
            t = glf::wshl96(L[3], 1); glf::wadd(t, L[3]); glf::wadd(t, sum); L[3] = t;                // 3
            L[4] = glf::wshl96(L[4], 2); glf::wadd(L[4], sum);                                        // 4
            t = sump; glf::wsub(t, glf::whalf(L[5])); L[5] = t;                                       // -1/2
            { W t3 = glf::wshl96(L[6], 1); glf::wadd(t3, L[6]); t = sump; glf::wsub(t, t3); L[6] = t; }   // -3
            t = sump; glf::wsub(t, glf::wshl96(L[7], 2)); L[7] = t;                                   // -4
            L[8] = glf::wdiv2k<2>(L[8]); glf::wadd(L[8], sum);                                        // 1/4
            t = sump; glf::wsub(t, glf::wdiv2k<2>(L[9])); L[9] = t;                                   // -1/4
            L[10] = glf::wdiv2k<3>(L[10]); glf::wadd(L[10], sum);                                     // 1/8
#if !defined(__CUDA_ARCH__) && defined(P2F_TRACK_BOUNDS)
            for (int i = 0; i < 11; i++) if (L[i].hi > p2f_max_hi) p2f_max_hi = L[i].hi;
#endif
        }
#pragma unroll
        for (int i = 0; i < 11; i++) L[i] = glf::wide(glf::wred(L[i]));
    }
    s[0] = s0;
#pragma unroll
    for (int i = 0; i < 11; i++) s[i + 1] = L[i].lo;
}

#ifdef __CUDA_ARCH__
#define P2F_RC_EXT_INITIAL p2::D_RC_EXT_INITIAL
#define P2F_RC_EXT_TERMINAL p2::D_RC_EXT_TERMINAL
#define P2F_RC_INTERNAL p2::D_RC_INTERNAL
#else
#define P2F_RC_EXT_INITIAL p2::P2_RC_EXT_INITIAL
#define P2F_RC_EXT_TERMINAL p2::P2_RC_EXT_TERMINAL
#define P2F_RC_INTERNAL p2::P2_RC_INTERNAL
#endif

// The 22 internal rounds stay a rolled loop (~26 KB of code; a fully unrolled permutation, 93 KB, stalled on
// instruction fetch).
// Output words are arbitrary representatives; canonicalise with glf::canon before storing.
GL_HD void permute(u64* s) {
    external_layer(s);
#pragma unroll 1
    for (int phase = 0; phase < 2; phase++) {
        const u64* rc = phase ? P2F_RC_EXT_TERMINAL : P2F_RC_EXT_INITIAL;
#pragma unroll 1
        for (int r = 0; r < 4; r++) {
#pragma unroll
            for (int i = 0; i < 12; i++) s[i] = sbox(glf::add_const(s[i], rc[12 * r + i]));
            external_layer(s);
        }
        if (phase == 0) internal_rounds_lazy(s, P2F_RC_INTERNAL);
    }
}

}  // namespace p2f
