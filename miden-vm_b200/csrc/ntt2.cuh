// NTT block functions: the bodies of the NTT kernels of kernels.cu.  Data layout and index conventions in DESIGN.md
// "NTT index conventions"; reference: Radix2DitParallel::coset_lde_batch at crates/lifted-stark/src/prover/commit.rs:173,
// quotient.rs:186-209.  What keeps the instruction count per point down:
//
//   * the coset shift of the contiguous pass lives in the butterfly twiddles: stage s of the DIT over a
//     chunk evaluates polynomials in y^(N2/2^(s+1)) at G^(N2/2^(s+1)) * w_{2^(s+1)}^j (G = g^N1), so a
//     per-coset table of N2 - 1 "staged" twiddles replaces the premultiplication of every coefficient;
//   * the remaining per-chunk scalar g^j1 / N rides on the inter-pass twiddle, which each lane advances
//     geometrically (one multiplication to advance + one to apply per element);
//   * butterflies keep lazy representatives: only the multiplied operand is canonicalised (x + c and x - c
//     with c < p need a single carry fix each); values are canonicalised where they leave the transform;
//   * in the round with the smallest spans of the plain-table transforms the unit twiddles are skipped.
//
// Every function is __host__ __device__ and written as index-parallel loops separated by barriers
// (NTT2_FOR / NTT2_SYNC): on the device a loop runs over threadIdx.x with stride blockDim.x and the barrier
// is __syncthreads(); on the host the same loop runs over all indices and the barrier is empty, which is
// equivalent because iterations of one loop never depend on each other.  tests/cpp/test_ntt_v2.cpp runs
// these block functions on the CPU against a textbook transform.
#pragma once
#include "poseidon2_fast2.cuh"
#include "kernels.cuh"
#include "tma.cuh"

namespace ntt2 {
using gl::u64;
using gl::u32;

#if defined(__CUDA_ARCH__) || defined(MDN_EMULATED)   // MDN_EMULATED: tests/emu runs one fiber per CUDA thread
#define NTT2_FOR(i, n) for (u32 i = threadIdx.x; i < (u32)(n); i += blockDim.x)
#define NTT2_SYNC() __syncthreads()
#else
#define NTT2_FOR(i, n) for (u32 i = 0; i < (u32)(n); i++)
#define NTT2_SYNC() ((void)0)
#endif

// tile element (idx, cc) of the run-time schedules, idx < 2^m, cc < 2^log_cols; contiguous tiles are padded by one word every 8
GL_HD u32 tile_off(u32 idx, u32 cc, u32 log_cols) {
    u32 o = (idx << log_cols) + cc;
    return log_cols ? o : o + (o >> 3);
}
// Words of a tile: room for the layout of the run-time schedules (tile_off) and for that of the compile-time ones (pad16)
GL_HD u32 tile_words(u32 m, u32 log_cols) {
    u32 n = 1u << (m + log_cols);
    return log_cols ? n + (n >> 4) : n + (n >> 3) + 1;
}
// Shared memory of the four block functions: [tile | table (16-byte aligned: it is the destination of a bulk copy) |
// mbarrier].  tw_off = offset of the table in words.
GL_HD u32 tw_off(u32 m, u32 log_cols) { return (tile_words(m, log_cols) + 1u) & ~1u; }
GL_HD size_t smem_words_contig_fwd(u32 n2) { return (size_t)tw_off(n2, 0) + ((size_t)1 << n2) + 2; }
GL_HD size_t smem_words_contig_inv(u32 n2) { return (size_t)tw_off(n2, 0) + ((size_t)1 << n2) / 2 + 4; }
GL_HD size_t smem_words_strided(u32 n1, u32 log_c) { return (size_t)tw_off(n1, log_c) + ((size_t)1 << n1) / 2 + 4; }

// Contiguous chunk <-> padded tile with coalesced 128-bit global accesses (two words per thread per access; chunks are
// 16-byte aligned whenever they hold at least two words because every column and chunk length is a power of two).
// P16: the layout of the compile-time schedules (pad16), else that of the run-time ones (tile_off).
GL_HD u32 pad16(u32 o) { return o + (o >> 4); }
template <bool P16 = false>
GL_HD u32 chunk_off(u32 i) { return P16 ? pad16(i) : tile_off(i, 0, 0); }
template <bool P16 = false>
GL_HD void load_chunk(u64* x, const u64* src, u32 n) {
#if defined(__CUDA_ARCH__)
    if (n >= 2 && (((size_t)src) & 15) == 0) {
        const ulonglong2* s2 = reinterpret_cast<const ulonglong2*>(src);
        NTT2_FOR(i, n / 2) { ulonglong2 v = s2[i]; x[chunk_off<P16>(2 * i)] = v.x; x[chunk_off<P16>(2 * i + 1)] = v.y; }
        return;
    }
#endif
    NTT2_FOR(i, n) x[chunk_off<P16>(i)] = src[i];
}
template <bool P16 = false>
GL_HD void store_chunk_canon(u64* dst, const u64* x, u32 n) {
#if defined(__CUDA_ARCH__)
    if (n >= 2 && (((size_t)dst) & 15) == 0) {
        ulonglong2* d2 = reinterpret_cast<ulonglong2*>(dst);
        NTT2_FOR(i, n / 2) d2[i] = make_ulonglong2(glf::canon_cc(x[chunk_off<P16>(2 * i)]), glf::canon_cc(x[chunk_off<P16>(2 * i + 1)]));
        return;
    }
#endif
    NTT2_FOR(i, n) dst[i] = glf::canon_cc(x[chunk_off<P16>(i)]);
}

// Stage `words` u64 of a table into shared memory.  On the device: one bulk asynchronous copy (cp.async.bulk -> mbarrier)
// issued by thread 0 when the table is big enough and 16-byte aligned, overlapping the tile loads that follow; the
// matching table_wait() must come before the first use.  Host / emulator / small tables: a plain strided loop.
struct TableLoad { bool async; };
GL_HD TableLoad table_load(u64* dst, const u64* src, u32 words, u64* bar) {
#if defined(__CUDA_ARCH__)
    const u32 bytes = (words * 8u + 15u) & ~15u;      // the tables carry at least one spare word behind them
    if (words >= 64 && ((((size_t)src) | ((size_t)dst)) & 15) == 0) {
        if (threadIdx.x == 0) { tma::mbar_init(bar, 1); }
        __syncthreads();
        if (threadIdx.x == 0) { tma::expect_tx(bar, bytes); tma::bulk_g2s(dst, src, bytes, bar); }
        return TableLoad{true};
    }
#endif
    (void)bar;
    NTT2_FOR(i, words) dst[i] = src[i];
    return TableLoad{false};
}
GL_HD void table_wait(TableLoad t, u64* bar) {
#if defined(__CUDA_ARCH__)
    if (t.async) tma::wait(bar, 0);
#endif
    (void)t; (void)bar;
}

// Twiddle of stage s (span 2^s), butterfly index j < 2^s, of a size-2^m transform.
//   plain table : tw[j << (m-1-s)]      = w_{2^(s+1)}^j                          (2^(m-1) entries)
//   staged table: tw[(1 << s) - 1 + j]  = G^(2^(m-1-s)) * w_{2^(s+1)}^j          (2^m - 1 entries, per coset base)
template <bool STAGED>
GL_HD u64 tw_at(const u64* tw, u32 m, u32 s, u32 j) { return STAGED ? tw[((1u << s) - 1u) + j] : tw[j << (m - 1 - s)]; }

// DIT (bit-reversed -> natural) stages b .. b+LOGR-1 on the group g of 2^LOGR elements idx = base + k * 2^b.
// UNIT0: b == 0 on a plain table, so the twiddle with j == 0 is 1.
// The butterflies of one group on its registers v[k] = element base + k * 2^b, lo = base mod 2^b.
template <int LOGR, bool STAGED, bool UNIT0>
GL_HD void dit_bfly(u64* v, const u64* tw, u32 m, u32 b, u32 lo) {
    constexpr int R = 1 << LOGR;
#pragma unroll
    for (int st = 0; st < LOGR; st++) {
#pragma unroll
        for (int k = 0; k < R; k++) {
            if (k & (1 << st)) continue;
            const u32 jj = (u32)(k & ((1 << st) - 1));
            u64 c;
            if (UNIT0 && jj == 0) c = glf::canon_cc(v[k + (1 << st)]);
            else c = glf::cmul(v[k + (1 << st)], tw_at<STAGED>(tw, m, b + st, lo + (jj << b)));
            u64 a = v[k];
            v[k] = glf::add_const(a, c);            // a any representative, c < p
            v[k + (1 << st)] = glf::csub(a, c);     // one borrow fix is enough for c < p
        }
    }
}
template <int LOGR, bool STAGED, bool UNIT0>
GL_HD void dit_group(u64* x, const u64* tw, u32 m, u32 b, u32 log_cols, u32 g) {
    constexpr int R = 1 << LOGR;
    u32 cc = g & ((1u << log_cols) - 1), gg = g >> log_cols;
    u32 lo = gg & ((1u << b) - 1), hi = gg >> b;
    u32 base = (hi << (b + LOGR)) | lo;
    u64 v[R];
#pragma unroll
    for (int k = 0; k < R; k++) v[k] = x[tile_off(base + ((u32)k << b), cc, log_cols)];
    dit_bfly<LOGR, STAGED, UNIT0>(v, tw, m, b, lo);
#pragma unroll
    for (int k = 0; k < R; k++) x[tile_off(base + ((u32)k << b), cc, log_cols)] = v[k];
}
// DIF (natural -> bit-reversed) stages with spans 2^(b+LOGR-1) .. 2^b on the plain table.
// UNIT0: b == 0, so the twiddle with j == 0 is 1.
template <int LOGR, bool UNIT0>
GL_HD void dif_bfly(u64* v, const u64* tw, u32 m, u32 b, u32 lo) {
    constexpr int R = 1 << LOGR;
#pragma unroll
    for (int st = LOGR - 1; st >= 0; st--) {
#pragma unroll
        for (int k = 0; k < R; k++) {
            if (k & (1 << st)) continue;
            const u32 jj = (u32)(k & ((1 << st) - 1));
            u64 a = v[k], c = glf::canon_cc(v[k + (1 << st)]);
            v[k] = glf::add_const(a, c);
            u64 d = glf::csub(a, c);
            v[k + (1 << st)] = (UNIT0 && jj == 0) ? d : glf::mul(d, tw_at<false>(tw, m, b + st, lo + (jj << b)));
        }
    }
}
template <int LOGR, bool UNIT0>
GL_HD void dif_group(u64* x, const u64* tw, u32 m, u32 b, u32 log_cols, u32 g) {
    constexpr int R = 1 << LOGR;
    u32 cc = g & ((1u << log_cols) - 1), gg = g >> log_cols;
    u32 lo = gg & ((1u << b) - 1), hi = gg >> b;
    u32 base = (hi << (b + LOGR)) | lo;
    u64 v[R];
#pragma unroll
    for (int k = 0; k < R; k++) v[k] = x[tile_off(base + ((u32)k << b), cc, log_cols)];
    dif_bfly<LOGR, UNIT0>(v, tw, m, b, lo);
#pragma unroll
    for (int k = 0; k < R; k++) x[tile_off(base + ((u32)k << b), cc, log_cols)] = v[k];
}

template <int LOGR, bool STAGED, bool UNIT0>
GL_HD void dit_round(u64* x, const u64* tw, u32 m, u32 b, u32 log_cols) {
    NTT2_FOR(g, 1u << (m - LOGR + log_cols)) dit_group<LOGR, STAGED, UNIT0>(x, tw, m, b, log_cols, g);
    NTT2_SYNC();
}
template <int LOGR, bool UNIT0>
GL_HD void dif_round(u64* x, const u64* tw, u32 m, u32 b, u32 log_cols) {
    NTT2_FOR(g, 1u << (m - LOGR + log_cols)) dif_group<LOGR, UNIT0>(x, tw, m, b, log_cols, g);
    NTT2_SYNC();
}
// radix-8 rounds, finishing with 4 + ... never 1 + 3
template <bool STAGED>
GL_HD void smem_dit(u64* x, const u64* tw, u32 m, u32 log_cols) {
    u32 b = 0;
    while (b < m) {
        u32 left = m - b;
        if (left >= 3 && left != 4) {
            if (b == 0) dit_round<3, STAGED, !STAGED>(x, tw, m, b, log_cols); else dit_round<3, STAGED, false>(x, tw, m, b, log_cols);
            b += 3;
        } else if (left == 4 || left == 2) {
            if (b == 0) dit_round<2, STAGED, !STAGED>(x, tw, m, b, log_cols); else dit_round<2, STAGED, false>(x, tw, m, b, log_cols);
            b += 2;
        } else {
            if (b == 0) dit_round<1, STAGED, !STAGED>(x, tw, m, b, log_cols); else dit_round<1, STAGED, false>(x, tw, m, b, log_cols);
            b += 1;
        }
    }
}
GL_HD void smem_dif(u64* x, const u64* tw, u32 m, u32 log_cols) {
    u32 top = m;   // stages with spans below 2^top remain
    while (top > 0) {
        if (top >= 3 && top != 4) {
            if (top == 3) dif_round<3, true>(x, tw, m, 0, log_cols); else dif_round<3, false>(x, tw, m, top - 3, log_cols);
            top -= 3;
        } else if (top == 4 || top == 2) {
            if (top == 2) dif_round<2, true>(x, tw, m, 0, log_cols); else dif_round<2, false>(x, tw, m, top - 2, log_cols);
            top -= 2;
        } else {
            dif_round<1, true>(x, tw, m, 0, log_cols);    // top == 1
            top -= 1;
        }
    }
}

// ---- compile-time schedules: the split (n1, n2) and the tile shape are template constants -------------------------
// The kernels of the common sizes (NTT_SPECIALISED in kernels.cu, passes of 2^8 .. 2^11) are instantiated from these;
// every shift, mask and table stride of the index arithmetic folds away.  An element touches shared memory only between
// two register rounds: the first round loads its groups from global memory, the last applies the pass's output factor
// and stores to global memory, and the rounds are as wide as the registers allow (a radix-16 group is 16 u64).  The one
// exception is the span-1 side of a contiguous pass (the input of the forward, the output of the inverse): its groups
// are runs of adjacent words, which go through the tile so that the global accesses stay coalesced.
// Log radices of the rounds in the order of their spans, smallest first: the DIT runs them first to last, the DIF last
// to first.  2^8 takes one shared-memory exchange, 2^9 .. 2^11 take two.
GL_HD constexpr int sched_rounds(int m) { return m == 8 ? 2 : 3; }
GL_HD constexpr int sched_radix(int m, int i) { return m == 9 ? 3 : (i < 2 && (m != 10 || i == 0)) ? 4 : 3; }
GL_HD constexpr int sched_span(int m, int i) { return i == 0 ? 0 : sched_span(m, i - 1) + sched_radix(m, i - 1); }
// log2 of the words one thread holds at a time: one group of the widest round (kernels.cu sizes the blocks by it)
GL_HD constexpr int sched_log_elems(int m) { return m == 9 ? 3 : 4; }

// Tile word of element o = (idx << LC) + cc: pad16(o), one pad word every 16 words.  With the rounds above this keeps
// the shared-memory accesses of every round free of bank conflicts at 2^8, 2^10 and 2^11 (one round of 2^9 is 2-way).
template <int LOGR, int B, int LC>
GL_HD void tile_get(u64 (&v)[1 << LOGR], const u64* x, u32 base, u32 cc) {
#pragma unroll
    for (int k = 0; k < (1 << LOGR); k++) v[k] = x[pad16(((base + ((u32)k << B)) << LC) + cc)];
}
template <int LOGR, int B, int LC>
GL_HD void tile_put(u64* x, const u64 (&v)[1 << LOGR], u32 base, u32 cc) {
#pragma unroll
    for (int k = 0; k < (1 << LOGR); k++) x[pad16(((base + ((u32)k << B)) << LC) + cc)] = v[k];
}
// Round I of the compile-time schedule of a [2^M][2^LC] transform (DIT: I = 0, 1, ...; DIF: I = last, ..., 0) and the
// rounds after it.  Group g holds column cc and the elements idx = base + k * 2^B.  The first round reads its group with
// ld(v, base, cc) and then waits for the twiddle table; the last writes it with st(v, base, cc); the others go through
// the padded tile x.  The caller has made a table its threads copied themselves visible with a barrier.
template <bool STAGED, int M, int LC, int I, class Ld, class St>
GL_HD void dit_sched(u64* x, const u64* tw, TableLoad tl, u64* bar, const Ld& ld, const St& st) {
    constexpr int R = sched_radix(M, I), B = sched_span(M, I);
    constexpr bool FIRST = I == 0, LAST = I + 1 == sched_rounds(M);
    NTT2_FOR(g, 1u << (M + LC - R)) {
        const u32 cc = g & ((1u << LC) - 1), gg = g >> LC, lo = gg & ((1u << B) - 1);
        const u32 base = ((gg >> B) << (B + R)) | lo;
        u64 v[1 << R];
        if constexpr (FIRST) { ld(v, base, cc); table_wait(tl, bar); } else tile_get<R, B, LC>(v, x, base, cc);
        dit_bfly<R, STAGED, B == 0 && !STAGED>(v, tw, (u32)M, (u32)B, lo);
        if constexpr (LAST) st(v, base, cc); else tile_put<R, B, LC>(x, v, base, cc);
    }
    if constexpr (!LAST) {
        NTT2_SYNC();
        dit_sched<STAGED, M, LC, I + 1>(x, tw, tl, bar, ld, st);
    }
}
template <int M, int LC, int I, class Ld, class St>
GL_HD void dif_sched(u64* x, const u64* tw, TableLoad tl, u64* bar, const Ld& ld, const St& st) {
    constexpr int R = sched_radix(M, I), B = sched_span(M, I);
    constexpr bool FIRST = I + 1 == sched_rounds(M), LAST = I == 0;
    NTT2_FOR(g, 1u << (M + LC - R)) {
        const u32 cc = g & ((1u << LC) - 1), gg = g >> LC, lo = gg & ((1u << B) - 1);
        const u32 base = ((gg >> B) << (B + R)) | lo;
        u64 v[1 << R];
        if constexpr (FIRST) { ld(v, base, cc); table_wait(tl, bar); } else tile_get<R, B, LC>(v, x, base, cc);
        dif_bfly<R, B == 0>(v, tw, (u32)M, (u32)B, lo);
        if constexpr (LAST) st(v, base, cc); else tile_put<R, B, LC>(x, v, base, cc);
    }
    if constexpr (!LAST) {
        NTT2_SYNC();
        dif_sched<M, LC, I - 1>(x, tw, tl, bar, ld, st);
    }
}

GL_HD u64 w_pow(const u64* hi, const u64* lo, u32 lo_bits, u64 e) {
    return glf::mul(hi[e >> lo_bits], lo[e & ((1ull << lo_bits) - 1)]);
}

// Log width C of the tile of a strided pass: columns of the other factor side by side, C * N1 = 4096 words
template <int N1C, int N2C> GL_HD constexpr int strided_log_c() { return N1C >= 12 ? 0 : (12 - N1C < N2C ? 12 - N1C : N2C); }

// ---- inverse, step 1: strided tile [N1][C] of column `by`, columns j2_0 .. j2_0 + C --------------------
template <int N1C = -1, int N2C = -1>
GL_HD void intt_strided_block(u32 bx, u32 by, u64* sm, u64* cols, size_t col_stride, const mk::NttTables& T, u32 log_c_rt) {
    const u32 n1 = N1C >= 0 ? (u32)N1C : T.n1, n2 = N2C >= 0 ? (u32)N2C : T.n2;
    const u32 log_c = N1C >= 0 && N2C >= 0 ? (u32)strided_log_c<N1C, N2C>() : log_c_rt;
    u32 C = 1u << log_c, N1 = 1u << n1, N2 = 1u << n2;
    u64* x = sm; u64* tw = sm + tw_off(n1, log_c); u64* bar = tw + N1 / 2 + 2;
    u64* col = cols + (size_t)by * col_stride;
    u32 j2_0 = bx * C;
    TableLoad tl = table_load(tw, T.twi_n1, N1 / 2, bar);
    if constexpr (N1C >= 0 && N2C >= 0) {
        constexpr int LC = strided_log_c<N1C, N2C>(), NR = sched_rounds(N1C);
        constexpr int RF = sched_radix(N1C, NR - 1), BF = sched_span(N1C, NR - 1), RL = sched_radix(N1C, 0);
        static_assert(BF + RF == N1C, "the rounds cover the pass");
        if (!tl.async) NTT2_SYNC();
        auto ld = [&](u64 (&v)[1 << RF], u32 base, u32 cc) {
#pragma unroll
            for (int k = 0; k < (1 << RF); k++) v[k] = col[(size_t)(base + ((u32)k << BF)) * N2 + j2_0 + cc];
        };
        // slot p = bitrev(k1) of column j2 leaves multiplied by w_N^(-j2 * k1)
        auto st = [&](u64 (&v)[1 << RL], u32 base, u32 cc) {
            const u32 j2 = j2_0 + cc;
#pragma unroll
            for (int k = 0; k < (1 << RL); k++) {
                const u32 slot = base + (u32)k;
                u64 f = w_pow(T.wi_hi, T.wi_lo, T.lo_bits, (u64)j2 * gl::bitrev32(slot, n1));
                col[(size_t)slot * N2 + j2] = glf::cmul(v[k], f);
            }
        };
        dif_sched<N1C, LC, NR - 1>(x, tw, tl, bar, ld, st);
    } else {
        NTT2_FOR(idx, N1 * C) {
            u32 j1 = idx >> log_c, cc = idx & (C - 1);
            x[tile_off(j1, cc, log_c)] = col[(size_t)j1 * N2 + j2_0 + cc];
        }
        table_wait(tl, bar);
        NTT2_SYNC();
        smem_dif(x, tw, n1, log_c);
        NTT2_FOR(idx, N1 * C) {
            u32 slot = idx >> log_c, cc = idx & (C - 1);
            u32 k1 = gl::bitrev32(slot, n1);
            u32 j2 = j2_0 + cc;
            u64 f = w_pow(T.wi_hi, T.wi_lo, T.lo_bits, (u64)j2 * k1);
            col[(size_t)slot * N2 + j2] = glf::cmul(x[tile_off(slot, cc, log_c)], f);
        }
    }
}
// ---- inverse, step 3 (or the whole transform when n1 == 0): contiguous chunk bx of column by ------------
template <int N2C = -1>
GL_HD void intt_contig_block(u32 bx, u32 by, u64* sm, u64* cols, size_t col_stride, const mk::NttTables& T) {
    const u32 n2 = N2C >= 0 ? (u32)N2C : T.n2;
    u32 N2 = 1u << n2;
    u64* x = sm; u64* tw = sm + tw_off(n2, 0); u64* bar = tw + N2 / 2 + 2;
    u64* chunk = cols + (size_t)by * col_stride + (size_t)bx * N2;
    TableLoad tl = table_load(tw, T.twi_n2, N2 / 2, bar);
    if constexpr (N2C >= 0) {
        constexpr int NR = sched_rounds(N2C), RF = sched_radix(N2C, NR - 1), BF = sched_span(N2C, NR - 1), RL = sched_radix(N2C, 0);
        static_assert(BF + RF == N2C, "the rounds cover the pass");
        if (!tl.async) NTT2_SYNC();
        auto ld = [&](u64 (&v)[1 << RF], u32 base, u32) {
#pragma unroll
            for (int k = 0; k < (1 << RF); k++) v[k] = chunk[base + ((u32)k << BF)];
        };
        // the span-1 round leaves through the tile: stored from registers, a thread's adjacent words would put every
        // 16-byte access of a warp in a different cache line
        auto st = [&](u64 (&v)[1 << RL], u32 base, u32) { tile_put<RL, 0, 0>(x, v, base, 0); };
        dif_sched<N2C, 0, NR - 1>(x, tw, tl, bar, ld, st);
        NTT2_SYNC();
        store_chunk_canon<true>(chunk, x, N2);
    } else {
        load_chunk(x, chunk, N2);
        table_wait(tl, bar);
        NTT2_SYNC();
        smem_dif(x, tw, n2, 0);
        store_chunk_canon(chunk, x, N2);
    }
}
// ---- forward, step 1: contiguous chunk p_hi = bx of work item by, staged coset twiddles ------------------
static constexpr u32 FWD_LANES = 128;   // lanes of the inter-pass twiddle progression (independent of blockDim)
template <int N1C = -1, int N2C = -1>
GL_HD void fwd_contig_block(u32 bx, u32 by, u64* sm, const mk::FwdItem* items, const mk::NttTables& T, const mk::PremulTables& Pm) {
    const u32 n1 = N1C >= 0 ? (u32)N1C : T.n1, n2 = N2C >= 0 ? (u32)N2C : T.n2, n = N1C >= 0 && N2C >= 0 ? (u32)(N1C + N2C) : T.n;
    u32 N1 = 1u << n1, N2 = 1u << n2;
    u64* x = sm; u64* tw = sm + tw_off(n2, 0); u64* bar = tw + N2;
    mk::FwdItem it = items[by];
    u32 p_hi = bx;
    u32 j1 = gl::bitrev32(p_hi, n1);
    const u64* src = it.src + (size_t)p_hi * N2;
    u64* dst = it.dst + (size_t)p_hi * N2;
    u64 fb = Pm.tab_b[(size_t)it.base * N1 + j1];              // g^j1 / N
    const u64* tc = Pm.tab_c + (size_t)it.base * N2;           // staged twiddles of G = g^N1
    TableLoad tl = table_load(tw, tc, N2, bar);              // N2 - 1 staged twiddles + the unused last slot
    if constexpr (N1C >= 0 && N2C >= 0) {
        constexpr int NR = sched_rounds(N2C), RF = sched_radix(N2C, 0), RL = sched_radix(N2C, NR - 1), BL = sched_span(N2C, NR - 1);
        static_assert(BL + RL == N2C, "the rounds cover the pass");
        // the span-1 round starts from the tile, filled by coalesced 16-byte loads (see intt_contig_block); the barrier
        // also covers a table the threads copied themselves
        load_chunk<true>(x, src, N2);
        NTT2_SYNC();
        const u64 mask = ((u64)1 << n) - 1;
        const u64 step = w_pow(T.w_hi, T.w_lo, T.lo_bits, ((u64)j1 << BL) & mask);
        auto ld = [&](u64 (&v)[1 << RF], u32 base, u32) { tile_get<RF, 0, 0>(v, x, base, 0); };
        // dst[k2] = x[k2] * fb * w_N^(j1 * k2); the group's k2 = base + k * 2^BL advance by the factor `step`
        auto st = [&](u64 (&v)[1 << RL], u32 base, u32) {
            u64 f = glf::mul(fb, w_pow(T.w_hi, T.w_lo, T.lo_bits, ((u64)j1 * base) & mask));
#pragma unroll
            for (int k = 0; k < (1 << RL); k++) {
                dst[base + ((u32)k << BL)] = glf::cmul(v[k], f);
                if (k + 1 < (1 << RL)) f = glf::mul(f, step);
            }
        };
        dit_sched<true, N2C, 0, 0>(x, tw, tl, bar, ld, st);
    } else {
        load_chunk(x, src, N2);
        table_wait(tl, bar);
        NTT2_SYNC();
        smem_dit<true>(x, tw, n2, 0);
        // dst[k2] = x[k2] * fb * w_N^(j1 * k2): lane l walks k2 = l, l + LANES, ... multiplying by w_N^(j1 * LANES)
        u32 lanes = N2 < FWD_LANES ? N2 : FWD_LANES;
        NTT2_FOR(l, lanes) {
            u64 f = fb, step = 1;
            if (n1 > 0) {
                u64 mask = ((u64)1 << n) - 1;
                f = glf::mul(fb, w_pow(T.w_hi, T.w_lo, T.lo_bits, ((u64)j1 * l) & mask));
                step = w_pow(T.w_hi, T.w_lo, T.lo_bits, ((u64)j1 * lanes) & mask);
            }
            for (u32 k2 = l; k2 < N2; k2 += lanes) {
                dst[k2] = glf::cmul(x[tile_off(k2, 0, 0)], f);
                if (n1 > 0) f = glf::mul(f, step);
            }
        }
    }
}
// ---- forward, step 3: strided tile [N1][C], DIT along p_hi, in place ----------------------------------------
template <int N1C = -1, int N2C = -1>
GL_HD void fwd_strided_block(u32 bx, u32 by, u64* sm, const mk::FwdItem* items, const mk::NttTables& T, u32 log_c_rt) {
    const u32 n1 = N1C >= 0 ? (u32)N1C : T.n1, n2 = N2C >= 0 ? (u32)N2C : T.n2;
    const u32 log_c = N1C >= 0 && N2C >= 0 ? (u32)strided_log_c<N1C, N2C>() : log_c_rt;
    u32 C = 1u << log_c, N1 = 1u << n1, N2 = 1u << n2;
    u64* x = sm; u64* tw = sm + tw_off(n1, log_c); u64* bar = tw + N1 / 2 + 2;
    u64* col = items[by].dst;
    u32 k2_0 = bx * C;
    TableLoad tl = table_load(tw, T.tw_n1, N1 / 2, bar);
    if constexpr (N1C >= 0 && N2C >= 0) {
        constexpr int LC = strided_log_c<N1C, N2C>(), NR = sched_rounds(N1C), RF = sched_radix(N1C, 0);
        constexpr int RL = sched_radix(N1C, NR - 1), BL = sched_span(N1C, NR - 1);
        static_assert(BL + RL == N1C, "the rounds cover the pass");
        if (!tl.async) NTT2_SYNC();
        auto ld = [&](u64 (&v)[1 << RF], u32 base, u32 cc) {
#pragma unroll
            for (int k = 0; k < (1 << RF); k++) v[k] = col[(size_t)(base + (u32)k) * N2 + k2_0 + cc];
        };
        auto st = [&](u64 (&v)[1 << RL], u32 base, u32 cc) {
#pragma unroll
            for (int k = 0; k < (1 << RL); k++) col[(size_t)(base + ((u32)k << BL)) * N2 + k2_0 + cc] = glf::canon_cc(v[k]);
        };
        dit_sched<false, N1C, LC, 0>(x, tw, tl, bar, ld, st);
    } else {
        NTT2_FOR(idx, N1 * C) {
            u32 p_hi = idx >> log_c, cc = idx & (C - 1);
            x[tile_off(p_hi, cc, log_c)] = col[(size_t)p_hi * N2 + k2_0 + cc];
        }
        table_wait(tl, bar);
        NTT2_SYNC();
        smem_dit<false>(x, tw, n1, log_c);
        NTT2_FOR(idx, N1 * C) {
            u32 k1 = idx >> log_c, cc = idx & (C - 1);
            col[(size_t)k1 * N2 + k2_0 + cc] = glf::canon_cc(x[tile_off(k1, cc, log_c)]);
        }
    }
}

}  // namespace ntt2
