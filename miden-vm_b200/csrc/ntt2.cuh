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

// tile element (idx, cc), idx < 2^m, cc < 2^log_cols; contiguous tiles are padded by one word every 8
GL_HD u32 tile_off(u32 idx, u32 cc, u32 log_cols) {
    u32 o = (idx << log_cols) + cc;
    return log_cols ? o : o + (o >> 3);
}
GL_HD u32 tile_words(u32 m, u32 log_cols) {
    u32 n = 1u << (m + log_cols);
    return log_cols ? n : n + (n >> 3) + 1;
}
// Shared memory of the four block functions: [tile | table (16-byte aligned: it is the destination of a bulk copy) |
// mbarrier].  tw_off = offset of the table in words.
GL_HD u32 tw_off(u32 m, u32 log_cols) { return (tile_words(m, log_cols) + 1u) & ~1u; }
GL_HD size_t smem_words_contig_fwd(u32 n2) { return (size_t)tw_off(n2, 0) + ((size_t)1 << n2) + 2; }
GL_HD size_t smem_words_contig_inv(u32 n2) { return (size_t)tw_off(n2, 0) + ((size_t)1 << n2) / 2 + 4; }
GL_HD size_t smem_words_strided(u32 n1, u32 log_c) { return (size_t)tw_off(n1, log_c) + ((size_t)1 << n1) / 2 + 4; }

// Contiguous chunk <-> padded tile with 128-bit global accesses (two words per thread per access; chunks are 16-byte
// aligned whenever they hold at least two words because every column and chunk length is a power of two).
GL_HD void load_chunk(u64* x, const u64* src, u32 n) {
#if defined(__CUDA_ARCH__)
    if (n >= 2 && (((size_t)src) & 15) == 0) {
        const ulonglong2* s2 = reinterpret_cast<const ulonglong2*>(src);
        NTT2_FOR(i, n / 2) { ulonglong2 v = s2[i]; x[tile_off(2 * i, 0, 0)] = v.x; x[tile_off(2 * i + 1, 0, 0)] = v.y; }
        return;
    }
#endif
    NTT2_FOR(i, n) x[tile_off(i, 0, 0)] = src[i];
}
GL_HD void store_chunk_canon(u64* dst, const u64* x, u32 n) {
#if defined(__CUDA_ARCH__)
    if (n >= 2 && (((size_t)dst) & 15) == 0) {
        ulonglong2* d2 = reinterpret_cast<ulonglong2*>(dst);
        NTT2_FOR(i, n / 2) d2[i] = make_ulonglong2(glf::canon_cc(x[tile_off(2 * i, 0, 0)]), glf::canon_cc(x[tile_off(2 * i + 1, 0, 0)]));
        return;
    }
#endif
    NTT2_FOR(i, n) dst[i] = glf::canon_cc(x[tile_off(i, 0, 0)]);
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
template <int LOGR, bool STAGED, bool UNIT0>
GL_HD void dit_group(u64* x, const u64* tw, u32 m, u32 b, u32 log_cols, u32 g) {
    constexpr int R = 1 << LOGR;
    u32 cc = g & ((1u << log_cols) - 1), gg = g >> log_cols;
    u32 lo = gg & ((1u << b) - 1), hi = gg >> b;
    u32 base = (hi << (b + LOGR)) | lo;
    u64 v[R];
#pragma unroll
    for (int k = 0; k < R; k++) v[k] = x[tile_off(base + ((u32)k << b), cc, log_cols)];
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
#pragma unroll
    for (int k = 0; k < R; k++) x[tile_off(base + ((u32)k << b), cc, log_cols)] = v[k];
}
// DIF (natural -> bit-reversed) stages with spans 2^(b+LOGR-1) .. 2^b on the plain table.
// UNIT0: b == 0, so the twiddle with j == 0 is 1.
template <int LOGR, bool UNIT0>
GL_HD void dif_group(u64* x, const u64* tw, u32 m, u32 b, u32 log_cols, u32 g) {
    constexpr int R = 1 << LOGR;
    u32 cc = g & ((1u << log_cols) - 1), gg = g >> log_cols;
    u32 lo = gg & ((1u << b) - 1), hi = gg >> b;
    u32 base = (hi << (b + LOGR)) | lo;
    u64 v[R];
#pragma unroll
    for (int k = 0; k < R; k++) v[k] = x[tile_off(base + ((u32)k << b), cc, log_cols)];
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

// The same two schedules with the transform size and the tile shape as compile-time constants: every shift, mask and
// table stride of the index arithmetic folds away (ncu r2b: a quarter of the executed instructions of the passes were
// LEA / SHF / IMAD address arithmetic on run-time m, b, log_cols).  The kernels of the common sizes are instantiated
// from these (kernels.cu); other sizes keep the run-time schedules above.  Same rounds, same order, same results.
template <bool STAGED, int M, int LC, int B = 0>
GL_HD void smem_dit_t(u64* x, const u64* tw) {
    if constexpr (B < M) {
        constexpr int left = M - B;
        constexpr int R = (left >= 3 && left != 4) ? 3 : ((left == 4 || left == 2) ? 2 : 1);
        dit_round<R, STAGED, (B == 0) && !STAGED>(x, tw, (u32)M, (u32)B, (u32)LC);
        smem_dit_t<STAGED, M, LC, B + R>(x, tw);
    }
}
template <int M, int LC, int TOP = M>
GL_HD void smem_dif_t(u64* x, const u64* tw) {
    if constexpr (TOP > 0) {
        constexpr int R = (TOP >= 3 && TOP != 4) ? 3 : ((TOP == 4 || TOP == 2) ? 2 : 1);
        dif_round<R, (TOP - R) == 0>(x, tw, (u32)M, (u32)(TOP - R), (u32)LC);
        smem_dif_t<M, LC, TOP - R>(x, tw);
    }
}

GL_HD u64 w_pow(const u64* hi, const u64* lo, u32 lo_bits, u64 e) {
    return glf::mul(hi[e >> lo_bits], lo[e & ((1ull << lo_bits) - 1)]);
}

// ---- inverse, step 1: strided tile [N1][C] of column `by`, columns j2_0 .. j2_0 + C --------------------
template <int N1C = -1, int N2C = -1>
GL_HD void intt_strided_block(u32 bx, u32 by, u64* sm, u64* cols, size_t col_stride, const mk::NttTables& T, u32 log_c_rt) {
    const u32 n1 = N1C >= 0 ? (u32)N1C : T.n1, n2 = N2C >= 0 ? (u32)N2C : T.n2;
    const u32 log_c = N1C >= 0 && N2C >= 0 ? (u32)(N1C >= 12 ? 0 : (12 - N1C < N2C ? 12 - N1C : N2C)) : log_c_rt;
    u32 C = 1u << log_c, N1 = 1u << n1, N2 = 1u << n2;
    u64* x = sm; u64* tw = sm + tw_off(n1, log_c); u64* bar = tw + N1 / 2 + 2;
    u64* col = cols + (size_t)by * col_stride;
    u32 j2_0 = bx * C;
    TableLoad tl = table_load(tw, T.twi_n1, N1 / 2, bar);
    NTT2_FOR(idx, N1 * C) {
        u32 j1 = idx >> log_c, cc = idx & (C - 1);
        x[tile_off(j1, cc, log_c)] = col[(size_t)j1 * N2 + j2_0 + cc];
    }
    table_wait(tl, bar);
    NTT2_SYNC();
    if constexpr (N1C >= 0 && N2C >= 0) smem_dif_t<N1C, (N1C >= 12 ? 0 : (12 - N1C < N2C ? 12 - N1C : N2C))>(x, tw);
    else smem_dif(x, tw, n1, log_c);
    NTT2_FOR(idx, N1 * C) {
        u32 slot = idx >> log_c, cc = idx & (C - 1);
        u32 k1 = gl::bitrev32(slot, n1);
        u32 j2 = j2_0 + cc;
        u64 f = w_pow(T.wi_hi, T.wi_lo, T.lo_bits, (u64)j2 * k1);
        col[(size_t)slot * N2 + j2] = glf::cmul(x[tile_off(slot, cc, log_c)], f);
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
    load_chunk(x, chunk, N2);
    table_wait(tl, bar);
    NTT2_SYNC();
    if constexpr (N2C >= 0) smem_dif_t<N2C, 0>(x, tw); else smem_dif(x, tw, n2, 0);
    store_chunk_canon(chunk, x, N2);
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
    load_chunk(x, src, N2);
    table_wait(tl, bar);
    NTT2_SYNC();
    if constexpr (N2C >= 0) smem_dit_t<true, N2C, 0>(x, tw); else smem_dit<true>(x, tw, n2, 0);
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
// ---- forward, step 3: strided tile [N1][C], DIT along p_hi, in place ----------------------------------------
template <int N1C = -1, int N2C = -1>
GL_HD void fwd_strided_block(u32 bx, u32 by, u64* sm, const mk::FwdItem* items, const mk::NttTables& T, u32 log_c_rt) {
    const u32 n1 = N1C >= 0 ? (u32)N1C : T.n1, n2 = N2C >= 0 ? (u32)N2C : T.n2;
    const u32 log_c = N1C >= 0 && N2C >= 0 ? (u32)(N1C >= 12 ? 0 : (12 - N1C < N2C ? 12 - N1C : N2C)) : log_c_rt;
    u32 C = 1u << log_c, N1 = 1u << n1, N2 = 1u << n2;
    u64* x = sm; u64* tw = sm + tw_off(n1, log_c); u64* bar = tw + N1 / 2 + 2;
    u64* col = items[by].dst;
    u32 k2_0 = bx * C;
    TableLoad tl = table_load(tw, T.tw_n1, N1 / 2, bar);
    NTT2_FOR(idx, N1 * C) {
        u32 p_hi = idx >> log_c, cc = idx & (C - 1);
        x[tile_off(p_hi, cc, log_c)] = col[(size_t)p_hi * N2 + k2_0 + cc];
    }
    table_wait(tl, bar);
    NTT2_SYNC();
    if constexpr (N1C >= 0 && N2C >= 0) smem_dit_t<false, N1C, (N1C >= 12 ? 0 : (12 - N1C < N2C ? 12 - N1C : N2C))>(x, tw);
    else smem_dit<false>(x, tw, n1, log_c);
    NTT2_FOR(idx, N1 * C) {
        u32 k1 = idx >> log_c, cc = idx & (C - 1);
        col[(size_t)k1 * N2 + k2_0 + cc] = glf::canon_cc(x[tile_off(k1, cc, log_c)]);
    }
}

}  // namespace ntt2
