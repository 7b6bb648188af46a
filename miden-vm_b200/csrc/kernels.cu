// sm_90a (H100) kernels of the Miden STARK proving path.  See kernels.cuh for the data layout and
// DESIGN.md for the roofline of each kernel.  All arithmetic is 64-bit modular integer work
// (Goldilocks); the hot loops are (a) NTT butterflies through shared memory, (b) Poseidon2
// permutations held entirely in registers, (c) streaming reductions over LDE columns.
#include "kernels.cuh"
#include "poseidon2.cuh"
#include "poseidon2_fast2.cuh"    // host-checked by tests/cpp/test_arith_v2.cpp
#include "ntt2.cuh"               // host-checked by tests/cpp/test_ntt_v2.cpp
#include "blake3.cuh"
#include "keccak.cuh"
#include "rescue.cuh"
#include <algorithm>
#include <cstdio>

namespace mk {

static unsigned long long g_launches = 0;
unsigned long long launch_count() { return g_launches; }
void count_launch() { ++g_launches; }
void reset_launch_count() { g_launches = 0; }
#define COUNT_LAUNCH() (++g_launches)

void upload_constants() {
    cudaMemcpyToSymbol(p2::D_RC_EXT_INITIAL, p2::P2_RC_EXT_INITIAL, sizeof(u64) * 48);
    cudaMemcpyToSymbol(p2::D_RC_INTERNAL, p2::P2_RC_INTERNAL, sizeof(u64) * 22);
    cudaMemcpyToSymbol(p2::D_RC_EXT_TERMINAL, p2::P2_RC_EXT_TERMINAL, sizeof(u64) * 48);
    cudaMemcpyToSymbol(rsc::D_ARK1, rsc::RESCUE_ARK1, sizeof(u64) * 84);
    cudaMemcpyToSymbol(rsc::D_ARK2, rsc::RESCUE_ARK2, sizeof(u64) * 84);
}

// =============================================================================================
// Peer memory: pushes and the cross-GPU barrier (kernels.cuh "One proof on G GPUs")
// =============================================================================================
#ifdef MDN_EMULATED
static inline void st_release_sys(u64* p, u64 v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
static inline u64 ld_acquire_sys(const u64* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
static constexpr long long BARRIER_TIMEOUT = 600ll * 1000000000ll;   // emulated clock64() counts nanoseconds
#else
__device__ __forceinline__ void st_release_sys(u64* p, u64 v) { asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ u64 ld_acquire_sys(const u64* p) { u64 v; asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }
static constexpr long long BARRIER_TIMEOUT = 30000000000ll;          // ~15 s of SM clocks
#endif
// 16-byte store of element `idx` (in ulonglong2 units) to the destination(s) a PushDst selects
__device__ __forceinline__ void push_u2(const PushDst& d, size_t idx, size_t owner_key, ulonglong2 v) {
    if (d.mode == PUSH_ALL) {
        for (u32 g = 0; g < d.world; g++) reinterpret_cast<ulonglong2*>(d.pp.p[g])[idx] = v;
    } else {
        u32 g = d.mode == PUSH_OWNER ? (u32)(owner_key >> d.owner_shift) : d.rank;
        reinterpret_cast<ulonglong2*>(d.pp.p[g])[idx] = v;
    }
}
struct BarrierArgs { PeerPtrs flags; u32 rank, world; u64 epoch; u32* err; };
__global__ void k_barrier(BarrierArgs a) {
    u32 p = threadIdx.x;
    // every store of the kernels before this one on the stream (local and peer) is ordered before the signal
    if (p < a.world) { __threadfence_system(); st_release_sys(a.flags.p[p] + a.rank, a.epoch); }
    __syncthreads();
    if (p < a.world) {
        long long t0 = clock64();
        while (ld_acquire_sys(a.flags.p[a.rank] + p) < a.epoch) {
            if (clock64() - t0 > BARRIER_TIMEOUT) { atomicOr(a.err, 8u); break; }
#ifdef MDN_EMULATED
            emu::cpu_relax();
#endif
        }
    }
}
void launch_barrier(const PeerPtrs& flags, u32 rank, u32 world, u64 epoch, u32* err, cudaStream_t st) {
    BarrierArgs a; a.flags = flags; a.rank = rank; a.world = world; a.epoch = epoch; a.err = err;
    k_barrier<<<1, 32, 0, st>>>(a);
    COUNT_LAUNCH();
}
struct PushArgs { const u64* src; PeerPtrs dst; u32 rank, world; size_t n; };
__global__ void __launch_bounds__(256) k_push(PushArgs a) {
    size_t stride = (size_t)gridDim.x * blockDim.x, i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if ((a.n & 1) == 0 && (((size_t)a.src) & 15) == 0) {      // symmetric offsets: the peers' views share the alignment
        const ulonglong2* s2 = reinterpret_cast<const ulonglong2*>(a.src);
        for (size_t i = i0; i < a.n / 2; i += stride) {
            ulonglong2 v = s2[i];
            for (u32 g = 0; g < a.world; g++) if (g != a.rank) reinterpret_cast<ulonglong2*>(a.dst.p[g])[i] = v;
        }
    } else {
        for (size_t i = i0; i < a.n; i += stride) {
            u64 v = a.src[i];
            for (u32 g = 0; g < a.world; g++) if (g != a.rank) a.dst.p[g][i] = v;
        }
    }
}
void launch_push(const u64* src, const PeerPtrs& dst, u32 rank, u32 world, size_t n, cudaStream_t st) {
    if (!n || world <= 1) return;
    PushArgs a; a.src = src; a.dst = dst; a.rank = rank; a.world = world; a.n = n;
    unsigned blocks = (unsigned)std::min<size_t>((n / 2 + 255) / 256 + 1, 132 * 8);     // 8 blocks on each of the H100's 132 SMs
    k_push<<<blocks, 256, 0, st>>>(a);
    COUNT_LAUNCH();
}

// =============================================================================================
// transpose: row-major (n_rows x width) -> column-major
// =============================================================================================
// Rows [row0, row0 + n_rows) of a row-major matrix (src points at row row0) -> columns of height col_stride; the
// destination is one buffer (world == 1) or the same buffer on every rank (a proof split over ranks uploads a
// different row range on every rank and stores the transposed slice into all of them).
struct TransposeDst { PeerPtrs dst; PeerPtrs bad; u32 world; };
__global__ void k_transpose(const u64* __restrict__ src, TransposeDst d, u32 n_rows, u32 width, size_t col_stride, u32 row0) {
    __shared__ u64 tile[32][33];
    u32 r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    bool any_bad = false;
    for (u32 i = threadIdx.y; i < 32; i += 8) {
        u32 r = r0 + i, c = c0 + threadIdx.x;
        if (r < n_rows && c < width) {
            u64 v = src[(size_t)r * width + c];
            any_bad |= (v >= gl::P);        // Felt values are canonical by construction in the reference
            tile[i][threadIdx.x] = v;
        }
    }
    if (any_bad) for (u32 g = 0; g < d.world; g++) if (d.bad.p[g]) atomicOr(reinterpret_cast<u32*>(d.bad.p[g]), 1u);
    __syncthreads();
    for (u32 i = threadIdx.y; i < 32; i += 8) {
        u32 c = c0 + i, r = r0 + threadIdx.x;
        if (r < n_rows && c < width) {
            u64 v = tile[threadIdx.x][i];
            size_t o = (size_t)c * col_stride + row0 + r;
            for (u32 g = 0; g < d.world; g++) d.dst.p[g][o] = v;
        }
    }
}
void launch_transpose_rm_to_cm(const u64* src, u64* dst, u32 n_rows, u32 width, u32* d_bad_flag, cudaStream_t st) {
    TransposeDst d{}; d.dst.p[0] = dst; d.bad.p[0] = reinterpret_cast<u64*>(d_bad_flag); d.world = 1;
    dim3 grid((n_rows + 31) / 32, (width + 31) / 32), block(32, 8);
    k_transpose<<<grid, block, 0, st>>>(src, d, n_rows, width, (size_t)n_rows, 0u);
    COUNT_LAUNCH();
}
void launch_transpose_slice_push(const u64* src_slice, const PeerPtrs& dst_cm, const PeerPtrs& bad, u32 world, u32 row0, u32 n_rows_slice,
                                 u32 n_rows_total, u32 width, cudaStream_t st) {
    if (!n_rows_slice || !width) return;
    TransposeDst d{}; d.dst = dst_cm; d.bad = bad; d.world = world;
    dim3 grid((n_rows_slice + 31) / 32, (width + 31) / 32), block(32, 8);
    k_transpose<<<grid, block, 0, st>>>(src_slice, d, n_rows_slice, width, (size_t)n_rows_total, row0);
    COUNT_LAUNCH();
}

// =============================================================================================
// column-major ingest: a caller's device matrix (column c at c*N) -> its slot of a coefficient buffer
// =============================================================================================
// The layouts already agree, so this is a copy with the canonical check of k_transpose.  src == dst only checks (the
// columns a device aux builder wrote into their slot) and stores nothing.  The caller's base pointer is 16-byte aligned;
// a slot that follows a one-row matrix of odd width is not, and takes the scalar loop.
__global__ void __launch_bounds__(256) k_ingest_cm(const u64* __restrict__ src, u64* __restrict__ dst, size_t n, u32* bad) {
    const bool store = src != dst;
    size_t stride = (size_t)gridDim.x * blockDim.x, i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool any_bad = false;
    if (((((size_t)src) | ((size_t)dst)) & 15) == 0) {
        const ulonglong2* s2 = reinterpret_cast<const ulonglong2*>(src);
        ulonglong2* d2 = reinterpret_cast<ulonglong2*>(dst);
        for (size_t i = i0; i < n / 2; i += stride) {
            ulonglong2 v = s2[i];
            any_bad |= (v.x >= gl::P) | (v.y >= gl::P);
            if (store) d2[i] = v;
        }
        if ((n & 1) && i0 == 0) {          // N = 1 with an odd width
            u64 v = src[n - 1];
            any_bad |= v >= gl::P;
            if (store) dst[n - 1] = v;
        }
    } else {
        for (size_t i = i0; i < n; i += stride) {
            u64 v = src[i];
            any_bad |= v >= gl::P;
            if (store) dst[i] = v;
        }
    }
    if (any_bad) atomicOr(bad, 1u);
}
void launch_ingest_cm(const u64* src_cm, u64* dst_cm, size_t n, u32* d_bad_flag, cudaStream_t st) {
    if (!n) return;
    unsigned blocks = (unsigned)std::min<size_t>((n / 2 + 255) / 256 + 1, 132 * 8);     // 8 blocks on each of the H100's 132 SMs
    k_ingest_cm<<<blocks, 256, 0, st>>>(src_cm, dst_cm, n, d_bad_flag);
    COUNT_LAUNCH();
}

// =============================================================================================
// NTT.  N = N1 * N2.  Index conventions (see DESIGN.md "NTT"):
//   inverse (DIF): natural j = j1*N2 + j2  ->  slot p = bitrev(k1)*N2 + bitrev(k2), k = k1 + N1*k2
//   forward (DIT): slot p = p_hi*N2 + p_lo holds c[j], j = bitrev(p_lo)*N1 + bitrev(p_hi)
//                  ->  natural k = k1*N2 + k2
// =============================================================================================
static constexpr int NTT_THREADS = 256;
// One group of the widest register round per thread when possible: 2^log_elems words (radix 8 in the run-time schedules,
// ntt2::sched_log_elems in the compile-time ones, so that no thread idles in the round that holds the most registers).
static inline unsigned ntt_threads(u32 m, u32 log_cols, u32 log_elems) {
    u32 g = (m + log_cols >= log_elems) ? (1u << (m + log_cols - log_elems)) : 1u;
    if (g < 32) g = 32;
    if (g > 256) g = 256;
    return g;
}

__device__ __forceinline__ u64 w_pow(const u64* __restrict__ hi, const u64* __restrict__ lo, u32 lo_bits, u64 e) {
    return gl::mul(hi[e >> lo_bits], lo[e & ((1ull << lo_bits) - 1)]);
}

// ptxas chooses the register count (no minimum-resident-blocks bound)
#define NTT_BOUNDS __launch_bounds__(NTT_THREADS)
// Kernels are instantiated with the split (n1, n2) as compile-time constants for the trace heights that matter
// (2^16 .. 2^22: NTT_SPECIALISED below) and once with run-time sizes (<-1, -1>) for everything else.
template <int N1C, int N2C>
__global__ void NTT_BOUNDS k_intt_strided(u64* cols, size_t col_stride, NttTables T, u32 log_c) {
    extern __shared__ u64 sm[];
    ntt2::intt_strided_block<N1C, N2C>(blockIdx.x, blockIdx.y, sm, cols, col_stride, T, log_c);
}
template <int N2C>
__global__ void NTT_BOUNDS k_intt_contig(u64* cols, size_t col_stride, NttTables T) {
    extern __shared__ u64 sm[];
    ntt2::intt_contig_block<N2C>(blockIdx.x, blockIdx.y, sm, cols, col_stride, T);
}
template <int N1C, int N2C>
__global__ void NTT_BOUNDS k_fwd_contig(const FwdItem* __restrict__ items, NttTables T, PremulTables Pm) {
    extern __shared__ u64 sm[];
    ntt2::fwd_contig_block<N1C, N2C>(blockIdx.x, blockIdx.y, sm, items, T, Pm);
}
template <int N1C, int N2C>
__global__ void NTT_BOUNDS k_fwd_strided(const FwdItem* __restrict__ items, NttTables T, u32 log_c) {
    extern __shared__ u64 sm[];
    ntt2::fwd_strided_block<N1C, N2C>(blockIdx.x, blockIdx.y, sm, items, T, log_c);
}
// X(n1, n2) for every specialised split: split_n() of heights 16 .. 22
#define NTT_SPECIALISED(X) X(8, 8) X(8, 9) X(9, 9) X(9, 10) X(10, 10) X(10, 11) X(11, 11)

template <int N1C, int N2C>
static void launch_intt_t(u64* cols, size_t col_stride, u32 n_cols, const NttTables& T, u32 log_c, cudaStream_t st) {
    u32 N1 = 1u << T.n1, N2 = 1u << T.n2, C = 1u << log_c;
    constexpr u32 LOG_E1 = N1C >= 0 ? ntt2::sched_log_elems(N1C) : 3, LOG_E2 = N2C >= 0 ? ntt2::sched_log_elems(N2C) : 3;
    if (T.n1 > 0) {
        size_t smem = ntt2::smem_words_strided(T.n1, log_c) * sizeof(u64);
        cudaFuncSetAttribute(k_intt_strided<N1C, N2C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        k_intt_strided<N1C, N2C><<<dim3(N2 / C, n_cols), ntt_threads(T.n1, log_c, LOG_E1), smem, st>>>(cols, col_stride, T, log_c);
        COUNT_LAUNCH();
    }
    size_t smem = ntt2::smem_words_contig_inv(T.n2) * sizeof(u64);
    k_intt_contig<N2C><<<dim3(N1, n_cols), ntt_threads(T.n2, 0, LOG_E2), smem, st>>>(cols, col_stride, T);
    COUNT_LAUNCH();
}
void launch_intt(u64* cols, size_t col_stride, u32 n_cols, const NttTables& T, cudaStream_t st) {
    u32 log_c = T.n1 >= 12 ? 0 : 12 - T.n1; if (log_c > T.n2) log_c = T.n2;
#define X(a, b) if (T.n1 == a && T.n2 == b) { launch_intt_t<a, b>(cols, col_stride, n_cols, T, log_c, st); return; }
    NTT_SPECIALISED(X)
#undef X
    launch_intt_t<-1, -1>(cols, col_stride, n_cols, T, log_c, st);
}
template <int N1C, int N2C>
static void launch_fwd_t(const FwdItem* d_items, u32 n_items, const NttTables& T, const PremulTables& Pm, u32 log_c, cudaStream_t st) {
    u32 N1 = 1u << T.n1, N2 = 1u << T.n2, C = 1u << log_c;
    constexpr u32 LOG_E1 = N1C >= 0 ? ntt2::sched_log_elems(N1C) : 3, LOG_E2 = N2C >= 0 ? ntt2::sched_log_elems(N2C) : 3;
    size_t smem = ntt2::smem_words_contig_fwd(T.n2) * sizeof(u64);
    k_fwd_contig<N1C, N2C><<<dim3(N1, n_items), ntt_threads(T.n2, 0, LOG_E2), smem, st>>>(d_items, T, Pm);
    COUNT_LAUNCH();
    if (T.n1 > 0) {
        size_t smem2 = ntt2::smem_words_strided(T.n1, log_c) * sizeof(u64);
        cudaFuncSetAttribute(k_fwd_strided<N1C, N2C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2);
        k_fwd_strided<N1C, N2C><<<dim3(N2 / C, n_items), ntt_threads(T.n1, log_c, LOG_E1), smem2, st>>>(d_items, T, log_c);
        COUNT_LAUNCH();
    }
}
void launch_fwd_ntt(const FwdItem* d_items, u32 n_items, const NttTables& T, const PremulTables& Pm, cudaStream_t st) {
    u32 log_c = T.n1 >= 12 ? 0 : 12 - T.n1; if (log_c > T.n2) log_c = T.n2;
#define X(a, b) if (T.n1 == a && T.n2 == b) { launch_fwd_t<a, b>(d_items, n_items, T, Pm, log_c, st); return; }
    NTT_SPECIALISED(X)
#undef X
    launch_fwd_t<-1, -1>(d_items, n_items, T, Pm, log_c, st);
}

// =============================================================================================
// Poseidon2 hashing
// =============================================================================================
static constexpr int HASH_THREADS = 128;
// Minimum resident blocks the compiler must allow: the kernels are bound by the two integer pipes and more warps per
// scheduler interleave their FMA and ALU bursts.  For sm_90a ptxas gives the Poseidon2 kernels about 62 registers
// without the bound (8 blocks per SM), under the cap of any value up to 8.
static constexpr int HASH_MIN_BLOCKS = 6;

// The permutation of the algebraic configurations (air/src/config.rs:225-273: one LMCS / challenger type, generic in P):
// PERM_P2 = Poseidon2 (the metric's; lazy representatives, canonicalised on store), PERM_RPO / PERM_RPX = rescue.cuh (canonical in,
// canonical out; functional coverage of `rpo_config` / `rpx_config`, ~9x / ~5x the field multiplications of Poseidon2).
enum { PERM_P2 = 0, PERM_RPO = 3, PERM_RPX = 4 };     // = mdn_hash_kind
template <int PERM>
__device__ __forceinline__ void alg_permute(u64* s) {
    if constexpr (PERM == PERM_RPO) rsc::rpo_permute(s);
    else if constexpr (PERM == PERM_RPX) rsc::rpx_permute(s);
    else p2f::permute(s);
}
#define ALG_BOUNDS(PERM) __launch_bounds__(HASH_THREADS, (PERM) == PERM_P2 ? HASH_MIN_BLOCKS : 1)
#define ALG_DISPATCH(perm, CALL) do { if ((perm) == PERM_RPO) { CALL(PERM_RPO); } else if ((perm) == PERM_RPX) { CALL(PERM_RPX); } else { CALL(PERM_P2); } } while (0)

template <int PERM>
__global__ void ALG_BOUNDS(PERM) k_leaf_hash(LeafArgs a, u32 log_n, u32 log_b, const u64* __restrict__ prev,
                                                            u32 prev_log_n, u64* __restrict__ states_out,
                                                            PushDst dig, u32 has_dig, u32 t0, u32 nt) {
    // all rows of cosets t0 .. t0 + nt (the whole tree when t0 = 0, nt = B; this rank's cosets when one proof is
    // split over several GPUs): a contiguous slab [t0 * N, (t0 + nt) * N) of every LDE column
    size_t L = (size_t)1 << (log_n + log_b);
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= ((size_t)nt << log_n)) return;
    u32 t = t0 + (u32)(idx >> log_n);
    u32 r = (u32)(idx & (((size_t)1 << log_n) - 1));
    size_t pos = ((size_t)t << log_n) + r;
    u64 s[12];
    if (prev) {
        size_t Lp = (size_t)1 << (prev_log_n + log_b);
        size_t pp = ((size_t)t << prev_log_n) + (r & ((1u << prev_log_n) - 1));
#pragma unroll
        for (int k = 0; k < 12; k++) s[k] = prev[k * Lp + pp];
    } else {
#pragma unroll
        for (int k = 0; k < 12; k++) s[k] = 0;
    }
    for (int m = 0; m < a.n_mats; m++) {
        const u64* base = a.m[m].base + pos;
        u32 w = a.m[m].width;
        for (u32 c0 = 0; c0 < w; c0 += 8) {
#pragma unroll
            for (u32 k = 0; k < 8; k++) s[k] = (c0 + k < w) ? base[(size_t)(c0 + k) * L] : 0ull;
            alg_permute<PERM>(s);
        }
    }
    if (states_out) {
#pragma unroll
        for (int k = 0; k < 12; k++) states_out[k * L + pos] = glf::canon(s[k]);
    }
    if (has_dig) {
        size_t i = ((size_t)r << log_b) | t;       // Merkle leaf = domain index
        push_u2(dig, 2 * i, i, make_ulonglong2(glf::canon(s[0]), glf::canon(s[1])));
        push_u2(dig, 2 * i + 1, i, make_ulonglong2(glf::canon(s[2]), glf::canon(s[3])));
    }
}
template <int PERM>
static void launch_leaf_hash_t(const LeafArgs& a, u32 log_n, u32 log_blowup, const u64* prev_states, u32 prev_log_n,
                               u64* states_out, const PushDst* dig, u32 t0, u32 nt, cudaStream_t st) {
    size_t cnt = (size_t)nt << log_n;
    unsigned blocks = (unsigned)((cnt + HASH_THREADS - 1) / HASH_THREADS);
    PushDst d = dig ? *dig : local_dst(nullptr);
    k_leaf_hash<PERM><<<blocks, HASH_THREADS, 0, st>>>(a, log_n, log_blowup, prev_states, prev_log_n, states_out, d, dig ? 1u : 0u, t0, nt);
    COUNT_LAUNCH();
}
void launch_leaf_hash(const LeafArgs& a, u32 log_n, u32 log_blowup, const u64* prev_states, u32 prev_log_n,
                      u64* states_out, const PushDst* dig, u32 t0, u32 nt, cudaStream_t st, int perm) {
#define X(PM) launch_leaf_hash_t<PM>(a, log_n, log_blowup, prev_states, prev_log_n, states_out, dig, t0, nt, st)
    ALG_DISPATCH(perm, X);
#undef X
}

template <int PERM>
__global__ void ALG_BOUNDS(PERM) k_compress(const u64* __restrict__ ch, u64* __restrict__ par, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const ulonglong2* c = reinterpret_cast<const ulonglong2*>(ch + i * 8);
    ulonglong2 a0 = c[0], a1 = c[1], b0 = c[2], b1 = c[3];
    u64 s[12] = {a0.x, a0.y, a1.x, a1.y, b0.x, b0.y, b1.x, b1.y, 0, 0, 0, 0};
    alg_permute<PERM>(s);
    ulonglong2* d = reinterpret_cast<ulonglong2*>(par + i * 4);
    d[0] = make_ulonglong2(glf::canon(s[0]), glf::canon(s[1]));
    d[1] = make_ulonglong2(glf::canon(s[2]), glf::canon(s[3]));
}
template <int PERM>
static void launch_compress_layer_t(const u64* children, u64* parents, size_t n_parents, cudaStream_t st) {
    unsigned blocks = (unsigned)((n_parents + HASH_THREADS - 1) / HASH_THREADS);
    k_compress<PERM><<<blocks, HASH_THREADS, 0, st>>>(children, parents, n_parents);
    COUNT_LAUNCH();
}
void launch_compress_layer(const u64* children, u64* parents, size_t n_parents, cudaStream_t st, int perm) {
#define X(PM) launch_compress_layer_t<PM>(children, parents, n_parents, st)
    ALG_DISPATCH(perm, X);
#undef X
}

// FRI round leaf: physical row of 2^la extension values [f[i + bitrev_la(j) * q]]_j (fri/prover.rs:137-165),
// flattened to 2 * 2^la felts and absorbed with the rate-8 sponge (unaligned tree).
template <int PERM>
__global__ void __launch_bounds__(HASH_THREADS) k_fri_leaf(const u64* __restrict__ ev, size_t q, u32 la, PushDst dig, u32 log_b, u32 t0, u32 log_nt) {
    // thread -> leaf i with (i mod B) in [t0, t0 + nt): the leaves whose 2^la values (stride q, a multiple of B) this rank holds
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= ((q >> log_b) << log_nt)) return;
    size_t i = ((idx >> log_nt) << log_b) | (t0 + (idx & ((1u << log_nt) - 1)));
    const ulonglong2* e = reinterpret_cast<const ulonglong2*>(ev);
    u64 s[12];
#pragma unroll
    for (int k = 0; k < 12; k++) s[k] = 0;
    u32 a = 1u << la;
    for (u32 j0 = 0; j0 < a; j0 += 4) {
#pragma unroll
        for (u32 j = 0; j < 4; j++) {
            if (j0 + j < a) {
                ulonglong2 v = e[i + (size_t)gl::bitrev32(j0 + j, la) * q];
                s[2 * j] = v.x; s[2 * j + 1] = v.y;
            } else { s[2 * j] = 0; s[2 * j + 1] = 0; }
        }
        alg_permute<PERM>(s);
    }
    push_u2(dig, 2 * i, i, make_ulonglong2(glf::canon(s[0]), glf::canon(s[1])));
    push_u2(dig, 2 * i + 1, i, make_ulonglong2(glf::canon(s[2]), glf::canon(s[3])));
}
static inline u32 log2_exact(u32 v) { u32 l = 0; while ((1u << l) < v) l++; return l; }
template <int PERM>
static void launch_fri_leaf_hash_t(const u64* evals, size_t rows, u32 log_arity, const PushDst& digests, u32 log_b, u32 t0, u32 nt, cudaStream_t st) {
    if (rows < ((size_t)1 << log_b)) { log_b = 0; t0 = 0; nt = 1; }      // tiny layers are never split
    size_t cnt = (rows >> log_b) * nt;
    unsigned blocks = (unsigned)((cnt + HASH_THREADS - 1) / HASH_THREADS);
    k_fri_leaf<PERM><<<blocks, HASH_THREADS, 0, st>>>(evals, rows, log_arity, digests, log_b, t0, log2_exact(nt));
    COUNT_LAUNCH();
}
void launch_fri_leaf_hash(const u64* evals, size_t rows, u32 log_arity, const PushDst& digests, u32 log_b, u32 t0, u32 nt, cudaStream_t st, int perm) {
#define X(PM) launch_fri_leaf_hash_t<PM>(evals, rows, log_arity, digests, log_b, t0, nt, st)
    ALG_DISPATCH(perm, X);
#undef X
}

__global__ void k_p2_batch(u64* st, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    u64 s[12];
#pragma unroll
    for (int k = 0; k < 12; k++) s[k] = st[i * 12 + k];
    p2f::permute(s);
#pragma unroll
    for (int k = 0; k < 12; k++) st[i * 12 + k] = glf::canon(s[k]);
}
void launch_poseidon2_batch(u64* states, size_t n, cudaStream_t st) {
    k_p2_batch<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(states, n);
    COUNT_LAUNCH();
}

// =============================================================================================
// BLAKE3 hashing: the reference's `HashFunction::Blake3_256` configuration (air/src/config.rs:276-307).
//   leaf   : ChainingHasher -- state (32 bytes, zero at the start) <- blake3(state || little-endian u64 of every felt
//            of the row), once per matrix in ascending height, states duplicated between heights exactly like the
//            sponge states (crates/stateful-hasher/src/chaining.rs:31-52; lmcs/lifted_tree.rs:363-417)
//   node   : blake3(left || right), one compression (CompressionFunctionFromHasher<Blake3, 2, 32>)
//   digest : 32 bytes = the four u64 slots of every tree, little-endian
// Same launch geometry, coset ranges and peer-store destinations as the Poseidon2 kernels above.
// =============================================================================================
__global__ void __launch_bounds__(HASH_THREADS) k_leaf_hash_b3(LeafArgs a, u32 log_n, u32 log_b, const u64* __restrict__ prev, u32 prev_log_n,
                                                               u64* __restrict__ states_out, PushDst dig, u32 has_dig, u32 t0, u32 nt) {
    size_t L = (size_t)1 << (log_n + log_b);
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= ((size_t)nt << log_n)) return;
    u32 t = t0 + (u32)(idx >> log_n);
    u32 r = (u32)(idx & (((size_t)1 << log_n) - 1));
    size_t pos = ((size_t)t << log_n) + r;
    u64 st[4] = {0, 0, 0, 0};
    if (prev) {
        size_t Lp = (size_t)1 << (prev_log_n + log_b);
        size_t pp = ((size_t)t << prev_log_n) + (r & ((1u << prev_log_n) - 1));
#pragma unroll
        for (int k = 0; k < 4; k++) st[k] = prev[k * Lp + pp];
    }
    for (int m = 0; m < a.n_mats; m++) {
        const u64* base = a.m[m].base + pos;
        u32 w = a.m[m].width;
        b3::Hasher h; h.init();
#pragma unroll
        for (int k = 0; k < 4; k++) h.push64(st[k]);
        for (u32 c = 0; c < w; c++) h.push64(base[(size_t)c * L]);     // LDE values are canonical
        u32 o[8];
        h.finish(o);
        b3::words_to_u64(o, st);
    }
    if (states_out) {
#pragma unroll
        for (int k = 0; k < 4; k++) states_out[k * L + pos] = st[k];
    }
    if (has_dig) {
        size_t i = ((size_t)r << log_b) | t;
        push_u2(dig, 2 * i, i, make_ulonglong2(st[0], st[1]));
        push_u2(dig, 2 * i + 1, i, make_ulonglong2(st[2], st[3]));
    }
}
void launch_leaf_hash_b3(const LeafArgs& a, u32 log_n, u32 log_blowup, const u64* prev_states, u32 prev_log_n,
                         u64* states_out, const PushDst* dig, u32 t0, u32 nt, cudaStream_t st) {
    size_t cnt = (size_t)nt << log_n;
    unsigned blocks = (unsigned)((cnt + HASH_THREADS - 1) / HASH_THREADS);
    PushDst d = dig ? *dig : local_dst(nullptr);
    k_leaf_hash_b3<<<blocks, HASH_THREADS, 0, st>>>(a, log_n, log_blowup, prev_states, prev_log_n, states_out, d, dig ? 1u : 0u, t0, nt);
    COUNT_LAUNCH();
}
__global__ void __launch_bounds__(256) k_compress_b3(const u64* __restrict__ ch, u64* __restrict__ par, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const ulonglong2* c = reinterpret_cast<const ulonglong2*>(ch + i * 8);
    ulonglong2 a0 = c[0], a1 = c[1], b0 = c[2], b1 = c[3];
    u64 l[4] = {a0.x, a0.y, a1.x, a1.y}, r[4] = {b0.x, b0.y, b1.x, b1.y}, o[4];
    b3::compress2(l, r, o);
    ulonglong2* d = reinterpret_cast<ulonglong2*>(par + i * 4);
    d[0] = make_ulonglong2(o[0], o[1]);
    d[1] = make_ulonglong2(o[2], o[3]);
}
void launch_compress_layer_b3(const u64* children, u64* parents, size_t n_parents, cudaStream_t st) {
    k_compress_b3<<<(unsigned)((n_parents + 255) / 256), 256, 0, st>>>(children, parents, n_parents);
    COUNT_LAUNCH();
}
// FRI round leaf (fri/prover.rs:137-165): blake3(zero state || the row's 2^la extension values as 2 * 2^la little-endian u64)
__global__ void __launch_bounds__(256) k_fri_leaf_b3(const u64* __restrict__ ev, size_t q, u32 la, PushDst dig, u32 log_b, u32 t0, u32 log_nt) {
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= ((q >> log_b) << log_nt)) return;
    size_t i = ((idx >> log_nt) << log_b) | (t0 + (idx & ((1u << log_nt) - 1)));
    const ulonglong2* e = reinterpret_cast<const ulonglong2*>(ev);
    b3::Hasher h; h.init();
    for (int k = 0; k < 4; k++) h.push64(0);
    u32 a = 1u << la;
    for (u32 j = 0; j < a; j++) {
        ulonglong2 v = e[i + (size_t)gl::bitrev32(j, la) * q];
        h.push64(v.x); h.push64(v.y);
    }
    u32 o[8]; u64 d[4];
    h.finish(o);
    b3::words_to_u64(o, d);
    push_u2(dig, 2 * i, i, make_ulonglong2(d[0], d[1]));
    push_u2(dig, 2 * i + 1, i, make_ulonglong2(d[2], d[3]));
}
void launch_fri_leaf_hash_b3(const u64* evals, size_t rows, u32 log_arity, const PushDst& digests, u32 log_b, u32 t0, u32 nt, cudaStream_t st) {
    if (rows < ((size_t)1 << log_b)) { log_b = 0; t0 = 0; nt = 1; }
    size_t cnt = (rows >> log_b) * nt;
    k_fri_leaf_b3<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(evals, rows, log_arity, digests, log_b, t0, log2_exact(nt));
    COUNT_LAUNCH();
}
// Proof-of-work for the hash challenger: smallest w such that, after observing w (8 little-endian bytes) on top of the
// `n_words` 32-bit words of the challenger's input buffer, the low `bits` bits of the first sampled u64 are zero.  The
// HashChallenger samples bytes from the BACK of the 32-byte output: u64::from_le_bytes([out[31], out[30], ..., out[24]]).
__global__ void __launch_bounds__(128) k_grind_b3(const u32* __restrict__ input, u32 n_words, u64 mask, u64 start, u64 count, u64* result) {
    u64 idx = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    u64 w = start + idx;
    b3::Hasher h; h.init();
    for (u32 i = 0; i < n_words; i++) h.push(input[i]);
    h.push64(w);
    u32 o[8];
    h.finish(o);
    u64 v = (u64)b3::bswap(o[7]) | ((u64)b3::bswap(o[6]) << 32);   // bytes 31..24 of the output become bytes 0..7
    if ((v & mask) == 0) atomicMin(reinterpret_cast<unsigned long long*>(result), (unsigned long long)w);
}
void launch_grind_b3(const u32* d_input_words, u32 n_words, u32 bits, u64 start, u64 count, u64* d_result, cudaStream_t st) {
    u64 mask = (1ull << bits) - 1;
    k_grind_b3<<<(unsigned)((count + 127) / 128), 128, 0, st>>>(d_input_words, n_words, mask, start, count, d_result);
    COUNT_LAUNCH();
}

// =============================================================================================
// Keccak hashing: the reference's `HashFunction::Keccak` configuration (air/src/config.rs:309-353).
//   leaf   : the same overwrite-mode stateful sponge as Poseidon2 (crates/stateful-hasher/src/field_sponge.rs:41-59) over 25 u64
//            lanes with rate 17, fed the canonical u64 of every felt (serializing_sponge.rs:72-86); alignment 17
//   node   : PaddingFreeSponge<KeccakF, 25, 17, 4> on the 8 words of two digests -- one permutation
//   digest : lanes 0..4 = the four u64 slots of every tree
// 25 lanes of state travel between height groups (SoA [25][B << log_n]).  Bit-wise work on the ALU pipe only: nothing of the
// Goldilocks multiplier is involved, so these kernels are an independent load on the SM from the NTT / constraint kernels.
// =============================================================================================
__global__ void __launch_bounds__(HASH_THREADS) k_leaf_hash_kk(LeafArgs a, u32 log_n, u32 log_b, const u64* __restrict__ prev, u32 prev_log_n,
                                                               u64* __restrict__ states_out, PushDst dig, u32 has_dig, u32 t0, u32 nt) {
    size_t L = (size_t)1 << (log_n + log_b);
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= ((size_t)nt << log_n)) return;
    u32 t = t0 + (u32)(idx >> log_n);
    u32 r = (u32)(idx & (((size_t)1 << log_n) - 1));
    size_t pos = ((size_t)t << log_n) + r;
    u64 st[25];
    if (prev) {
        size_t Lp = (size_t)1 << (prev_log_n + log_b);
        size_t pp = ((size_t)t << prev_log_n) + (r & ((1u << prev_log_n) - 1));
#pragma unroll
        for (int k = 0; k < 25; k++) st[k] = prev[k * Lp + pp];
    } else {
#pragma unroll
        for (int k = 0; k < 25; k++) st[k] = 0;
    }
    for (int m = 0; m < a.n_mats; m++) {
        const u64* base = a.m[m].base + pos;
        u32 w = a.m[m].width;
        for (u32 c0 = 0; c0 < w; c0 += 17) {
#pragma unroll
            for (u32 k = 0; k < 17; k++) st[k] = (c0 + k < w) ? base[(size_t)(c0 + k) * L] : 0ull;     // LDE values are canonical
            kk::permute(st);
        }
    }
    if (states_out) {
#pragma unroll
        for (int k = 0; k < 25; k++) states_out[k * L + pos] = st[k];
    }
    if (has_dig) {
        size_t i = ((size_t)r << log_b) | t;
        push_u2(dig, 2 * i, i, make_ulonglong2(st[0], st[1]));
        push_u2(dig, 2 * i + 1, i, make_ulonglong2(st[2], st[3]));
    }
}
void launch_leaf_hash_kk(const LeafArgs& a, u32 log_n, u32 log_blowup, const u64* prev_states, u32 prev_log_n,
                         u64* states_out, const PushDst* dig, u32 t0, u32 nt, cudaStream_t st) {
    size_t cnt = (size_t)nt << log_n;
    unsigned blocks = (unsigned)((cnt + HASH_THREADS - 1) / HASH_THREADS);
    PushDst d = dig ? *dig : local_dst(nullptr);
    k_leaf_hash_kk<<<blocks, HASH_THREADS, 0, st>>>(a, log_n, log_blowup, prev_states, prev_log_n, states_out, d, dig ? 1u : 0u, t0, nt);
    COUNT_LAUNCH();
}
__global__ void __launch_bounds__(128) k_compress_kk(const u64* __restrict__ ch, u64* __restrict__ par, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const ulonglong2* c = reinterpret_cast<const ulonglong2*>(ch + i * 8);
    ulonglong2 a0 = c[0], a1 = c[1], b0 = c[2], b1 = c[3];
    u64 l[4] = {a0.x, a0.y, a1.x, a1.y}, r[4] = {b0.x, b0.y, b1.x, b1.y}, o[4];
    kk::compress2(l, r, o);
    ulonglong2* d = reinterpret_cast<ulonglong2*>(par + i * 4);
    d[0] = make_ulonglong2(o[0], o[1]);
    d[1] = make_ulonglong2(o[2], o[3]);
}
void launch_compress_layer_kk(const u64* children, u64* parents, size_t n_parents, cudaStream_t st) {
    k_compress_kk<<<(unsigned)((n_parents + 127) / 128), 128, 0, st>>>(children, parents, n_parents);
    COUNT_LAUNCH();
}
// FRI round leaf (fri/prover.rs:137-165): the sponge from the zero state over the row's 2^la extension values (2 * 2^la lanes)
__global__ void __launch_bounds__(128) k_fri_leaf_kk(const u64* __restrict__ ev, size_t q, u32 la, PushDst dig, u32 log_b, u32 t0, u32 log_nt) {
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= ((q >> log_b) << log_nt)) return;
    size_t i = ((idx >> log_nt) << log_b) | (t0 + (idx & ((1u << log_nt) - 1)));
    const ulonglong2* e = reinterpret_cast<const ulonglong2*>(ev);
    u64 st[25];
#pragma unroll
    for (int k = 0; k < 25; k++) st[k] = 0;
    u32 n = 2u << la;                       // lanes in the row (4, 8 or 16: one chunk of the rate)
#pragma unroll
    for (u32 j = 0; j < 8; j++) {
        if (2 * j < n) {
            ulonglong2 v = e[i + (size_t)gl::bitrev32(j, la) * q];
            st[2 * j] = v.x; st[2 * j + 1] = v.y;
        }
    }
    kk::permute(st);
    push_u2(dig, 2 * i, i, make_ulonglong2(st[0], st[1]));
    push_u2(dig, 2 * i + 1, i, make_ulonglong2(st[2], st[3]));
}
void launch_fri_leaf_hash_kk(const u64* evals, size_t rows, u32 log_arity, const PushDst& digests, u32 log_b, u32 t0, u32 nt, cudaStream_t st) {
    if (rows < ((size_t)1 << log_b)) { log_b = 0; t0 = 0; nt = 1; }
    size_t cnt = (rows >> log_b) * nt;
    k_fri_leaf_kk<<<(unsigned)((cnt + 127) / 128), 128, 0, st>>>(evals, rows, log_arity, digests, log_b, t0, log2_exact(nt));
    COUNT_LAUNCH();
}
// Proof-of-work for the Keccak-256 hash challenger: like k_grind_b3, over whole 64-bit words of the input buffer; the first
// sampled u64 is u64::from_le_bytes([out[31], ..., out[24]]) = lane 3 of the output with its bytes reversed.
__global__ void __launch_bounds__(128) k_grind_kk(const u64* __restrict__ input, u32 n_words, u64 mask, u64 start, u64 count, u64* result) {
    u64 idx = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    u64 w = start + idx;
    kk::Hash256 h; h.init();
    for (u32 i = 0; i < n_words; i++) h.push64(input[i]);
    h.push64(w);
    u64 o[4];
    h.finish(o);
    u64 v = ((u64)b3::bswap((u32)o[3]) << 32) | (u64)b3::bswap((u32)(o[3] >> 32));
    if ((v & mask) == 0) atomicMin(reinterpret_cast<unsigned long long*>(result), (unsigned long long)w);
}
void launch_grind_kk(const u64* d_input_words, u32 n_words, u32 bits, u64 start, u64 count, u64* d_result, cudaStream_t st) {
    u64 mask = (1ull << bits) - 1;
    k_grind_kk<<<(unsigned)((count + 127) / 128), 128, 0, st>>>(d_input_words, n_words, mask, start, count, d_result);
    COUNT_LAUNCH();
}

// =============================================================================================
// The small layers of a Merkle (sub-)tree in ONE block: layers d_from-1 ... lg of the sub-tree of `rank` (2^(d - lg) nodes of
// layer d, starting at node rank << (d - lg); the whole tree with lg = 0, rank = 0).  A layer with fewer nodes than the GPU has
// threads costs one permutation latency plus a launch when it is its own kernel; here consecutive layers are separated by a
// block barrier only (the block's own global stores are visible to it after __syncthreads()).  HK = mdn_hash_kind.
// =============================================================================================
template <int HK>
__device__ __forceinline__ void compress_pair(const u64* l, const u64* r, u64* o) {
    if constexpr (HK == 1) b3::compress2(l, r, o);
    else if constexpr (HK == 2) kk::compress2(l, r, o);
    else {
        u64 s[12] = {l[0], l[1], l[2], l[3], r[0], r[1], r[2], r[3], 0, 0, 0, 0};
        alg_permute<HK>(s);
#pragma unroll
        for (int k = 0; k < 4; k++) o[k] = glf::canon(s[k]);
    }
}
template <int HK>
__global__ void __launch_bounds__(256) k_compress_top(u64* tree, u32 d_from, u32 lg, u32 rank) {
    for (u32 d = d_from; d-- > lg;) {
        const u32 cnt = 1u << (d - lg);
        const size_t start = (size_t)rank << (d - lg);
        const u64* child = tree + (((size_t)2 << d) - 1) * 4;      // layer d + 1
        u64* par = tree + (((size_t)1 << d) - 1) * 4;
        for (u32 i = threadIdx.x; i < cnt; i += blockDim.x) {
            const size_t node = start + i;
            const ulonglong2* c = reinterpret_cast<const ulonglong2*>(child + node * 8);
            ulonglong2 a0 = c[0], a1 = c[1], b0 = c[2], b1 = c[3];
            u64 l[4] = {a0.x, a0.y, a1.x, a1.y}, r[4] = {b0.x, b0.y, b1.x, b1.y}, o[4];
            compress_pair<HK>(l, r, o);
            ulonglong2* dst = reinterpret_cast<ulonglong2*>(par + node * 4);
            dst[0] = make_ulonglong2(o[0], o[1]);
            dst[1] = make_ulonglong2(o[2], o[3]);
        }
        __syncthreads();
    }
}
template <int HK>
static void launch_compress_top_t(u64* tree, u32 d_from, u32 lg, u32 rank, cudaStream_t st) {
    k_compress_top<HK><<<1, 256, 0, st>>>(tree, d_from, lg, rank);
    COUNT_LAUNCH();
}
void launch_compress_top(u64* tree, u32 d_from, u32 lg, u32 rank, int hash_kind, cudaStream_t st) {
    if (d_from <= lg) return;
    switch (hash_kind) {
        case 1: launch_compress_top_t<1>(tree, d_from, lg, rank, st); break;
        case 2: launch_compress_top_t<2>(tree, d_from, lg, rank, st); break;
        case 3: launch_compress_top_t<3>(tree, d_from, lg, rank, st); break;
        case 4: launch_compress_top_t<4>(tree, d_from, lg, rank, st); break;
        default: launch_compress_top_t<0>(tree, d_from, lg, rank, st); break;
    }
}

// =============================================================================================
// Constraint evaluation (op-list interpreter) + quotient accumulation
// =============================================================================================
struct ConstraintKArgs {
    const u64* main_lde; const u64* aux_lde; const u64* prep_lde;
    u32 log_n, log_b;
    AirDev air;
    const u64* publics; const u64* challenges; const u64* aux_values;
    E2 alpha, beta;
    const u64* acc_in; u32 acc_in_log_n;
    u64* acc_out;
    const u64* w_hi; const u64* w_lo; u32 lo_bits;   // w_N powers
    u64 shift, w_l, w_h_inv;                          // LDE shift, w_L, w_H^-1
    u64 zh[16], inv_zh[16];                           // per coset t
    u32 t0, nt;                                       // cosets [t0, t0 + nt)
};

template <int MAXS>
__global__ void __launch_bounds__(128) k_constraints(ConstraintKArgs a) {
    size_t L = (size_t)1 << (a.log_n + a.log_b);
    size_t pos = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= ((size_t)a.nt << a.log_n)) return;
    pos += (size_t)a.t0 << a.log_n;
    u32 N = 1u << a.log_n;
    u32 t = (u32)(pos >> a.log_n), r = (u32)(pos & (N - 1));
    size_t pos_next = ((size_t)t << a.log_n) + ((r + 1) & (N - 1));
    E2 is_first = gl::e2(0, 0), is_last = is_first, is_trans = is_first;
    if (a.air.uses_selectors) {
        u64 x = gl::mul(gl::mul(a.shift, gl::pow(a.w_l, t)), w_pow(a.w_hi, a.w_lo, a.lo_bits, r));
        u64 d_first = gl::sub(x, 1), d_last = gl::sub(x, a.w_h_inv);
        u64 inv = gl::inv(gl::mul(d_first, d_last));    // x is never in H on the LDE coset
        is_first.a = gl::mul(a.zh[t], gl::mul(inv, d_last));
        is_last.a = gl::mul(a.zh[t], gl::mul(inv, d_first));
        is_trans.a = d_last;
    }
    size_t per_idx = ((size_t)(r & ((1u << a.air.log_max_period) - 1)) << a.log_b) | t;
    size_t per_stride = (size_t)1 << (a.air.log_max_period + a.log_b);
    E2 slot[MAXS];
    E2 acc = gl::e2(0, 0);
    const uint4* code = reinterpret_cast<const uint4*>(a.air.code);
    for (u32 i = 0; i < a.air.n_instr; i++) {
        uint4 ins = code[i];
        u32 op = ins.x & 0xff, ext = ins.x >> 8, x = ins.z, y = ins.w;
        E2 v;
        switch (op) {
            case 0: v = gl::e2(a.main_lde[(size_t)y * L + (x ? pos_next : pos)], 0); break;
            case 1: { size_t p = x ? pos_next : pos; v = gl::e2(a.aux_lde[(size_t)(2 * y) * L + p], a.aux_lde[(size_t)(2 * y + 1) * L + p]); break; }
            case 2: v = gl::e2(a.publics[x], 0); break;
            case 3: v = gl::e2(a.challenges[2 * x], a.challenges[2 * x + 1]); break;
            case 4: v = gl::e2(a.aux_values[2 * x], a.aux_values[2 * x + 1]); break;
            case 5: v = is_first; break;
            case 6: v = is_last; break;
            case 7: v = is_trans; break;
            case 8: v = gl::e2(a.air.consts[x], 0); break;
            case 9: v = gl::e2(a.air.consts[x], a.air.consts[x + 1]); break;
            case 10: v = ext ? gl::e2_add(slot[x], slot[y]) : gl::e2(gl::add(slot[x].a, slot[y].a), 0); break;
            case 11: v = ext ? gl::e2_sub(slot[x], slot[y]) : gl::e2(gl::sub(slot[x].a, slot[y].a), 0); break;
            case 12: v = ext ? gl::e2_mul(slot[x], slot[y]) : gl::e2(gl::mul(slot[x].a, slot[y].a), 0); break;
            case 13: v = ext ? gl::e2_neg(slot[x]) : gl::e2(gl::neg(slot[x].a), 0); break;
            case 14: v = gl::e2(a.air.periodic[x * per_stride + per_idx], 0); break;
            case 16: v = gl::e2(a.prep_lde[(size_t)y * L + (x ? pos_next : pos)], 0); break;
            default: acc = gl::e2_add(gl::e2_mul(acc, a.alpha), slot[x]); continue;
        }
        slot[ins.y] = v;
    }
    E2 q = gl::e2_mulf(acc, a.inv_zh[t]);
    if (a.acc_in) {
        size_t Lin = (size_t)1 << (a.acc_in_log_n + a.log_b);
        size_t pa = ((size_t)t << a.acc_in_log_n) + (r & ((1u << a.acc_in_log_n) - 1));
        E2 prev = gl::e2(a.acc_in[pa], a.acc_in[Lin + pa]);
        q = gl::e2_add(gl::e2_mul(prev, a.beta), q);
    }
    a.acc_out[pos] = q.a;
    a.acc_out[L + pos] = q.b;
}

int launch_constraints(const ConstraintArgs& a, cudaStream_t st) {
    ConstraintKArgs k;
    k.main_lde = a.main_lde; k.aux_lde = a.aux_lde; k.prep_lde = a.prep_lde; k.log_n = a.log_n; k.log_b = a.log_blowup; k.air = a.air;
    k.publics = a.publics; k.challenges = a.challenges; k.aux_values = a.aux_values;
    k.alpha = a.alpha; k.beta = a.beta; k.acc_in = a.acc_in; k.acc_in_log_n = a.acc_in_log_n; k.acc_out = a.acc_out;
    k.w_hi = a.T->w_hi; k.w_lo = a.T->w_lo; k.lo_bits = a.T->lo_bits;
    u32 log_lde = a.log_n + a.log_blowup;
    k.shift = gl::lde_shift(log_lde);
    k.w_l = gl::two_adic_generator(log_lde);
    k.w_h_inv = gl::inv(gl::two_adic_generator(a.log_n));
    u32 B = 1u << a.log_blowup;
    if (B > 16) return -1;
    // Z_H(x) on coset t: s^N * w_B^t - 1   (domain.rs:742-749)
    u64 s_pow_n = gl::exp_pow2(k.shift, a.log_n), w_b = gl::two_adic_generator(a.log_blowup), x = 1;
    for (u32 t = 0; t < B; t++) { k.zh[t] = gl::sub(gl::mul(s_pow_n, x), 1); k.inv_zh[t] = gl::inv(k.zh[t]); x = gl::mul(x, w_b); }
    k.t0 = a.nt ? a.t0 : 0; k.nt = a.nt ? a.nt : B;
    size_t cnt = (size_t)k.nt << a.log_n;
    unsigned blocks = (unsigned)((cnt + 127) / 128);
    if (a.air.n_slots <= 16) k_constraints<16><<<blocks, 128, 0, st>>>(k);
    else if (a.air.n_slots <= 64) k_constraints<64><<<blocks, 128, 0, st>>>(k);
    else if (a.air.n_slots <= 256) k_constraints<256><<<blocks, 128, 0, st>>>(k);
    else if (a.air.n_slots <= 1024) k_constraints<1024><<<blocks, 128, 0, st>>>(k);
    else return -1;
    COUNT_LAUNCH();
    return 0;
}

// =============================================================================================
// LogUp aux trace (trace-domain interpreter + EF scan)
// =============================================================================================
template <int MAXS>
__global__ void __launch_bounds__(128) k_logup_rows(LogupArgs a) {
    size_t N = (size_t)1 << a.log_n;
    size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N) return;
    size_t rn = (r + 1) & (N - 1);
    size_t per_row = (r & (((size_t)1 << a.prog.log_max_period) - 1)) * a.prog.n_periodic;
    E2 slot[MAXS];
    E2 V[LOGUP_MAX_COLS], U[LOGUP_MAX_COLS];
    for (u32 c = 0; c < a.n_cols; c++) { V[c] = gl::e2(0, 0); U[c] = gl::e2(1, 0); }
    const uint4* code = reinterpret_cast<const uint4*>(a.prog.code);
    for (u32 i = 0; i < a.prog.n_instr; i++) {
        uint4 ins = code[i];
        u32 op = ins.x & 0xff, ext = ins.x >> 8, x = ins.z, y = ins.w;
        E2 v;
        switch (op) {
            case 0: v = gl::e2(a.main_cm[(size_t)y * N + (x ? rn : r)], 0); break;
            case 2: v = gl::e2(a.publics[x], 0); break;
            case 3: v = gl::e2(a.challenges[2 * x], a.challenges[2 * x + 1]); break;
            case 8: v = gl::e2(a.prog.consts[x], 0); break;
            case 9: v = gl::e2(a.prog.consts[x], a.prog.consts[x + 1]); break;
            case 10: v = ext ? gl::e2_add(slot[x], slot[y]) : gl::e2(gl::add(slot[x].a, slot[y].a), 0); break;
            case 11: v = ext ? gl::e2_sub(slot[x], slot[y]) : gl::e2(gl::sub(slot[x].a, slot[y].a), 0); break;
            case 12: v = ext ? gl::e2_mul(slot[x], slot[y]) : gl::e2(gl::mul(slot[x].a, slot[y].a), 0); break;
            case 13: v = ext ? gl::e2_neg(slot[x]) : gl::e2(gl::neg(slot[x].a), 0); break;
            case 14: v = gl::e2(a.prog.periodic[per_row + x], 0); break;
            default: {   // 17 EMIT
                u32 c = ins.y, fs = x & 0xffffu, ms = x >> 16;
                if (fs != 0xffffu && slot[fs].a == 0) continue;          // prover.rs:357: flag == 0 skips the push
                E2 d = slot[y];
                if (d.a == 0 && d.b == 0) { *a.bad_flag = 2; continue; }
                u64 m = slot[ms].a;
                V[c] = gl::e2_add(gl::e2_mul(V[c], d), gl::e2_mulf(U[c], m));
                U[c] = gl::e2_mul(U[c], d);
                continue;
            }
        }
        slot[ins.y] = v;
    }
    E2 t = gl::e2(0, 0);
    for (u32 c = 0; c < a.n_cols; c++) {
        E2 f = V[c];
        if (!(U[c].a == 1 && U[c].b == 0)) f = gl::e2_mul(V[c], gl::e2_inv(U[c]));
        t = gl::e2_add(t, f);
        if (c > 0) { a.aux_cm[(size_t)(2 * c) * N + r] = f.a; a.aux_cm[(size_t)(2 * c + 1) * N + r] = f.b; }
    }
    reinterpret_cast<ulonglong2*>(a.totals)[r] = make_ulonglong2(t.a, t.b);
}
int launch_logup_rows(const LogupArgs& a, cudaStream_t st) {
    if (a.n_cols == 0 || a.n_cols > LOGUP_MAX_COLS) return -1;
    size_t N = (size_t)1 << a.log_n;
    unsigned blocks = (unsigned)((N + 127) / 128);
    if (a.prog.n_slots <= 16) k_logup_rows<16><<<blocks, 128, 0, st>>>(a);
    else if (a.prog.n_slots <= 64) k_logup_rows<64><<<blocks, 128, 0, st>>>(a);
    else if (a.prog.n_slots <= 256) k_logup_rows<256><<<blocks, 128, 0, st>>>(a);
    else if (a.prog.n_slots <= 1024) k_logup_rows<1024><<<blocks, 128, 0, st>>>(a);
    else return -1;
    COUNT_LAUNCH();
    return 0;
}

// =============================================================================================
// Constraint check on the trace domain (debug.rs check_constraints): the constraint program of k_constraints, read
// on raw rows with exact 0/1 selectors; FOLD k tests constraint k instead of folding it
// =============================================================================================
template <int MAXS>
__global__ void __launch_bounds__(128) k_check_rows(CheckArgs a) {
    size_t N = (size_t)1 << a.log_n;
    size_t r = a.row0 + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.row0 + a.n_rows) return;
    size_t rn = (r + 1) & (N - 1);
    E2 is_first = gl::e2(r == 0, 0), is_last = gl::e2(r == N - 1, 0), is_trans = gl::e2(r != N - 1, 0);
    size_t per_row = (r & (((size_t)1 << a.prog.log_max_period) - 1)) * a.prog.n_periodic;
    E2 slot[MAXS];
    u32 k = 0, first_k = 0xFFFFFFFFu;
    const uint4* code = reinterpret_cast<const uint4*>(a.prog.code);
    for (u32 i = 0; i < a.prog.n_instr; i++) {
        uint4 ins = code[i];
        u32 op = ins.x & 0xff, ext = ins.x >> 8, x = ins.z, y = ins.w;
        E2 v;
        switch (op) {
            case 0: v = gl::e2(a.main_cm[(size_t)y * N + (x ? rn : r)], 0); break;
            case 1: { size_t p = x ? rn : r; v = gl::e2(a.aux_cm[(size_t)(2 * y) * N + p], a.aux_cm[(size_t)(2 * y + 1) * N + p]); break; }
            case 2: v = gl::e2(a.publics[x], 0); break;
            case 3: v = gl::e2(a.challenges[2 * x], a.challenges[2 * x + 1]); break;
            case 4: v = gl::e2(a.aux_values[2 * x], a.aux_values[2 * x + 1]); break;
            case 5: v = is_first; break;
            case 6: v = is_last; break;
            case 7: v = is_trans; break;
            case 8: v = gl::e2(a.prog.consts[x], 0); break;
            case 9: v = gl::e2(a.prog.consts[x], a.prog.consts[x + 1]); break;
            case 10: v = ext ? gl::e2_add(slot[x], slot[y]) : gl::e2(gl::add(slot[x].a, slot[y].a), 0); break;
            case 11: v = ext ? gl::e2_sub(slot[x], slot[y]) : gl::e2(gl::sub(slot[x].a, slot[y].a), 0); break;
            case 12: v = ext ? gl::e2_mul(slot[x], slot[y]) : gl::e2(gl::mul(slot[x].a, slot[y].a), 0); break;
            case 13: v = ext ? gl::e2_neg(slot[x]) : gl::e2(gl::neg(slot[x].a), 0); break;
            case 14: v = gl::e2(a.prog.periodic[per_row + x], 0); break;
            case 16: v = gl::e2(a.prep_cm[(size_t)y * N + (x ? rn : r)], 0); break;
            default: {   // 15: the compiler places the k-th FOLD for constraint k (emission order)
                E2 c = slot[x];
                if (a.probe_value && k == a.probe_k) { a.probe_value[0] = c.a; a.probe_value[1] = c.b; }
                if ((c.a | c.b) != 0 && first_k == 0xFFFFFFFFu) first_k = k;
                k++;
                continue;
            }
        }
        slot[ins.y] = v;
    }
    if (first_k != 0xFFFFFFFFu) {
        atomicMin(a.first, (unsigned long long)(((u64)r << 32) | first_k));
        atomicAdd(a.failing_rows, 1ull);
    }
}
int launch_check_rows(const CheckArgs& a, cudaStream_t st) {
    if (a.n_rows == 0) return 0;
    unsigned blocks = (unsigned)((a.n_rows + 127) / 128);
    if (a.prog.n_slots <= 16) k_check_rows<16><<<blocks, 128, 0, st>>>(a);
    else if (a.prog.n_slots <= 64) k_check_rows<64><<<blocks, 128, 0, st>>>(a);
    else if (a.prog.n_slots <= 256) k_check_rows<256><<<blocks, 128, 0, st>>>(a);
    else if (a.prog.n_slots <= 1024) k_check_rows<1024><<<blocks, 128, 0, st>>>(a);
    else return -1;
    COUNT_LAUNCH();
    return 0;
}

// three-phase scan, 2048 rows per block (8 per thread): block totals -> serial scan of the (<= 2048) block
// totals by one block -> per-block exclusive prefix with the block offset
static constexpr int SCAN_T = 256, SCAN_E = 8, SCAN_B = SCAN_T * SCAN_E;
__device__ __forceinline__ E2 ld_e2(const u64* p, size_t i) { ulonglong2 v = reinterpret_cast<const ulonglong2*>(p)[i]; return gl::e2(v.x, v.y); }
__global__ void __launch_bounds__(SCAN_T) k_scan_block_totals(const u64* __restrict__ totals, size_t n, u64* __restrict__ block_sums) {
    __shared__ u64 sh[2 * SCAN_T];
    size_t base = (size_t)blockIdx.x * SCAN_B + (size_t)threadIdx.x * SCAN_E;
    E2 s = gl::e2(0, 0);
    for (int e = 0; e < SCAN_E; e++) if (base + e < n) s = gl::e2_add(s, ld_e2(totals, base + e));
    sh[2 * threadIdx.x] = s.a; sh[2 * threadIdx.x + 1] = s.b;
    __syncthreads();
    for (int off = SCAN_T / 2; off > 0; off >>= 1) {
        if (threadIdx.x < off) {
            sh[2 * threadIdx.x] = gl::add(sh[2 * threadIdx.x], sh[2 * (threadIdx.x + off)]);
            sh[2 * threadIdx.x + 1] = gl::add(sh[2 * threadIdx.x + 1], sh[2 * (threadIdx.x + off) + 1]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) { block_sums[2 * blockIdx.x] = sh[0]; block_sums[2 * blockIdx.x + 1] = sh[1]; }
}
__global__ void k_scan_block_sums(u64* block_sums, size_t n_blocks, u64* final2) {
    if (threadIdx.x || blockIdx.x) return;
    E2 acc = gl::e2(0, 0);
    for (size_t b = 0; b < n_blocks; b++) {
        E2 v = gl::e2(block_sums[2 * b], block_sums[2 * b + 1]);
        block_sums[2 * b] = acc.a; block_sums[2 * b + 1] = acc.b;
        acc = gl::e2_add(acc, v);
    }
    final2[0] = acc.a; final2[1] = acc.b;
}
__global__ void __launch_bounds__(SCAN_T) k_scan_apply(const u64* __restrict__ totals, size_t n, const u64* __restrict__ block_sums,
                                                       u64* __restrict__ acc0, u64* __restrict__ acc1) {
    __shared__ u64 sh[2 * SCAN_T];
    size_t base = (size_t)blockIdx.x * SCAN_B + (size_t)threadIdx.x * SCAN_E;
    E2 v[SCAN_E];
    E2 s = gl::e2(0, 0);
    for (int e = 0; e < SCAN_E; e++) { v[e] = base + e < n ? ld_e2(totals, base + e) : gl::e2(0, 0); s = gl::e2_add(s, v[e]); }
    sh[2 * threadIdx.x] = s.a; sh[2 * threadIdx.x + 1] = s.b;
    __syncthreads();
    // Hillis-Steele inclusive scan of the per-thread sums
    for (int off = 1; off < SCAN_T; off <<= 1) {
        u64 a0 = 0, a1 = 0;
        if ((int)threadIdx.x >= off) { a0 = sh[2 * (threadIdx.x - off)]; a1 = sh[2 * (threadIdx.x - off) + 1]; }
        __syncthreads();
        if ((int)threadIdx.x >= off) { sh[2 * threadIdx.x] = gl::add(sh[2 * threadIdx.x], a0); sh[2 * threadIdx.x + 1] = gl::add(sh[2 * threadIdx.x + 1], a1); }
        __syncthreads();
    }
    E2 run = gl::e2(block_sums[2 * blockIdx.x], block_sums[2 * blockIdx.x + 1]);
    if (threadIdx.x > 0) run = gl::e2_add(run, gl::e2(sh[2 * (threadIdx.x - 1)], sh[2 * (threadIdx.x - 1) + 1]));
    for (int e = 0; e < SCAN_E; e++) {
        if (base + e < n) { acc0[base + e] = run.a; acc1[base + e] = run.b; }
        run = gl::e2_add(run, v[e]);
    }
}
void launch_ef_exclusive_scan(const u64* totals, size_t n, u64* acc0, u64* acc1, u64* final2, u64* scratch, cudaStream_t st) {
    size_t nb = (n + SCAN_B - 1) / SCAN_B;
    k_scan_block_totals<<<(unsigned)nb, SCAN_T, 0, st>>>(totals, n, scratch);
    k_scan_block_sums<<<1, 32, 0, st>>>(scratch, nb, final2);
    k_scan_apply<<<(unsigned)nb, SCAN_T, 0, st>>>(totals, n, scratch, acc0, acc1);
    COUNT_LAUNCH(); COUNT_LAUNCH(); COUNT_LAUNCH();
}

// =============================================================================================
// OOD evaluation: dot products of coefficient columns with y^(bitrev(p))
// =============================================================================================
struct PowTable { E2 sq[24]; };   // sq[i] = y^(2^i)
// wvec[p] = y^(bitrev_n(p)) = A[p >> h] * B[p & (2^h - 1)]: the two half tables (2^(n-h) and 2^h entries, built
// by k_pow_tables with at most n/2 multiplications per entry) replace the per-element product over up to n
// squares (was 4.8 ms of the 2^20 proof for 18 vectors; now one extension multiplication per element).
__global__ void k_pow_tables(PowTable tab, u32 n, u32 h, u64* __restrict__ A, u64* __restrict__ B) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    u32 na = 1u << (n - h), nb = 1u << h;
    if (i >= na + nb) return;
    bool is_a = i < na;
    u32 idx = is_a ? i : i - na, bits = is_a ? n - h : h, off = is_a ? h : 0;
    E2 w = gl::e2(1, 0);
    for (u32 b = 0; b < bits; b++)
        if ((idx >> b) & 1) w = gl::e2_mul(w, tab.sq[n - 1 - (off + b)]);   // bit (off + b) of p <-> exponent bit n-1-(off+b)
    u64* dst = is_a ? A : B;
    reinterpret_cast<ulonglong2*>(dst)[idx] = make_ulonglong2(w.a, w.b);
}
__global__ void k_pow_bitrev(const u64* __restrict__ A, const u64* __restrict__ B, u32 n, u32 h, u64* __restrict__ wvec_slice, size_t p0, size_t cnt) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cnt) return;
    size_t p = p0 + i;
    u64* wvec = wvec_slice - 2 * p0;
    ulonglong2 a = reinterpret_cast<const ulonglong2*>(A)[p >> h], b = reinterpret_cast<const ulonglong2*>(B)[p & ((1u << h) - 1)];
    E2 w = gl::e2_mul(gl::e2(a.x, a.y), gl::e2(b.x, b.y));
    reinterpret_cast<ulonglong2*>(wvec)[p] = make_ulonglong2(w.a, w.b);
}
void launch_pow_bitrev(E2 y, u32 n, u64* wvec, u64* scratch, size_t p0, size_t cnt, cudaStream_t st) {
    PowTable tab;
    E2 x = y;
    for (u32 i = 0; i < 24; i++) { tab.sq[i] = x; x = gl::e2_sqr(x); }
    u32 h = n / 2, na = 1u << (n - h), nb = 1u << h;
    u64* A = scratch; u64* B = scratch + 2 * (size_t)na;
    k_pow_tables<<<(na + nb + 127) / 128, 128, 0, st>>>(tab, n, h, A, B);
    k_pow_bitrev<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(A, B, n, h, wvec, p0, cnt);
    COUNT_LAUNCH(); COUNT_LAUNCH();
}

using glf::Acc160;      // 160-bit accumulator of unreduced products (poseidon2_fast2.cuh)
using glf::acc_mul;
using glf::acc_reduce;
// Column dot products with the two weight vectors of an opening point pair: like k_deep, the 128-bit products are accumulated
// unreduced (a thread adds chunk / 256 of them per accumulator) and reduced once; 2 columns x 4 weight coordinates per thread
// (8 accumulators of five registers, 72 registers for sm_90a): one reduction per accumulator instead of one per product.
static constexpr int OOD_COLS = 2;
__global__ void __launch_bounds__(256) k_ood_dot(const u64* __restrict__ coef, size_t col_stride, u32 n_cols, u32 n,
                                                 const u64* __restrict__ w0, const u64* __restrict__ w1,
                                                 u64* __restrict__ partial, u32 n_chunks) {
    __shared__ u64 red[8][OOD_COLS * 4];
    size_t N = (size_t)1 << n;
    size_t chunk = N / n_chunks;
    size_t p0 = (size_t)blockIdx.x * chunk;
    u32 c0 = blockIdx.y * OOD_COLS;
    const ulonglong2* W0 = reinterpret_cast<const ulonglong2*>(w0);
    const ulonglong2* W1 = reinterpret_cast<const ulonglong2*>(w1);
    u64 acc[OOD_COLS * 4];
    Acc160 A[OOD_COLS * 4];
#pragma unroll
    for (int i = 0; i < OOD_COLS * 4; i++) A[i] = Acc160{0, 0, 0};
    for (size_t p = p0 + threadIdx.x; p < p0 + chunk; p += blockDim.x) {
        ulonglong2 a = W0[p], b = W1[p];
        u64 v[OOD_COLS];
#pragma unroll
        for (int c = 0; c < OOD_COLS; c++) v[c] = (c0 + c < n_cols) ? coef[(size_t)(c0 + c) * col_stride + p] : 0ull;
#pragma unroll
        for (int c = 0; c < OOD_COLS; c++) {
            acc_mul(A[4 * c + 0], a.x, v[c]); acc_mul(A[4 * c + 1], a.y, v[c]);
            acc_mul(A[4 * c + 2], b.x, v[c]); acc_mul(A[4 * c + 3], b.y, v[c]);
        }
    }
#pragma unroll
    for (int i = 0; i < OOD_COLS * 4; i++) acc[i] = acc_reduce(A[i]);
#pragma unroll
    for (int i = 0; i < OOD_COLS * 4; i++) {
        u64 v = acc[i];
        for (int off = 16; off > 0; off >>= 1) v = gl::add(v, (u64)__shfl_down_sync(0xffffffffu, (unsigned long long)v, off));
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][i] = v;
    }
    __syncthreads();
    if (threadIdx.x < OOD_COLS * 4) {
        u64 v = 0;
        for (int w = 0; w < 8; w++) v = gl::add(v, red[w][threadIdx.x]);
        u32 c = c0 + threadIdx.x / 4;
        if (c < n_cols) partial[((size_t)c * n_chunks + blockIdx.x) * 4 + (threadIdx.x & 3)] = v;
    }
}
void launch_ood_dot(const u64* coef, size_t col_stride, u32 n_cols, u32 n, const u64* w0, const u64* w1, u64* partial,
                    u32 n_chunks, cudaStream_t st) {
    dim3 grid(n_chunks, (n_cols + OOD_COLS - 1) / OOD_COLS);
    k_ood_dot<<<grid, 256, 0, st>>>(coef, col_stride, n_cols, n, w0, w1, partial, n_chunks);
    COUNT_LAUNCH();
}
__global__ void k_ood_reduce(const u64* __restrict__ partial, u32 n_cols, u32 n_chunks, u64* __restrict__ out) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cols * 4) return;
    u32 c = i / 4, k = i & 3;
    u64 v = 0;
    for (u32 ch = 0; ch < n_chunks; ch++) v = gl::add(v, partial[((size_t)c * n_chunks + ch) * 4 + k]);
    out[i] = v;
}
void launch_ood_reduce(const u64* partial, u32 n_cols, u32 n_chunks, u64* out, cudaStream_t st) {
    k_ood_reduce<<<(n_cols * 4 + 127) / 128, 128, 0, st>>>(partial, n_cols, n_chunks, out);
    COUNT_LAUNCH();
}

// =============================================================================================
// DEEP quotient
// =============================================================================================
struct DeepKArgs {
    const DeepMat* m; int n_mats;
    u32 log_n, log_b;
    const u64* apow; u32 total_w;
    E2 z0, z1, fz0, fz1, beta;
    PushDst out;
    const u64* w_hi; const u64* w_lo; u32 lo_bits;
    u64 shift, w_l;
    u32 t0, nt;
};
// PTS points per thread: point k lies k/PTS of the rank's range further on, so every stream stays coalesced; PTS points multiply
// the independent column loads in flight (4 columns x PTS points) and share ONE field inversion for their denominators
// (z0 - x)(z1 - x) (Montgomery's trick) -- the inversion (a Fermat power, ~100 multiplications) is as much arithmetic as the
// 121-column dot products of a point.  PTS = 2 takes 64 registers for sm_90a.
static constexpr int DEEP_PTS = 2;
template <int PTS>
__global__ void __launch_bounds__(256) k_deep(DeepKArgs a) {
    extern __shared__ u64 sm_apow[];
    for (u32 i = threadIdx.x; i < 2 * a.total_w; i += blockDim.x) sm_apow[i] = a.apow[i];
    __syncthreads();
    const size_t per = ((size_t)a.nt << a.log_n) / PTS;          // launch_deep picks PTS so that it divides the range
    size_t pos0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos0 >= per) return;
    pos0 += (size_t)a.t0 << a.log_n;
    // f_red(x) = sum_i alpha^(W-1-i) col_i(x): two base-field dot products (one per extension coordinate of the alpha
    // powers).  The 128-bit products are accumulated UNREDUCED in 160-bit accumulators and reduced once at the end
    // (at most 2^32 terms fit; a proof has a few hundred columns): a column costs two wide multiplications and two
    // three-word additions instead of two modular multiplications and their reductions (ncu r2b: the kernel was bound by
    // the integer pipes at ~85 instructions per column, not by HBM).
    Acc160 fa[PTS], fb[PTS];
    u32 t[PTS], r[PTS];
#pragma unroll
    for (int k = 0; k < PTS; k++) {
        fa[k] = Acc160{0, 0, 0}; fb[k] = Acc160{0, 0, 0};
        size_t pos = pos0 + (size_t)k * per;
        t[k] = (u32)(pos >> a.log_n); r[k] = (u32)(pos & (((size_t)1 << a.log_n) - 1));
    }
    for (int m = 0; m < a.n_mats; m++) {
        const DeepMat M = a.m[m];
        size_t Lm = (size_t)1 << (M.log_n + a.log_b);
        const u64* base[PTS];
#pragma unroll
        for (int k = 0; k < PTS; k++) base[k] = M.base + ((size_t)t[k] << M.log_n) + (r[k] & ((1u << M.log_n) - 1));
        const u64* ap = sm_apow + 2 * M.alpha_off;
        u32 c = 0;
        // four independent column loads in flight per point
        for (; c + 4 <= M.width; c += 4) {
            u64 v[PTS][4];
#pragma unroll
            for (int k = 0; k < PTS; k++)
#pragma unroll
                for (int j = 0; j < 4; j++) v[k][j] = base[k][(size_t)(c + j) * Lm];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                u64 pa = ap[2 * (c + j)], pb = ap[2 * (c + j) + 1];
#pragma unroll
                for (int k = 0; k < PTS; k++) { acc_mul(fa[k], pa, v[k][j]); acc_mul(fb[k], pb, v[k][j]); }
            }
        }
        for (; c < M.width; c++) {
#pragma unroll
            for (int k = 0; k < PTS; k++) {
                u64 v = base[k][(size_t)c * Lm];
                acc_mul(fa[k], ap[2 * c], v); acc_mul(fb[k], ap[2 * c + 1], v);
            }
        }
    }
    E2 d0[PTS], d1[PTS], den[PTS];
#pragma unroll
    for (int k = 0; k < PTS; k++) {
        u64 x = gl::mul(gl::mul(a.shift, gl::pow(a.w_l, t[k])), w_pow(a.w_hi, a.w_lo, a.lo_bits, r[k]));
        d0[k] = gl::e2(gl::sub(a.z0.a, x), a.z0.b); d1[k] = gl::e2(gl::sub(a.z1.a, x), a.z1.b);
        den[k] = gl::e2_mul(d0[k], d1[k]);
    }
    E2 inv[PTS], prefix[PTS];
    prefix[0] = den[0];
#pragma unroll
    for (int k = 1; k < PTS; k++) prefix[k] = gl::e2_mul(prefix[k - 1], den[k]);
    E2 run = gl::e2_inv(prefix[PTS - 1]);              // 1 / (den_0 ... den_(PTS-1)), peeled from the back
#pragma unroll
    for (int k = PTS - 1; k > 0; k--) { inv[k] = gl::e2_mul(run, prefix[k - 1]); run = gl::e2_mul(run, den[k]); }
    inv[0] = run;
#pragma unroll
    for (int k = 0; k < PTS; k++) {
        E2 fr = gl::e2(acc_reduce(fa[k]), acc_reduce(fb[k]));
        E2 i0 = gl::e2_mul(inv[k], d1[k]), i1 = gl::e2_mul(inv[k], d0[k]);
        E2 q = gl::e2_add(gl::e2_mul(i0, gl::e2_sub(a.fz0, fr)),
                          gl::e2_mul(a.beta, gl::e2_mul(i1, gl::e2_sub(a.fz1, fr))));
        size_t i = ((size_t)r[k] << a.log_b) | t[k];
        push_u2(a.out, i, i, make_ulonglong2(q.a, q.b));
    }
}
void launch_deep(const DeepArgs& a, cudaStream_t st) {
    DeepKArgs k;
    k.m = a.m; k.n_mats = a.n_mats; k.log_n = a.log_n_max; k.log_b = a.log_blowup; k.apow = a.apow; k.total_w = a.total_w;
    k.z0 = a.z0; k.z1 = a.z1; k.fz0 = a.fz0; k.fz1 = a.fz1; k.beta = a.beta; k.out = a.out;
    k.w_hi = a.T->w_hi; k.w_lo = a.T->w_lo; k.lo_bits = a.T->lo_bits;
    u32 log_lde = a.log_n_max + a.log_blowup;
    k.shift = gl::lde_shift(log_lde); k.w_l = gl::two_adic_generator(log_lde);
    u32 B = 1u << a.log_blowup;
    k.t0 = a.nt ? a.t0 : 0; k.nt = a.nt ? a.nt : B;
    size_t cnt = (size_t)k.nt << a.log_n_max;
    if (cnt % (256 * DEEP_PTS) == 0) k_deep<DEEP_PTS><<<(unsigned)(cnt / (256 * DEEP_PTS)), 256, 2 * a.total_w * sizeof(u64), st>>>(k);
    else k_deep<1><<<(unsigned)((cnt + 255) / 256), 256, 2 * a.total_w * sizeof(u64), st>>>(k);
    COUNT_LAUNCH();
}

// =============================================================================================
// FRI fold (arity 2 / 4 / 8), natural domain order: interpolate the 2^la values of the coset
// s*<w_a> (inverse DFT), evaluate at beta/s, divide by the arity
// (pcs/fri/fold/arity2.rs, arity4.rs:46-121, arity8.rs:35-75 compute the same field element)
// =============================================================================================
struct FoldArgs { u64 winv[8]; u64 arity_inv; u64 w_dom_inv; u32 log_dom, la; E2 beta; };
__global__ void __launch_bounds__(256) k_fri_fold(const u64* __restrict__ ev, FoldArgs fa, PushDst next, u32 log_b, u32 t0, u32 log_nt) {
    size_t q = (size_t)1 << (fa.log_dom - fa.la);
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= ((q >> log_b) << log_nt)) return;
    size_t i = ((idx >> log_nt) << log_b) | (t0 + (idx & ((1u << log_nt) - 1)));
    const ulonglong2* e = reinterpret_cast<const ulonglong2*>(ev);
    u32 a = 1u << fa.la;
    E2 y[8];
    for (u32 k = 0; k < a; k++) { ulonglong2 v = e[i + (size_t)k * q]; y[k] = gl::e2(v.x, v.y); }   // y_k = f(s * w_a^k)
    u64 s_inv = gl::pow(fa.w_dom_inv, (u64)i);
    E2 x = gl::e2_mulf(fa.beta, s_inv);
    E2 acc = gl::e2(0, 0);
    for (u32 m = a; m-- > 0;) {                      // Horner over c_m = sum_k y_k * w_a^(-m k)
        E2 c = y[0];
        for (u32 k = 1; k < a; k++) c = gl::e2_add(c, gl::e2_mulf(y[k], fa.winv[(m * k) & (a - 1)]));
        acc = gl::e2_add(gl::e2_mul(acc, x), c);
    }
    acc = gl::e2_mulf(acc, fa.arity_inv);
    push_u2(next, i, i, make_ulonglong2(acc.a, acc.b));
}
void launch_fri_fold(const u64* evals, u32 log_dom, u32 log_arity, E2 beta, const PushDst& next, u32 log_b, u32 t0, u32 nt, cudaStream_t st) {
    size_t q = (size_t)1 << (log_dom - log_arity);
    if (q < ((size_t)1 << log_b)) { log_b = 0; t0 = 0; nt = 1; }
    FoldArgs fa;
    u32 a = 1u << log_arity;
    u64 wi = gl::inv(gl::two_adic_generator(log_arity)), x = 1;
    for (u32 j = 0; j < 8; j++) { fa.winv[j] = j < a ? x : 0; x = gl::mul(x, wi); }
    fa.arity_inv = gl::inv((u64)a); fa.w_dom_inv = gl::inv(gl::two_adic_generator(log_dom));
    fa.log_dom = log_dom; fa.la = log_arity; fa.beta = beta;
    size_t cnt = (q >> log_b) * nt;
    k_fri_fold<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(evals, fa, next, log_b, t0, log2_exact(nt));
    COUNT_LAUNCH();
}

// =============================================================================================
// Proof-of-work grinding
// =============================================================================================
template <int PERM>
__global__ void __launch_bounds__(128) k_grind(const u64* __restrict__ st12, u32 in_len, u64 mask, u64 start, u64 count,
                                               u64* result) {
    u64 idx = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    u64 w = start + idx;
    u64 s[12];
#pragma unroll
    for (int k = 0; k < 12; k++) s[k] = st12[k];
#pragma unroll
    for (u32 k = 0; k < 8; k++) {
        if (k == in_len) s[k] = w;
        else if (k > in_len) s[k] = 0;
    }
    s[8] = gl::add(s[8], (u64)(in_len + 1));
    alg_permute<PERM>(s);
    if ((glf::canon(s[7]) & mask) == 0) atomicMin(reinterpret_cast<unsigned long long*>(result), (unsigned long long)w);
}
template <int PERM>
static void launch_grind_t(const u64* d_state12, u32 in_len, u32 bits, u64 start, u64 count, u64* d_result, cudaStream_t st) {
    u64 mask = (1ull << bits) - 1;
    k_grind<PERM><<<(unsigned)((count + 127) / 128), 128, 0, st>>>(d_state12, in_len, mask, start, count, d_result);
    COUNT_LAUNCH();
}
void launch_grind(const u64* d_state12, u32 in_len, u32 bits, u64 start, u64 count, u64* d_result, cudaStream_t st, int perm) {
#define X(PM) launch_grind_t<PM>(d_state12, in_len, bits, start, count, d_result, st)
    ALG_DISPATCH(perm, X);
#undef X
}

__global__ void k_compare(const u64* __restrict__ a, const u64* __restrict__ b, size_t n, u32* flag) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && a[i] != b[i]) atomicOr(flag, 4u);
}
void launch_compare(const u64* a, const u64* b, size_t n, u32* flag, cudaStream_t st) {
    k_compare<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, b, n, flag);
    COUNT_LAUNCH();
}

__global__ void k_gather(const u64* const* __restrict__ ptrs, u64* __restrict__ out, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = *ptrs[i];
}
void launch_gather(const u64* const* d_ptrs, u64* d_out, size_t n, cudaStream_t st) {
    if (!n) return;
    k_gather<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_ptrs, d_out, n);
    COUNT_LAUNCH();
}

__global__ void k_gather_push(const u64* const* __restrict__ ptrs, const int* __restrict__ owner, PeerPtrs out, u32 rank, u32 world, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int o = owner[i];
    if (o < 0) out.p[rank][i] = *ptrs[i];
    else if ((u32)o == rank) { u64 v = *ptrs[i]; for (u32 g = 0; g < world; g++) out.p[g][i] = v; }
}
void launch_gather_push(const u64* const* d_ptrs, const int* d_owner, const PeerPtrs& out, u32 rank, u32 world, size_t n, cudaStream_t st) {
    if (!n) return;
    k_gather_push<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_ptrs, d_owner, out, rank, world, n);
    COUNT_LAUNCH();
}

__global__ void k_export_lde(const u64* __restrict__ lde, u32 log_n, u32 log_b, u32 width, u64* __restrict__ out) {
    size_t L = (size_t)1 << (log_n + log_b);
    size_t pos = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= L) return;
    u32 t = (u32)(pos >> log_n), r = (u32)(pos & (((size_t)1 << log_n) - 1));
    u32 i = (r << log_b) | t;
    size_t row = gl::bitrev32(i, log_n + log_b);
    for (u32 c = 0; c < width; c++) out[row * width + c] = lde[(size_t)c * L + pos];
}
void launch_export_lde_bitrev_rm(const u64* lde, u32 log_n, u32 log_blowup, u32 width, u64* out_rm, cudaStream_t st) {
    size_t L = (size_t)1 << (log_n + log_blowup);
    k_export_lde<<<(unsigned)((L + 255) / 256), 256, 0, st>>>(lde, log_n, log_blowup, width, out_rm);
    COUNT_LAUNCH();
}

}  // namespace mk
