// Run-time specialisation of the constraint evaluator (a4) for large AIRs.
//
// The op-list interpreter (k_constraints) pays an instruction fetch, a switch and local-memory slot traffic
// per node -- fine for the 19-node DummyMidenAir, ~4x too slow for the ~5 k-node Miden AIRs
// (air/src/lib.rs:342-355,442-454,523-528).  For programs above a node threshold the session lowers the SAME
// validated op-list into straight-line CUDA C++ (typed: base values are u64, extension values E2; constants
// are literals; the alpha fold uses precomputed alpha powers, which is the reference's own base/ext split,
// prover/constraints/folder.rs:88-105), compiles it once per AIR with NVRTC for sm_90a and launches the
// cubin through the driver API.  Field arithmetic is exact, so the result is bit-identical to the interpreter
// (asserted in tests/test_gpu_parity.py).  libnvrtc / libcuda are dlopen'ed on first use; when NVRTC is
// missing the session keeps using the interpreter and says so in mdn_get_info(MDN_INFO_JIT).  The same lowering also
// gives the LogUp row kernel (MODE_LOOKUP), the trace-check row kernels (MODE_CHECK, MDN_INFO_JIT_CHECK) and the
// lookup-check row kernels (MODE_LOOKUP_CHECK, MDN_INFO_JIT_LOOKUP_CHECK).
#pragma once
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

namespace jit {

// Kernel arguments: layout must equal `struct JitArgs` in PRELUDE below (pointers and u64 first, then u32).
struct JitArgs {
    const uint64_t* main_lde; const uint64_t* aux_lde; const uint64_t* prep_lde;
    const uint64_t* publics; const uint64_t* challenges; const uint64_t* aux_values;
    const uint64_t* periodic; const uint64_t* apow;
    const uint64_t* acc_in; uint64_t* acc_out;
    const uint64_t* w_hi; const uint64_t* w_lo;
    uint64_t shift, w_l, w_h_inv;
    uint64_t zh[16], inv_zh[16];
    uint64_t beta_a, beta_b;
    uint32_t log_n, log_b, acc_in_log_n, lo_bits, log_max_period, pad;
};

// Arguments of the generated LogUp row kernel (same member names as JitArgs where the leaf code is shared).
struct LookupJitArgs {
    const uint64_t* main_lde;      // raw main trace, column-major [col][row]
    const uint64_t* prep_lde;      // raw preprocessed trace, column-major [col][row], or NULL (the program reads none)
    const uint64_t* publics; const uint64_t* challenges; const uint64_t* periodic;   // periodic: raw row-major matrix
    uint64_t* aux_cm; uint64_t* totals;
    uint32_t* bad_flag;
    uint32_t log_n, n_periodic, log_max_period, pad;
};

// Arguments of the generated trace-check kernels k_jit_check / k_jit_census (the semantics of k_check_rows /
// k_census_rows, kernels.cuh CheckArgs / CensusArgs); layout must equal `struct CheckJitArgs` in PRELUDE_CHECK below.
struct CheckJitArgs {
    const uint64_t* main_lde; const uint64_t* aux_lde; const uint64_t* prep_lde;   // raw column-major traces (L = N)
    const uint64_t* publics; const uint64_t* challenges; const uint64_t* aux_values;
    const uint64_t* periodic;                         // raw row-major matrix (max_period x n_periodic)
    unsigned long long* first; unsigned long long* failing_rows;   // k_jit_check: init ~0 / 0; census: failing_rows only
    uint32_t* row_count; unsigned long long* tally;  // k_jit_census: 2^log_n counts, 3 * n_cons tally words; check: NULL
    uint64_t row0, n_rows;                           // k_jit_check: rows [row0, row0 + n_rows)
    uint32_t log_n, n_cons, n_periodic, log_max_period;
};
// per-block shared tallies of k_jit_census up to this many constraints (kernels.cuh CENSUS_SHARED_K)
static constexpr uint32_t CENSUS_SHARED_K = 256;

// Arguments of the generated lookup-check kernels k_jit_balance / k_jit_fold / k_jit_fold_census (the semantics of
// k_balance_rows / k_fold_rows / k_fold_census_rows, kernels.cuh BalanceArgs / LookupFoldArgs / FoldCensusArgs); one
// struct for the three, each reading its own members.  Layout must equal `struct LookupCheckJitArgs` in
// PRELUDE_LOOKUP_CHECK below.
struct LookupCheckJitArgs {
    const uint64_t* main_lde; const uint64_t* prep_lde;   // raw column-major traces (L = N); prep: NULL when unread
    const uint64_t* publics; const uint64_t* challenges; const uint64_t* periodic;   // periodic: raw row-major matrix
    // k_jit_balance: mutex annotation, the table (BalanceTable), counters and lists
    const uint32_t* mutex_pos; const uint32_t* mutex_group; const uint32_t* mutex_site;
    uint64_t* t_keys; uint64_t* t_sums; unsigned long long* t_count; unsigned long long* t_first;
    unsigned long long* counters; uint64_t* mutex_out; uint64_t* contrib_out;
    // k_jit_fold / k_jit_fold_census
    const uint32_t* marks; const uint64_t* aux_cm; uint64_t* folds_out;
    unsigned long long* first; unsigned long long* failing_rows; unsigned long long* zero_u;
    uint32_t* row_count; unsigned long long* tally;
    uint64_t t_mask, final_a, final_b, row0, n_rows;   // k_jit_fold: rows [row0, row0 + n_rows)
    uint32_t log_n, n_periodic, log_max_period, n_cols, instance, mode, n_mutex, folds_cm;
};
// activity words of the mutex sites per row (kernels.cuh BALANCE_MUTEX_MAX / 64)
static constexpr uint32_t LOOKUP_CHECK_MUTEX_WORDS = 16;

// what generate() emits: the proof's constraint kernel, the LogUp row kernel, the two trace-check kernels, or the three
// lookup-check kernels
enum Mode : uint32_t { MODE_CONSTRAINTS = 0, MODE_LOOKUP = 1, MODE_CHECK = 2, MODE_LOOKUP_CHECK = 3 };

static const char PRELUDE[] = R"CUDA(
typedef unsigned long long u64;
typedef unsigned int u32;
struct E2 { u64 a, b; };
struct JitArgs {
    const u64* main_lde; const u64* aux_lde; const u64* prep_lde;
    const u64* publics; const u64* challenges; const u64* aux_values;
    const u64* periodic; const u64* apow;
    const u64* acc_in; u64* acc_out;
    const u64* w_hi; const u64* w_lo;
    u64 shift, w_l, w_h_inv;
    u64 zh[16], inv_zh[16];
    u64 beta_a, beta_b;
    u32 log_n, log_b, acc_in_log_n, lo_bits, log_max_period, pad;
};
#define GP 0xFFFFFFFF00000001ull
// canonical (< p) Goldilocks arithmetic on the carry flag
__device__ __forceinline__ u64 fsub(u64 a, u64 b) {
    u64 d; u32 m;
    asm("sub.cc.u64 %0, %2, %3;\n\tsubc.u32 %1, 0, 0;" : "=l"(d), "=r"(m) : "l"(a), "l"(b));
    return d - (u64)m;
}
__device__ __forceinline__ u64 fadd(u64 a, u64 b) { return fsub(a, GP - b); }
__device__ __forceinline__ u64 fneg(u64 a) { return a ? GP - a : 0ull; }
)CUDA";
// field multiplication: one 128-bit product as in poseidon2_fast2.cuh (needs --device-int128), the carry folded by an
// IMAD.WIDE
static const char PRELUDE_FMUL_G2[] = R"CUDA(__device__ __forceinline__ u64 fmul(u64 x, u64 y) {
    unsigned __int128 q = (unsigned __int128)x * y;
    u64 lo = (u64)q, hi = (u64)(q >> 64);
    u32 hl = (u32)hi, hh = (u32)(hi >> 32);
    u64 t, m, r; u32 b, c;
    asm("sub.cc.u64 %0, %2, %3;\n\tsubc.u32 %1, 0, 0;" : "=l"(t), "=r"(b) : "l"(lo), "l"((u64)hh));
    t -= (u64)b;
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(m) : "r"(hl), "r"(0xFFFFFFFFu));
    asm("add.cc.u64 %0, %2, %3;\n\taddc.u32 %1, 0, 0;" : "=l"(r), "=r"(c) : "l"(t), "l"(m));
    r = (u64)c * 0xFFFFFFFFull + r;
    u64 q2; u32 k;
    asm("sub.cc.u64 %0, %2, %3;\n\tsubc.u32 %1, 0, 0;" : "=l"(q2), "=r"(k) : "l"(r), "l"(GP));
    return q2 - (u64)k;
}
)CUDA";
static const char PRELUDE_B[] = R"CUDA(__device__ __forceinline__ u64 fmul7(u64 x) { return fmul(x, 7ull); }
__device__ u64 fpow(u64 b, u64 e) { u64 r = 1; while (e) { if (e & 1) r = fmul(r, b); b = fmul(b, b); e >>= 1; } return r; }
__device__ u64 finv(u64 a) { return fpow(a, GP - 2); }
__device__ __forceinline__ E2 mk(u64 a, u64 b) { E2 r; r.a = a; r.b = b; return r; }
__device__ __forceinline__ E2 eadd(E2 x, E2 y) { return mk(fadd(x.a, y.a), fadd(x.b, y.b)); }
__device__ __forceinline__ E2 esub(E2 x, E2 y) { return mk(fsub(x.a, y.a), fsub(x.b, y.b)); }
__device__ __forceinline__ E2 eneg(E2 x) { return mk(fneg(x.a), fneg(x.b)); }
__device__ __forceinline__ E2 emul(E2 x, E2 y) {
    return mk(fadd(fmul(x.a, y.a), fmul7(fmul(x.b, y.b))), fadd(fmul(x.a, y.b), fmul(x.b, y.a)));
}
__device__ __forceinline__ E2 emulf(E2 x, u64 s) { return mk(fmul(x.a, s), fmul(x.b, s)); }
__device__ __forceinline__ E2 eaddf(E2 x, u64 s) { return mk(fadd(x.a, s), x.b); }
__device__ __forceinline__ E2 esubf(E2 x, u64 s) { return mk(fsub(x.a, s), x.b); }      // x - s
__device__ __forceinline__ E2 efsub(u64 s, E2 x) { return mk(fsub(s, x.a), fneg(x.b)); } // s - x
__device__ __forceinline__ E2 ldapow(const u64* __restrict__ p, u32 k) { return mk(p[2 * k], p[2 * k + 1]); }
__device__ E2 einv(E2 x) { u64 n = fsub(fmul(x.a, x.a), fmul7(fmul(x.b, x.b))); u64 ni = finv(n); return mk(fmul(x.a, ni), fneg(fmul(x.b, ni))); }
)CUDA";
// the lookup mode's argument struct (host mirror: LookupJitArgs above)
static const char PRELUDE_LOOKUP_ARGS[] = R"CUDA(struct LookupJitArgs {
    const u64* main_lde; const u64* prep_lde; const u64* publics; const u64* challenges; const u64* periodic;
    u64* aux_cm; u64* totals;
    u32* bad_flag;
    u32 log_n, n_periodic, log_max_period, pad;
};
)CUDA";
// what the constraint and check modes emit in its place: the struct without prep_lde, which they do not use; kept so
// that their generated source, and with it their cubins, stay exactly as they were before the lookup mode read
// preprocessed columns
static const char PRELUDE_LOOKUP_ARGS_UNUSED[] = R"CUDA(struct LookupJitArgs {
    const u64* main_lde; const u64* publics; const u64* challenges; const u64* periodic;
    u64* aux_cm; u64* totals;
    u32* bad_flag;
    u32 log_n, n_periodic, log_max_period, pad;
};
)CUDA";
// check mode only (the constraint and lookup modes emit the preludes above and nothing else): the argument struct
// and the failure record of one (row, constraint) -- a count, a least row and a greatest row per constraint, in the
// block's shared table `sh` ([3][CENSUS_SHARED_K]) or, when sh is NULL, straight in the global tally
static const char PRELUDE_CHECK[] = R"CUDA(struct CheckJitArgs {
    const u64* main_lde; const u64* aux_lde; const u64* prep_lde;
    const u64* publics; const u64* challenges; const u64* aux_values;
    const u64* periodic;
    unsigned long long* first; unsigned long long* failing_rows;
    u32* row_count; unsigned long long* tally;
    u64 row0, n_rows;
    u32 log_n, n_cons, n_periodic, log_max_period;
};
template <class T> __device__ __forceinline__ T census_max(T* p, T v) { return atomicMax(p, v); }
__device__ __noinline__ void tally(const CheckJitArgs& a, u32* sh, u32 r, u32 k) {
    if (sh) { atomicAdd(&sh[k], 1u); atomicMin(&sh[CENSUS_SHARED_K + k], r); census_max(&sh[2 * CENSUS_SHARED_K + k], r); }
    else {
        atomicAdd(&a.tally[3 * k], 1ull);
        atomicMin(&a.tally[3 * k + 1], (unsigned long long)r);
        census_max(&a.tally[3 * k + 2], (unsigned long long)r);
    }
}
)CUDA";
// lookup-check mode only, after `#define LK_NC <columns>` and `#define LK_MUTEX_WORDS <words>`: the argument struct, the
// per-row state every chunk carries by reference, the balance table of kernels.cu (the same hash, probe order and
// atomics; the 128-bit compare-and-swap in PTX, which every NVRTC that targets sm_90 accepts), the fold steps of
// fold_walk / fold_divide / fold_verdict in the same operation order, and lk_hook, which the chunks call once per
// interaction in interaction order.  Field results are exact, so every word equals the interpreter's.
static const char PRELUDE_LOOKUP_CHECK[] = R"CUDA(struct LookupCheckJitArgs {
    const u64* main_lde; const u64* prep_lde;
    const u64* publics; const u64* challenges; const u64* periodic;
    const u32* mutex_pos; const u32* mutex_group; const u32* mutex_site;
    u64* t_keys; u64* t_sums; unsigned long long* t_count; unsigned long long* t_first;
    unsigned long long* counters; u64* mutex_out; u64* contrib_out;
    const u32* marks; const u64* aux_cm; u64* folds_out;
    unsigned long long* first; unsigned long long* failing_rows; unsigned long long* zero_u;
    u32* row_count; unsigned long long* tally;
    u64 t_mask, final_a, final_b, row0, n_rows;
    u32 log_n, n_periodic, log_max_period, n_cols, instance, mode, n_mutex, folds_cm;
};
// mode 0 / 1 / 2: the balance pass of that mode; 3: the fold
struct LkRow {
    E2 V[LK_NC], U[LK_NC];                 // the columns' folds
    E2 bn, bd, vg, ug; u64 bf; u32 cur;    // the open batch (N, D) and its flag, the open group (V_g, U_g) and its column
    u32 mode;
    u64 act[LK_MUTEX_WORDS];               // activity of the annotated interactions (bit mutex_pos[k])
    unsigned long long pushes;
};
template <class T> __device__ __forceinline__ T census_max(T* p, T v) { return atomicMax(p, v); }
struct alignas(16) K2 { u64 x, y; };
__device__ __forceinline__ u64 balance_hash(u64 c0, u64 c1) {
    u64 h = c0 * 0x9E3779B97F4A7C15ull ^ (c1 + 0x632BE59BD9B4E019ull) * 0xC2B2AE3D27D4EB4Full;
    return h ^ (h >> 29) ^ (h >> 47);
}
__device__ __forceinline__ u64 balance_key(u32 inst, u64 row, u32 k) { return ((u64)inst << 48) | (row << 24) | k; }
__device__ __forceinline__ K2 cas128(u64* p, u64 c0, u64 c1, u64 n0, u64 n1) {
    K2 o;
    asm volatile("{\n\t.reg .b128 d, b, c;\n\tmov.b128 b, {%2, %3};\n\tmov.b128 c, {%4, %5};\n\t"
                 "atom.global.cas.b128 d, [%6], b, c;\n\tmov.b128 {%0, %1}, d;\n\t}"
                 : "=l"(o.x), "=l"(o.y) : "l"(c0), "l"(c1), "l"(n0), "l"(n1), "l"(p) : "memory");
    return o;
}
__device__ __forceinline__ u64 balance_insert(const LookupCheckJitArgs& a, u64 c0, u64 c1) {
    K2* keys = reinterpret_cast<K2*>(a.t_keys);
    for (u64 s = balance_hash(c0, c1) & a.t_mask;; s = (s + 1) & a.t_mask) {
        K2 cur = keys[s];
        if (cur.x == c0 && cur.y == c1) return s;
        if (cur.x != ~0ull && cur.y != ~0ull) continue;
        K2 old = cas128(a.t_keys + 2 * s, ~0ull, ~0ull, c0, c1);
        if ((old.x == ~0ull && old.y == ~0ull) || (old.x == c0 && old.y == c1)) return s;
    }
}
__device__ __forceinline__ u64 balance_find(const LookupCheckJitArgs& a, u64 c0, u64 c1) {
    const K2* keys = reinterpret_cast<const K2*>(a.t_keys);
    u64 s = balance_hash(c0, c1) & a.t_mask;
    for (;; s = (s + 1) & a.t_mask) { K2 cur = keys[s]; if (cur.x == c0 && cur.y == c1) return s; }
}
__device__ __forceinline__ void balance_add(const LookupCheckJitArgs& a, u64 s, u64 m, u64 key) {
    unsigned long long* sum = reinterpret_cast<unsigned long long*>(a.t_sums) + 2 * s;
    unsigned long long old = atomicAdd(sum, (unsigned long long)m);
    if (old + m < old) atomicAdd(sum + 1, 1ull);
    atomicAdd(a.t_count + s, 1ull);
    atomicMin(a.t_first + s, (unsigned long long)key);
}
__device__ __forceinline__ void lk_close_batch(LkRow& st) {
    st.ug = eadd(st.ug, emulf(esub(st.bd, mk(1ull, 0ull)), st.bf));
    st.vg = eadd(st.vg, emulf(st.bn, st.bf));
    st.bn = mk(0ull, 0ull); st.bd = mk(1ull, 0ull);
}
__device__ __forceinline__ void lk_close_group(LkRow& st) {
    st.V[st.cur] = eadd(emul(st.V[st.cur], st.ug), emul(st.vg, st.U[st.cur]));
    st.U[st.cur] = emul(st.U[st.cur], st.ug);
    st.vg = mk(0ull, 0ull); st.ug = mk(1ull, 0ull);
}
// interaction k of column col at row r, its flag (1 when it has none), multiplicity and denominator
__device__ __noinline__ void lk_hook(const LookupCheckJitArgs& a, size_t r, LkRow& st, u32 k, u32 col, u64 flag, u64 m, E2 d) {
    if (st.mode == 3) {   // fold_walk: every interaction takes part whatever its flag
        const u32 mark = a.marks ? a.marks[k] : 3u;
        if (mark & 1) lk_close_batch(st);
        if (mark & 2) { lk_close_group(st); st.cur = col; }
        if (mark & 1) st.bf = flag;
        st.bn = eadd(emul(st.bn, d), emulf(st.bd, m));
        st.bd = emul(st.bd, d);
        return;
    }
    if (flag == 0ull) return;   // a zero flag skips the push
    if (a.n_mutex) { const u32 b = a.mutex_pos[k]; if (b != 0xFFFFFFFFu) st.act[b >> 6] |= 1ull << (b & 63); }
    if (st.mode == 0) { st.pushes++; return; }
    const u64 key = balance_key(a.instance, r, k);   // a zero denominator is an ordinary key
    if (st.mode == 1) { balance_add(a, balance_insert(a, d.a, d.b), m, key); return; }
    const u64 s = balance_find(a, d.a, d.b);
    if (a.t_sums[2 * s + 1]) {
        const unsigned long long p = atomicAdd(a.counters + 2, 1ull);
        a.contrib_out[3 * p] = s; a.contrib_out[3 * p + 1] = key; a.contrib_out[3 * p + 2] = m;
    }
}
__device__ __forceinline__ void lk_fold_init(LkRow& st) {
    for (u32 c = 0; c < LK_NC; c++) { st.V[c] = mk(0ull, 0ull); st.U[c] = mk(1ull, 0ull); }
    st.bn = st.vg = mk(0ull, 0ull); st.bd = st.ug = mk(1ull, 0ull); st.bf = 0; st.cur = 0; st.mode = 3;
}
// fold_divide: F[c] = V_c / U_c with one inversion, F[c] = 0 where U_c is zero; the mask of those columns
__device__ __forceinline__ u32 lk_fold_divide(const LkRow& st, E2* F, E2& total) {
    u32 zero_mask = 0;
    E2 acc = mk(1ull, 0ull);
    for (u32 c = 0; c < LK_NC; c++) {
        F[c] = acc;
        if ((st.U[c].a | st.U[c].b) == 0ull) zero_mask |= 1u << c; else acc = emul(acc, st.U[c]);
    }
    E2 inv = einv(acc);
    total = mk(0ull, 0ull);
    for (u32 c = LK_NC; c-- > 0;) {
        if ((zero_mask >> c) & 1) { F[c] = mk(0ull, 0ull); continue; }
        F[c] = emul(st.V[c], emul(inv, F[c]));
        inv = emul(inv, st.U[c]);
        total = eadd(total, F[c]);
    }
    return zero_mask;
}
// fold_verdict: 0 agrees, 1 fraction column, 2 accumulator, 3 zero U
__device__ __forceinline__ u32 lk_fold_verdict(const LookupCheckJitArgs& a, size_t N, size_t r, u32 c, const E2* F, E2 total, u32 zero_mask) {
    E2 expected = F[c], actual = mk(a.aux_cm[(size_t)(2 * c) * N + r], a.aux_cm[(size_t)(2 * c + 1) * N + r]);
    if (c == 0) {
        E2 next = r == N - 1 ? mk(a.final_a, a.final_b) : mk(a.aux_cm[r + 1], a.aux_cm[N + r + 1]);
        expected = total; actual = esub(next, actual);
    }
    const bool eq = expected.a == actual.a && expected.b == actual.b;
    if ((zero_mask >> c) & 1) return 3;
    if (c == 0 ? (zero_mask == 0 && !eq) : !eq) return c ? 1 : 2;
    return 0;
}
)CUDA";
// lookup-check mode: the three entry points, after lk_row (the chunks on one row)
static const char LOOKUP_CHECK_ENTRIES[] = R"CUDA(// k_balance_rows: the pushes of row r by mode, then the row's mutex groups in (column, group) order
extern "C" __global__ void __launch_bounds__(128) k_jit_balance(const KArgs a) {
  const size_t N = (size_t)1 << a.log_n, r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= N) return;
  LkRow st;
  st.mode = a.mode; st.pushes = 0;
  for (u32 w = 0; w < (a.n_mutex + 63) / 64; w++) st.act[w] = 0;
  lk_row(a, r, st);
  if (st.pushes) atomicAdd(a.counters, st.pushes);
  if (!a.n_mutex || a.mode == 2) return;
  u32 cur_g = a.mutex_group[0], cur_s = a.mutex_site[0], cnt = 0;
  bool counted = false;
  for (u32 b = 0;; b++) {
    const bool end = b == a.n_mutex;
    u32 g = end ? 0xFFFFFFFFu : a.mutex_group[b], s = end ? 0xFFFFFFFFu : a.mutex_site[b];
    if (end || g != cur_g) {
      if (cnt > 1) {
        unsigned long long p = atomicAdd(a.counters + 1, 1ull);
        if (a.mode == 1) {
          a.mutex_out[3 * p] = ((u64)a.instance << 32) | r;
          a.mutex_out[3 * p + 1] = ((u64)(cur_g >> 16) << 32) | (cur_g & 0xffffu);
          a.mutex_out[3 * p + 2] = cnt;
        }
      }
      if (end) break;
      cur_g = g; cur_s = s; cnt = 0; counted = false;
    } else if (s != cur_s) { cur_s = s; counted = false; }
    if (!counted && ((st.act[b >> 6] >> (b & 63)) & 1)) { cnt++; counted = true; }
  }
}
// k_fold_rows on rows [row0, row0 + n_rows)
extern "C" __global__ void __launch_bounds__(128) k_jit_fold(const KArgs a) {
  const size_t N = (size_t)1 << a.log_n, r = a.row0 + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.row0 + a.n_rows) return;
  LkRow st;
  lk_fold_init(st);
  lk_row(a, r, st);
  lk_close_batch(st); lk_close_group(st);
  if (a.folds_out && a.folds_cm) {
    for (u32 c = 0; c < LK_NC; c++) {
      u64* o = a.folds_out + (size_t)(4 * c) * N + r;
      o[0] = st.V[c].a; o[N] = st.V[c].b; o[2 * N] = st.U[c].a; o[3 * N] = st.U[c].b;
    }
  } else if (a.folds_out) {
    K2* o = reinterpret_cast<K2*>(a.folds_out) + 2 * r * LK_NC;
    for (u32 c = 0; c < LK_NC; c++) { o[2 * c].x = st.V[c].a; o[2 * c].y = st.V[c].b; o[2 * c + 1].x = st.U[c].a; o[2 * c + 1].y = st.U[c].b; }
  }
  E2 F[LK_NC], total;
  const u32 zero_mask = lk_fold_divide(st, F, total);
  u32 first_c = 0xFFFFFFFFu, n_zero = 0;
  for (u32 c = 0; c < LK_NC; c++) {
    const u32 kind = lk_fold_verdict(a, N, r, c, F, total, zero_mask);
    n_zero += kind == 3;
    if (kind && first_c == 0xFFFFFFFFu) first_c = c;
  }
  if (first_c != 0xFFFFFFFFu) {
    atomicMin(a.first, (unsigned long long)(((u64)r << 32) | first_c));
    atomicAdd(a.failing_rows, 1ull);
  }
  if (n_zero) atomicAdd(a.zero_u, (unsigned long long)n_zero);
}
// k_fold_census_rows: every row's count of disagreeing columns; per column the block's tallies in shared memory, one
// global atomic of each kind per (block, disagreeing column)
extern "C" __global__ void __launch_bounds__(128) k_jit_fold_census(const KArgs a) {
  __shared__ u32 s_cnt[LK_NC], s_zero[LK_NC], s_min[LK_NC], s_max[LK_NC];
  __shared__ u32 s_rows;
  for (u32 c = threadIdx.x; c < LK_NC; c += blockDim.x) { s_cnt[c] = 0; s_zero[c] = 0; s_min[c] = 0xFFFFFFFFu; s_max[c] = 0; }
  if (threadIdx.x == 0) s_rows = 0;
  __syncthreads();
  const size_t N = (size_t)1 << a.log_n, r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < N) {
    LkRow st;
    lk_fold_init(st);
    lk_row(a, r, st);
    lk_close_batch(st); lk_close_group(st);
    E2 F[LK_NC], total;
    const u32 zero_mask = lk_fold_divide(st, F, total);
    u32 n_fail = 0;
    for (u32 c = 0; c < LK_NC; c++) {
      const u32 kind = lk_fold_verdict(a, N, r, c, F, total, zero_mask);
      if (!kind) continue;
      n_fail++;
      atomicAdd(&s_cnt[c], 1u);
      if (kind == 3) atomicAdd(&s_zero[c], 1u);
      atomicMin(&s_min[c], (u32)r); census_max(&s_max[c], (u32)r);
    }
    a.row_count[r] = n_fail;
    if (n_fail) atomicAdd(&s_rows, 1u);
  }
  __syncthreads();
  for (u32 c = threadIdx.x; c < LK_NC; c += blockDim.x) {
    if (!s_cnt[c]) continue;
    atomicAdd(&a.tally[4 * c], (unsigned long long)s_cnt[c]);
    if (s_zero[c]) atomicAdd(&a.tally[4 * c + 1], (unsigned long long)s_zero[c]);
    atomicMin(&a.tally[4 * c + 2], (unsigned long long)s_min[c]);
    census_max(&a.tally[4 * c + 3], (unsigned long long)s_max[c]);
  }
  if (threadIdx.x == 0 && s_rows) atomicAdd(a.failing_rows, (unsigned long long)s_rows);
}
)CUDA";

// ---------------------------------------------------------------------------------------------
// code generation
// ---------------------------------------------------------------------------------------------
struct GenInfo { uint32_t n_constraints = 0; bool uses_sel = false; uint32_t n_chunks = 0, spill_base = 0, spill_ext = 0; };

// `w` is an op-list already validated by compile_oplist (session.cu).
//
// NVRTC's optimiser is superlinear in the size of one function (2 k nodes: 5 s, 10 k nodes: 8 min in one basic
// block), so the arithmetic nodes are cut into chunks of CHUNK nodes, one `__noinline__` device function each.
// Leaves (trace cells, constants, challenges ...) are re-materialised in every chunk that reads them; arithmetic
// values that live across a chunk boundary travel through two small per-thread arrays (Sb: base, Se: extension)
// whose slots are assigned by chunk-granular liveness.
inline uint32_t chunk_nodes() { const char* e = getenv("MDN_JIT_CHUNK"); uint32_t v = e ? (uint32_t)atoi(e) : 0; return v ? v : 512; }

// MODE_LOOKUP: `w` is a lowered LookupAir ("MLKP": 4-word interactions instead of constraint ids) and the
// kernel is the row kernel of build_logup_aux_trace (one (V, U) rational per aux column, see k_logup_rows).
// MODE_CHECK: `w` is a constraint program evaluated on the TRACE domain as CHECK_NODE_CASES does (kernels.cu): raw
// column-major traces with L = N, the raw row-major periodic matrix, selectors exactly 0 or 1.  Each constraint is
// tested instead of folded; a chunk returns its failures' count and least constraint index, so the row's result does
// not depend on the order the chunks visit the constraints in.  Two entry points share the chunks: k_jit_check (the
// semantics of k_check_rows) and k_jit_census (those of k_census_rows).
// MODE_LOOKUP_CHECK: `w` is a lowered LookupAir with `n_cols` columns, read on the trace domain as MODE_LOOKUP reads it.
// Every interaction calls lk_hook (PRELUDE_LOOKUP_CHECK) with its literal index once its operands are defined, in
// interaction order (an interaction never runs in an earlier chunk than the one before it), with one LkRow of per-row
// state passed by reference through the chunks.  Three entry points share the chunks: k_jit_balance (the semantics of
// k_balance_rows, all three modes), k_jit_fold (k_fold_rows) and k_jit_fold_census (k_fold_census_rows).
inline std::string generate(const uint32_t* w, GenInfo* info, Mode mode = MODE_CONSTRAINTS, uint32_t n_cols = 0) {
    const bool lookup = mode == MODE_LOOKUP, check = mode == MODE_CHECK, lkc = mode == MODE_LOOKUP_CHECK;
    const bool interactions = lookup || lkc;   // 4-word interaction items instead of constraint node ids
    const uint32_t nn = w[2], nc = w[3];
    const uint32_t* cons = w + 5 + 3 * (size_t)nn;
    const uint32_t* kw = cons + (interactions ? 4 : 1) * (size_t)nc;
    const uint32_t NOFLAG = 0xFFFFFFFFu;
    // operand nodes of item k (constraint: the node itself; interaction: flag?, multiplicity, denominator)
    auto item_ops = [&](uint32_t k, uint32_t out[3]) -> int {
        if (!interactions) { out[0] = cons[k]; return 1; }
        const uint32_t* it = cons + 4 * (size_t)k;
        int n = 0;
        if (it[1] != NOFLAG) out[n++] = it[1];
        out[n++] = it[2]; out[n++] = it[3];
        return n;
    };
    std::vector<uint8_t> ext(nn, 0), used(nn, 0), leaf(nn, 0);
    bool uses_sel = false;
    auto OP = [&](uint32_t j) { return w[5 + 3 * j]; };
    auto X = [&](uint32_t j) { return w[6 + 3 * j]; };
    auto Y = [&](uint32_t j) { return w[7 + 3 * j]; };
    for (uint32_t j = 0; j < nn; j++) {
        uint32_t op = OP(j);
        if (op >= 10 && op <= 12) ext[j] = ext[X(j)] | ext[Y(j)];
        else if (op == 13) ext[j] = ext[X(j)];
        else { ext[j] = (op == 1 || op == 3 || op == 4 || op == 9); leaf[j] = 1; }
        if (op >= 5 && op <= 7) uses_sel = true;
    }
    for (uint32_t k = 0; k < nc; k++) { uint32_t o[3]; int n = item_ops(k, o); for (int q = 0; q < n; q++) used[o[q]] = 1; }
    for (uint32_t j = nn; j-- > 0;) {
        if (!used[j] || leaf[j]) continue;
        used[X(j)] = 1;
        if (OP(j) != 13) used[Y(j)] = 1;
    }
    // chunk assignment of the arithmetic nodes, in definition order
    const uint32_t NONE = 0xFFFFFFFFu, CHUNK = chunk_nodes();
    std::vector<uint32_t> chunk_of(nn, NONE), last_chunk(nn, 0);
    uint32_t n_arith = 0;
    for (uint32_t j = 0; j < nn; j++) if (used[j] && !leaf[j]) chunk_of[j] = n_arith++ / CHUNK;
    const uint32_t n_chunks = std::max(1u, (n_arith + CHUNK - 1) / CHUNK);
    for (uint32_t j = 0; j < nn; j++) {
        if (chunk_of[j] == NONE) continue;
        last_chunk[j] = std::max(last_chunk[j], chunk_of[j]);
        uint32_t ops[2] = {X(j), OP(j) == 13 ? X(j) : Y(j)};
        for (uint32_t o : ops) if (chunk_of[o] != NONE) last_chunk[o] = std::max(last_chunk[o], chunk_of[j]);
    }
    // every item (constraint fold / interaction) runs in the last chunk that defines one of its operands
    std::vector<uint32_t> item_chunk(nc, 0);
    for (uint32_t k = 0; k < nc; k++) {
        uint32_t o[3]; int n = item_ops(k, o);
        for (int q = 0; q < n; q++) if (chunk_of[o[q]] != NONE) item_chunk[k] = std::max(item_chunk[k], chunk_of[o[q]]);
        if (lkc && k) item_chunk[k] = std::max(item_chunk[k], item_chunk[k - 1]);   // the folds walk interactions in order
        for (int q = 0; q < n; q++) if (chunk_of[o[q]] != NONE) last_chunk[o[q]] = std::max(last_chunk[o[q]], item_chunk[k]);
    }
    // slots for values that cross a chunk boundary
    std::vector<uint32_t> slot(nn, NONE);
    std::vector<std::vector<uint32_t>> defined(n_chunks), dying(n_chunks);
    for (uint32_t j = 0; j < nn; j++) if (chunk_of[j] != NONE && last_chunk[j] > chunk_of[j]) { defined[chunk_of[j]].push_back(j); dying[last_chunk[j]].push_back(j); }
    std::vector<uint32_t> free_b, free_e;
    uint32_t nb = 0, ne = 0;
    for (uint32_t c = 0; c < n_chunks; c++) {
        for (uint32_t j : dying[c]) (ext[j] ? free_e : free_b).push_back(slot[j]);   // read at the top of chunk c, free afterwards
        for (uint32_t j : defined[c]) {
            std::vector<uint32_t>& fl = ext[j] ? free_e : free_b;
            if (!fl.empty()) { slot[j] = fl.back(); fl.pop_back(); } else slot[j] = ext[j] ? ne++ : nb++;
        }
    }
    // NB: a slot freed by a value dying in chunk c may be re-used by a value defined in chunk c; chunk c loads
    // all its live-ins before it stores any live-out, so that is safe.
    char buf[256];
    auto nm = [&](uint32_t j) { char b[24]; snprintf(b, sizeof b, "%c%u", ext[j] ? 'e' : 'b', j); return std::string(b); };
    auto leaf_def = [&](uint32_t j) {
        uint32_t op = OP(j), x = X(j), y = Y(j);
        std::string d = std::string("  const ") + (ext[j] ? "E2 " : "u64 ") + nm(j) + " = ";
        switch (op) {
            case 0: snprintf(buf, sizeof buf, "a.main_lde[(size_t)%u * L + %s];\n", y, x ? "pn" : "pos"); break;
            case 1: snprintf(buf, sizeof buf, "mk(a.aux_lde[(size_t)%u * L + %s], a.aux_lde[(size_t)%u * L + %s]);\n", 2 * y, x ? "pn" : "pos", 2 * y + 1, x ? "pn" : "pos"); break;
            case 2: snprintf(buf, sizeof buf, "a.publics[%u];\n", x); break;
            case 3: snprintf(buf, sizeof buf, "mk(a.challenges[%u], a.challenges[%u]);\n", 2 * x, 2 * x + 1); break;
            case 4: snprintf(buf, sizeof buf, "mk(a.aux_values[%u], a.aux_values[%u]);\n", 2 * x, 2 * x + 1); break;
            case 5: snprintf(buf, sizeof buf, "c.is_first;\n"); break;
            case 6: snprintf(buf, sizeof buf, "c.is_last;\n"); break;
            case 7: snprintf(buf, sizeof buf, "c.is_trans;\n"); break;
            case 8: { uint64_t v = (uint64_t)kw[2 * x] | ((uint64_t)kw[2 * x + 1] << 32); snprintf(buf, sizeof buf, "0x%llxull;\n", (unsigned long long)v); break; }
            case 9: {
                uint64_t v0 = (uint64_t)kw[2 * x] | ((uint64_t)kw[2 * x + 1] << 32), v1 = (uint64_t)kw[2 * x + 2] | ((uint64_t)kw[2 * x + 3] << 32);
                snprintf(buf, sizeof buf, "mk(0x%llxull, 0x%llxull);\n", (unsigned long long)v0, (unsigned long long)v1); break;
            }
            case 14: snprintf(buf, sizeof buf, "a.periodic[(size_t)%u * per_stride + per_idx];\n", x); break;
            case 15: snprintf(buf, sizeof buf, "a.prep_lde[(size_t)%u * L + %s];\n", y, x ? "pn" : "pos"); break;
            default: throw std::runtime_error("jit: unknown leaf op");
        }
        return d + buf;
    };
    auto arith_def = [&](uint32_t j) {
        uint32_t op = OP(j), x = X(j), y = Y(j);
        std::string d = std::string("  const ") + (ext[j] ? "E2 " : "u64 ") + nm(j) + " = ";
        if (op == 13) return d + (ext[x] ? "eneg(" : "fneg(") + nm(x) + ");\n";
        const char* fb = op == 10 ? "fadd" : op == 11 ? "fsub" : "fmul";
        const char* fe = op == 10 ? "eadd" : op == 11 ? "esub" : "emul";
        if (!ext[x] && !ext[y]) return d + fb + "(" + nm(x) + ", " + nm(y) + ");\n";
        if (ext[x] && ext[y]) return d + fe + "(" + nm(x) + ", " + nm(y) + ");\n";
        if (ext[x]) return d + (op == 10 ? "eaddf" : op == 11 ? "esubf" : "emulf") + "(" + nm(x) + ", " + nm(y) + ");\n";
        return d + (op == 10 ? "eaddf" : op == 11 ? "efsub" : "emulf") + "(" + (op == 11 ? nm(x) + ", " + nm(y) : nm(y) + ", " + nm(x)) + ");\n";
    };
    // constraint folds: in the chunk of their node (leaf constraints: chunk 0); weights alpha^(K-1-k) make the
    // order irrelevant
    std::vector<std::vector<uint32_t>> folds(n_chunks);
    for (uint32_t k = 0; k < nc; k++) folds[item_chunk[k]].push_back(k);

    std::string s;
    s.reserve(80 * (size_t)nn + 16384);
    s += PRELUDE;
    s += PRELUDE_FMUL_G2;
    s += PRELUDE_B;
    s += lookup ? PRELUDE_LOOKUP_ARGS : PRELUDE_LOOKUP_ARGS_UNUSED;
    if (check) {
        snprintf(buf, sizeof buf, "#define CENSUS_SHARED_K %uu\n", CENSUS_SHARED_K);
        s += buf;
        s += PRELUDE_CHECK;
    }
    if (lkc) {
        snprintf(buf, sizeof buf, "#define LK_NC %uu\n#define LK_MUTEX_WORDS %uu\n", std::max(1u, n_cols), LOOKUP_CHECK_MUTEX_WORDS);
        s += buf;
        s += PRELUDE_LOOKUP_CHECK;
    }
    s += lookup ? "typedef LookupJitArgs KArgs;\n" : check ? "typedef CheckJitArgs KArgs;\n" : lkc ? "typedef LookupCheckJitArgs KArgs;\n" : "typedef JitArgs KArgs;\n";
    s += "struct Ctx { size_t L, pos, pn, per_idx, per_stride; u64 is_first, is_last, is_trans; };\n";
    std::vector<uint8_t> seen(nn, 0);
    for (uint32_t c = 0; c < n_chunks; c++) {
        if (lookup) snprintf(buf, sizeof buf, "__device__ __noinline__ void chunk%u(const KArgs& a, const Ctx& c, u64* __restrict__ Sb, E2* __restrict__ Se, E2* __restrict__ V, E2* __restrict__ U) {\n", c);
        else if (check) snprintf(buf, sizeof buf, "__device__ __noinline__ u64 chunk%u(const KArgs& a, const Ctx& c, u64* __restrict__ Sb, E2* __restrict__ Se, u32* sh) {\n", c);
        else if (lkc) snprintf(buf, sizeof buf, "__device__ __noinline__ void chunk%u(const KArgs& a, const Ctx& c, u64* __restrict__ Sb, E2* __restrict__ Se, LkRow& st) {\n", c);
        else snprintf(buf, sizeof buf, "__device__ __noinline__ void chunk%u(const KArgs& a, const Ctx& c, u64* __restrict__ Sb, E2* __restrict__ Se, E2& acc) {\n", c);
        s += buf;
        s += "  const size_t L = c.L, pos = c.pos, pn = c.pn, per_idx = c.per_idx, per_stride = c.per_stride;\n"
             "  (void)L; (void)pos; (void)pn; (void)per_idx; (void)per_stride; (void)Sb; (void)Se;\n";
        if (check) s += "  u32 f = 0xFFFFFFFFu, n = 0;   /* least failing constraint, failures */\n";
        // operands needed by this chunk: leaves (re-materialised) and live-in arithmetic values (loaded)
        std::vector<uint32_t> need;
        auto want = [&](uint32_t o) { if (!seen[o]) { seen[o] = 1; need.push_back(o); } };
        for (uint32_t j = 0; j < nn; j++) {
            if (chunk_of[j] != c) continue;
            uint32_t ops[2] = {X(j), OP(j) == 13 ? X(j) : Y(j)};
            for (uint32_t o : ops) if (leaf[o] || chunk_of[o] != c) want(o);
        }
        for (uint32_t k : folds[c]) { uint32_t o[3]; int n = item_ops(k, o); for (int q = 0; q < n; q++) if (leaf[o[q]] || chunk_of[o[q]] != c) want(o[q]); }
        for (uint32_t o : need) {
            if (leaf[o]) s += leaf_def(o);
            else { snprintf(buf, sizeof buf, "  const %s %s = %s[%u];\n", ext[o] ? "E2" : "u64", nm(o).c_str(), ext[o] ? "Se" : "Sb", slot[o]); s += buf; }
            seen[o] = 0;
        }
        for (uint32_t j = 0; j < nn; j++) if (chunk_of[j] == c) s += arith_def(j);
        for (uint32_t k : folds[c]) {
            if (check) {
                uint32_t cn = cons[k];
                std::string nz = ext[cn] ? "(" + nm(cn) + ".a | " + nm(cn) + ".b) != 0ull" : nm(cn) + " != 0ull";
                snprintf(buf, sizeof buf, "  if (%s) { n++; f = f < %uu ? f : %uu; if (a.tally) tally(a, sh, (u32)pos, %uu); }\n", nz.c_str(), k, k, k);
                s += buf;
                continue;
            }
            if (lkc) {
                const uint32_t* it = cons + 4 * (size_t)k;
                auto base = [&](uint32_t j) { return ext[j] ? nm(j) + ".a" : nm(j); };
                const std::string den = ext[it[3]] ? nm(it[3]) : "mk(" + nm(it[3]) + ", 0ull)";
                const std::string flag = it[1] == NOFLAG ? "1ull" : base(it[1]);
                snprintf(buf, sizeof buf, "  lk_hook(a, pos, st, %uu, %uu, %s, %s, %s);\n", k, it[0], flag.c_str(), base(it[2]).c_str(), den.c_str());
                s += buf;
                continue;
            }
            if (!lookup) {
                uint32_t cn = cons[k];
                snprintf(buf, sizeof buf, "  acc = eadd(acc, %s(ldapow(a.apow, %u), %s));\n", ext[cn] ? "emul" : "emulf", k, nm(cn).c_str());
                s += buf;
                continue;
            }
            // ProverGroup::insert (air/src/lookup/prover.rs:338-362): push (multiplicity, denominator) unless the flag is zero
            const uint32_t* it = cons + 4 * (size_t)k;
            std::string den = ext[it[3]] ? nm(it[3]) : "mk(" + nm(it[3]) + ", 0ull)";
            std::string cond = it[1] == NOFLAG ? "true" : nm(it[1]) + " != 0ull";
            s += "  if (" + cond + ") { const E2 d = " + den + "; if ((d.a | d.b) == 0ull) *a.bad_flag = 2u; else { ";
            snprintf(buf, sizeof buf, "V[%u] = eadd(emul(V[%u], d), emulf(U[%u], %s)); U[%u] = emul(U[%u], d); } }\n", it[0], it[0], it[0], nm(it[2]).c_str(), it[0], it[0]);
            s += buf;
        }
        for (uint32_t j : defined[c]) { snprintf(buf, sizeof buf, "  %s[%u] = %s;\n", ext[j] ? "Se" : "Sb", slot[j], nm(j).c_str()); s += buf; }
        if (check) s += "  return (u64)n << 32 | f;\n";
        s += "}\n";
    }
    if (check) {
        // row r of the trace domain: (failures << 32) | least failing constraint (0xFFFFFFFF: none)
        s += "__device__ __forceinline__ u64 check_row(const KArgs& a, size_t r, u32* sh) {\n"
             "  Ctx c;\n"
             "  c.L = (size_t)1 << a.log_n;\n"
             "  c.pos = r;\n"
             "  c.pn = (r + 1) & (c.L - 1);\n"
             "  c.per_idx = (r & (((size_t)1 << a.log_max_period) - 1)) * a.n_periodic;\n"
             "  c.per_stride = 1;\n"
             "  c.is_first = r == 0; c.is_last = r == c.L - 1; c.is_trans = r != c.L - 1;\n";
        snprintf(buf, sizeof buf, "  u64 Sb[%u]; E2 Se[%u];\n  u32 f = 0xFFFFFFFFu, n = 0;\n", std::max(1u, nb), std::max(1u, ne));
        s += buf;
        for (uint32_t c = 0; c < n_chunks; c++) {
            snprintf(buf, sizeof buf, "  { const u64 o = chunk%u(a, c, Sb, Se, sh); n += (u32)(o >> 32); f = f < (u32)o ? f : (u32)o; }\n", c);
            s += buf;
        }
        s += "  return (u64)n << 32 | f;\n"
             "}\n"
             // k_check_rows: a failing row does one atomicMin(first, row << 32 | least k) and counts once
             "extern \"C\" __global__ void __launch_bounds__(128) k_jit_check(const KArgs a) {\n"
             "  const size_t r = a.row0 + (size_t)blockIdx.x * blockDim.x + threadIdx.x;\n"
             "  if (r >= a.row0 + a.n_rows) return;\n"
             "  const u32 f = (u32)check_row(a, r, nullptr);\n"
             "  if (f != 0xFFFFFFFFu) {\n"
             "    atomicMin(a.first, (unsigned long long)(((u64)r << 32) | f));\n"
             "    atomicAdd(a.failing_rows, 1ull);\n"
             "  }\n"
             "}\n"
             // k_census_rows: every row's failure count; per constraint count, least and greatest row, per block in
             // shared memory up to CENSUS_SHARED_K constraints, else straight to the global tally
             "extern \"C\" __global__ void __launch_bounds__(128) k_jit_census(const KArgs a) {\n"
             "  __shared__ u32 s_t[3 * CENSUS_SHARED_K];\n"
             "  __shared__ u32 s_rows;\n"
             "  const bool shared_tally = a.n_cons <= CENSUS_SHARED_K;\n"
             "  if (shared_tally) for (u32 k = threadIdx.x; k < a.n_cons; k += blockDim.x) { s_t[k] = 0; s_t[CENSUS_SHARED_K + k] = 0xFFFFFFFFu; s_t[2 * CENSUS_SHARED_K + k] = 0; }\n"
             "  if (threadIdx.x == 0) s_rows = 0;\n"
             "  __syncthreads();\n"
             "  const size_t N = (size_t)1 << a.log_n, r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;\n"
             "  if (r < N) {\n"
             "    const u32 n = (u32)(check_row(a, r, shared_tally ? s_t : nullptr) >> 32);\n"
             "    a.row_count[r] = n;\n"
             "    if (n) atomicAdd(&s_rows, 1u);\n"
             "  }\n"
             "  __syncthreads();\n"
             "  if (shared_tally) for (u32 k = threadIdx.x; k < a.n_cons; k += blockDim.x) {\n"
             "    if (!s_t[k]) continue;\n"
             "    atomicAdd(&a.tally[3 * k], (unsigned long long)s_t[k]);\n"
             "    atomicMin(&a.tally[3 * k + 1], (unsigned long long)s_t[CENSUS_SHARED_K + k]);\n"
             "    census_max(&a.tally[3 * k + 2], (unsigned long long)s_t[2 * CENSUS_SHARED_K + k]);\n"
             "  }\n"
             "  if (threadIdx.x == 0 && s_rows) atomicAdd(a.failing_rows, (unsigned long long)s_rows);\n"
             "}\n";
        if (info) { info->n_constraints = nc; info->uses_sel = uses_sel; info->n_chunks = n_chunks; info->spill_base = nb; info->spill_ext = ne; }
        return s;
    }
    if (lkc) {
        // row r of the trace domain, the chunks in order on one LkRow
        s += "__device__ __forceinline__ void lk_row(const KArgs& a, size_t r, LkRow& st) {\n"
             "  Ctx c;\n"
             "  c.L = (size_t)1 << a.log_n;\n"
             "  c.pos = r;\n"
             "  c.pn = (r + 1) & (c.L - 1);\n"
             "  c.per_idx = (r & (((size_t)1 << a.log_max_period) - 1)) * a.n_periodic;\n"
             "  c.per_stride = 1;\n"
             "  c.is_first = c.is_last = c.is_trans = 0ull;\n";
        snprintf(buf, sizeof buf, "  u64 Sb[%u]; E2 Se[%u];\n", std::max(1u, nb), std::max(1u, ne));
        s += buf;
        for (uint32_t c = 0; c < n_chunks; c++) { snprintf(buf, sizeof buf, "  chunk%u(a, c, Sb, Se, st);\n", c); s += buf; }
        s += "}\n";
        s += LOOKUP_CHECK_ENTRIES;
        if (info) { info->n_constraints = nc; info->uses_sel = false; info->n_chunks = n_chunks; info->spill_base = nb; info->spill_ext = ne; }
        return s;
    }
    if (lookup) {
        s += "extern \"C\" __global__ void __launch_bounds__(128) k_jit(const KArgs a) {\n"
             "  Ctx c;\n"
             "  c.L = (size_t)1 << a.log_n;\n"
             "  c.pos = (size_t)blockIdx.x * blockDim.x + threadIdx.x;\n"
             "  if (c.pos >= c.L) return;\n"
             "  c.pn = (c.pos + 1) & (c.L - 1);\n"
             "  c.per_idx = (c.pos & (((size_t)1 << a.log_max_period) - 1)) * a.n_periodic;\n"
             "  c.per_stride = 1;\n"
             "  c.is_first = c.is_last = c.is_trans = 0ull;\n";
        snprintf(buf, sizeof buf, "  u64 Sb[%u]; E2 Se[%u];\n  E2 V[%u], U[%u];\n  for (int i = 0; i < %u; i++) { V[i] = mk(0ull, 0ull); U[i] = mk(1ull, 0ull); }\n",
                 std::max(1u, nb), std::max(1u, ne), std::max(1u, n_cols), std::max(1u, n_cols), n_cols);
        s += buf;
        for (uint32_t c = 0; c < n_chunks; c++) { snprintf(buf, sizeof buf, "  chunk%u(a, c, Sb, Se, V, U);\n", c); s += buf; }
        snprintf(buf, sizeof buf, "  E2 t = mk(0ull, 0ull);\n  for (u32 i = 0; i < %uu; i++) {\n", n_cols);
        s += buf;
        s += "    E2 f = V[i];\n"
             "    if (!(U[i].a == 1ull && U[i].b == 0ull)) f = emul(V[i], einv(U[i]));\n"
             "    t = eadd(t, f);\n"
             "    if (i > 0) { a.aux_cm[(size_t)(2 * i) * c.L + c.pos] = f.a; a.aux_cm[(size_t)(2 * i + 1) * c.L + c.pos] = f.b; }\n"
             "  }\n"
             "  a.totals[2 * c.pos] = t.a; a.totals[2 * c.pos + 1] = t.b;\n"
             "}\n";
        if (info) { info->n_constraints = nc; info->uses_sel = false; info->n_chunks = n_chunks; info->spill_base = nb; info->spill_ext = ne; }
        return s;
    }
    s += "extern \"C\" __global__ void __launch_bounds__(128) k_jit(const JitArgs a) {\n"
         "  Ctx c;\n"
         "  c.L = (size_t)1 << (a.log_n + a.log_b);\n"
         "  c.pos = (size_t)blockIdx.x * blockDim.x + threadIdx.x;\n"
         "  { const u32 ct0 = a.pad & 0xffu, cnt = (a.pad >> 8) & 0xffu;   /* cosets [ct0, ct0 + cnt); cnt == 0: all */\n"
         "    if (c.pos >= (cnt ? (size_t)cnt << a.log_n : c.L)) return;\n"
         "    c.pos += (size_t)ct0 << a.log_n; }\n"
         "  const u32 N = 1u << a.log_n;\n"
         "  const u32 t = (u32)(c.pos >> a.log_n), r = (u32)(c.pos & (N - 1));\n"
         "  c.pn = ((size_t)t << a.log_n) + ((r + 1) & (N - 1));\n"
         "  c.per_idx = ((size_t)(r & ((1u << a.log_max_period) - 1)) << a.log_b) | t;\n"
         "  c.per_stride = (size_t)1 << (a.log_max_period + a.log_b);\n"
         "  c.is_first = c.is_last = c.is_trans = 0ull;\n";
    if (uses_sel)
        s += "  {\n"
             "    u64 x = fmul(fmul(a.shift, fpow(a.w_l, t)), fmul(a.w_hi[r >> a.lo_bits], a.w_lo[r & ((1u << a.lo_bits) - 1)]));\n"
             "    u64 d_first = fsub(x, 1ull), d_last = fsub(x, a.w_h_inv);\n"
             "    u64 inv = finv(fmul(d_first, d_last));\n"
             "    c.is_first = fmul(a.zh[t], fmul(inv, d_last));\n"
             "    c.is_last = fmul(a.zh[t], fmul(inv, d_first));\n"
             "    c.is_trans = d_last;\n"
             "  }\n";
    snprintf(buf, sizeof buf, "  u64 Sb[%u]; E2 Se[%u];\n  E2 acc = mk(0ull, 0ull);\n", std::max(1u, nb), std::max(1u, ne));
    s += buf;
    for (uint32_t c = 0; c < n_chunks; c++) { snprintf(buf, sizeof buf, "  chunk%u(a, c, Sb, Se, acc);\n", c); s += buf; }
    s += "  E2 q = emulf(acc, a.inv_zh[t]);\n"
         "  if (a.acc_in) {\n"
         "    const size_t Lin = (size_t)1 << (a.acc_in_log_n + a.log_b);\n"
         "    const size_t pa = ((size_t)t << a.acc_in_log_n) + (r & ((1u << a.acc_in_log_n) - 1));\n"
         "    q = eadd(emul(mk(a.acc_in[pa], a.acc_in[Lin + pa]), mk(a.beta_a, a.beta_b)), q);\n"
         "  }\n"
         "  a.acc_out[c.pos] = q.a;\n"
         "  a.acc_out[c.L + c.pos] = q.b;\n"
         "}\n";
    if (info) { info->n_constraints = nc; info->uses_sel = uses_sel; info->n_chunks = n_chunks; info->spill_base = nb; info->spill_ext = ne; }
    return s;
}

// ---------------------------------------------------------------------------------------------
// NVRTC + driver API, loaded lazily
// ---------------------------------------------------------------------------------------------
struct Nvrtc {
    void* h = nullptr;
    int (*CreateProgram)(void**, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
    int (*CompileProgram)(void*, int, const char* const*) = nullptr;
    int (*GetCUBINSize)(void*, size_t*) = nullptr;
    int (*GetCUBIN)(void*, char*) = nullptr;
    int (*GetProgramLogSize)(void*, size_t*) = nullptr;
    int (*GetProgramLog)(void*, char*) = nullptr;
    int (*DestroyProgram)(void**) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    std::string why; int version = 0;
    bool ok() const { return h != nullptr; }
};
inline Nvrtc& nvrtc() {
    static Nvrtc n;
    static std::once_flag once;
    std::call_once(once, [] {
        // Toolkit paths first: a process that imported torch already holds torch's bundled libnvrtc (12.8 here)
        // under the bare soname, and that build was seen to miscompile large chunk functions (the self-check in
        // tests/run_jit_old_nvrtc.py); a full path loads the toolkit's own copy next to it.
        std::vector<std::string> names;
        for (const char* env : {"MDN_NVRTC_PATH"}) if (const char* v = getenv(env)) names.push_back(v);
        for (const char* env : {"CUDA_HOME", "CUDA_PATH"}) if (const char* v = getenv(env)) names.push_back(std::string(v) + "/lib64/libnvrtc.so.12");
        names.push_back("/usr/local/cuda/lib64/libnvrtc.so.12");
        names.push_back("libnvrtc.so.12");
        for (const std::string& nm : names) {
            void* h = dlopen(nm.c_str(), RTLD_NOW | RTLD_LOCAL);
            if (!h) continue;
            auto ver = (int (*)(int*, int*))dlsym(h, "nvrtcVersion");
            int maj = 0, mn = 0;
            if (ver) ver(&maj, &mn);
            if (maj > 12 || (maj == 12 && mn >= 9) || getenv("MDN_NVRTC_ALLOW_OLD")) { n.h = h; n.version = maj * 100 + mn; n.why.clear(); break; }
            n.why = "libnvrtc " + std::to_string(maj) + "." + std::to_string(mn) + " is older than 12.9";
            dlclose(h);
        }
        if (!n.h && n.why.empty()) n.why = "libnvrtc not found";
        if (!n.h) return;
        auto sym = [&](const char* s) { void* p = dlsym(n.h, s); if (!p) n.why = std::string("missing symbol ") + s; return p; };
        n.CreateProgram = (decltype(n.CreateProgram))sym("nvrtcCreateProgram");
        n.CompileProgram = (decltype(n.CompileProgram))sym("nvrtcCompileProgram");
        n.GetCUBINSize = (decltype(n.GetCUBINSize))sym("nvrtcGetCUBINSize");
        n.GetCUBIN = (decltype(n.GetCUBIN))sym("nvrtcGetCUBIN");
        n.GetProgramLogSize = (decltype(n.GetProgramLogSize))sym("nvrtcGetProgramLogSize");
        n.GetProgramLog = (decltype(n.GetProgramLog))sym("nvrtcGetProgramLog");
        n.DestroyProgram = (decltype(n.DestroyProgram))sym("nvrtcDestroyProgram");
        n.GetErrorString = (decltype(n.GetErrorString))sym("nvrtcGetErrorString");
        if (!n.why.empty()) { dlclose(n.h); n.h = nullptr; }
    });
    return n;
}

// source -> sm_90a cubin (throws std::runtime_error with the compiler log on failure)
inline std::vector<char> compile(const std::string& src) {
    Nvrtc& n = nvrtc();
    if (!n.ok()) throw std::runtime_error("NVRTC unavailable: " + n.why);
    void* prog = nullptr;
    int rc = n.CreateProgram(&prog, src.c_str(), "mdn_constraints.cu", 0, nullptr, nullptr);
    if (rc) throw std::runtime_error(std::string("nvrtcCreateProgram: ") + n.GetErrorString(rc));
    // chunked functions keep NVRTC + ptxas -O3 linear (10 k nodes: 7 s); MDN_JIT_PTXAS overrides the level
    std::vector<const char*> opts = {"--gpu-architecture=sm_90a", "-std=c++17", "-lineinfo", "-default-device"};
    std::string po = std::string("--ptxas-options=") + (getenv("MDN_JIT_PTXAS") ? getenv("MDN_JIT_PTXAS") : "-O3");
    opts.push_back(po.c_str());
    opts.push_back("--device-int128");
    rc = n.CompileProgram(prog, (int)opts.size(), opts.data());
    if (rc) {
        size_t ls = 0; n.GetProgramLogSize(prog, &ls);
        std::string log(ls, '\0'); if (ls) n.GetProgramLog(prog, log.data());
        n.DestroyProgram(&prog);
        throw std::runtime_error(std::string("nvrtcCompileProgram: ") + n.GetErrorString(rc) + "\n" + log.substr(0, 2000));
    }
    size_t sz = 0; n.GetCUBINSize(prog, &sz);
    std::vector<char> cubin(sz);
    n.GetCUBIN(prog, cubin.data());
    n.DestroyProgram(&prog);
    return cubin;
}

struct Driver {
    void* h = nullptr;
    int (*ModuleLoadData)(void**, const void*) = nullptr;
    int (*ModuleGetFunction)(void**, void*, const char*) = nullptr;
    int (*ModuleUnload)(void*) = nullptr;
    int (*LaunchKernel)(void*, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, void*, void**, void**) = nullptr;
    int (*GetErrorString)(int, const char**) = nullptr;
    std::string why;
    bool ok() const { return h != nullptr; }
};
inline Driver& driver() {
    static Driver d;
    static std::once_flag once;
    std::call_once(once, [] {
        d.h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_LOCAL);
        if (!d.h) { d.why = "libcuda.so.1 not found"; return; }
        auto sym = [&](const char* s) { void* p = dlsym(d.h, s); if (!p) d.why = std::string("missing symbol ") + s; return p; };
        d.ModuleLoadData = (decltype(d.ModuleLoadData))sym("cuModuleLoadData");
        d.ModuleGetFunction = (decltype(d.ModuleGetFunction))sym("cuModuleGetFunction");
        d.ModuleUnload = (decltype(d.ModuleUnload))sym("cuModuleUnload");
        d.LaunchKernel = (decltype(d.LaunchKernel))sym("cuLaunchKernel");
        d.GetErrorString = (decltype(d.GetErrorString))sym("cuGetErrorString");
        if (!d.why.empty()) { dlclose(d.h); d.h = nullptr; }
    });
    return d;
}
inline std::string cu_err(int rc) { const char* s = nullptr; if (driver().GetErrorString) driver().GetErrorString(rc, &s); return s ? s : "unknown driver error"; }

struct Kernel {
    std::shared_ptr<void> module;   // shared by the entry points of one cubin (k_jit_check and k_jit_census)
    void* func = nullptr;
    int checked = 0;   // 0: not yet compared with the interpreter, 1: agreed, -1: disagreed (never used again)
    Kernel() {}
    Kernel(const Kernel&) = delete; Kernel& operator=(const Kernel&) = delete;
    // The caller's device must be current and its primary context initialised (any runtime call does that).
    void load(const std::vector<char>& cubin, const char* name = "k_jit") {
        Driver& d = driver();
        if (!d.ok()) throw std::runtime_error("CUDA driver unavailable: " + d.why);
        void* m = nullptr;
        int rc = d.ModuleLoadData(&m, cubin.data());
        if (rc) throw std::runtime_error("cuModuleLoadData: " + cu_err(rc));
        module = std::shared_ptr<void>(m, [](void* p) { if (driver().ok()) driver().ModuleUnload(p); });
        entry(name);
    }
    // another entry point of the module `other` loaded
    void load(const Kernel& other, const char* name) { module = other.module; entry(name); }
    void entry(const char* name) {
        int rc = driver().ModuleGetFunction(&func, module.get(), name);
        if (rc) throw std::runtime_error("cuModuleGetFunction: " + cu_err(rc));
    }
    template <class Args>
    void launch(const Args& a, unsigned blocks, unsigned threads, cudaStream_t st) const {
        void* params[] = {(void*)&a};
        int rc = driver().LaunchKernel(func, blocks, 1, 1, threads, 1, 1, 0, (void*)st, params, nullptr);
        if (rc) throw std::runtime_error("cuLaunchKernel: " + cu_err(rc));
    }
};

// process-wide cubin cache keyed by a hash of the program words (AIRs are fixed per deployment)
inline uint64_t fnv1a(const uint32_t* w, size_t n) {
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < n; i++) { h ^= w[i]; h *= 1099511628211ull; }
    return h;
}
inline const std::vector<char>& cubin_for(const uint32_t* w, size_t n_words, GenInfo* info, Mode mode = MODE_CONSTRAINTS, uint32_t n_cols = 0) {
    static std::mutex mu;
    static std::map<uint64_t, std::pair<std::vector<char>, GenInfo>> cache;
    uint64_t key = fnv1a(w, n_words) ^ (uint64_t)n_words << 40 ^ (uint64_t)chunk_nodes() << 20 ^ (uint64_t)n_cols << 8 ^ (uint64_t)mode;
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it == cache.end()) {
        GenInfo gi;
        std::string src = generate(w, &gi, mode, n_cols);
        if (const char* dump = getenv("MDN_JIT_DUMP")) { if (FILE* f = fopen(dump, "w")) { fwrite(src.data(), 1, src.size(), f); fclose(f); } }
        it = cache.emplace(key, std::make_pair(compile(src), gi)).first;
        if (const char* dump = getenv("MDN_JIT_DUMP_CUBIN")) { if (FILE* f = fopen(dump, "wb")) { fwrite(it->second.first.data(), 1, it->second.first.size(), f); fclose(f); } }
    }
    if (info) *info = it->second.second;
    return it->second.first;
}

}  // namespace jit
