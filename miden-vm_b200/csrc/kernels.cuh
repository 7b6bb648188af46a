// Kernel launch wrappers of the proving path (definitions in kernels.cu).
//
// Device data layout (DESIGN.md "Data layout in HBM"):
//   * every committed matrix is COLUMN-major; an LDE column of a height-N trace has L = B*N
//     entries ordered coset-major: entry t*N + r is the evaluation at x = s * w_L^(r*B + t),
//     i.e. domain (natural) index i = r*B + t.  Coset t is the H-coset s*w_L^t*H in natural order,
//     so "next row" is r+1 and the FRI/Merkle domain index is recovered arithmetically; nothing is
//     ever bit-reverse-permuted in memory (the reference stores bit-reversed rows,
//     prover/commit.rs:118-119; both index the same Merkle leaves by domain index).
//   * coefficient columns (after the inverse NTT) are stored bit-reversed: slot p holds c[bitrev(p)].
//   * extension-field vectors are interleaved (c0, c1) pairs unless noted.
#pragma once
#include "gl.cuh"
#include <cuda_runtime.h>

namespace mk {
using gl::u64;
using gl::u32;
using gl::E2;

// ---------------------------------------------------------------------------------------------
// One proof on G GPUs (DESIGN.md "Multi-GPU"): peer memory instead of collectives.
//   Every rank (one process per GPU) keeps its proof buffers in an arena whose slabs are mapped into every
//   other rank with CUDA IPC; all ranks allocate in the same order, so a buffer has the same offset everywhere
//   and `PeerPtrs` holds the G views of one such buffer (p[rank] = the local one).  Producers STORE their results
//   straight into the consumer's memory over NVLink (leaf digests into the owner of the Merkle leaf range,
//   sub-roots / quotient chunk coefficients / small FRI layers / opened values into every rank), and a
//   device-side flag barrier orders the stores before the consumers' next kernel.  No host round trip and no
//   library collective is on the data path.
//   Partition: rank g owns LDE cosets t in [t0, t0 + nt), nt = B / G (a contiguous slab [t0*N, (t0+nt)*N) of
//   every coset-major LDE column), and the Merkle sub-tree over leaves [g*L/G, (g+1)*L/G).
// ---------------------------------------------------------------------------------------------
static constexpr u32 MAX_RANKS = 8;
struct PeerPtrs { u64* p[MAX_RANKS]; };
// where a kernel's outputs go: 0 = local buffer only (p[rank]), 1 = the rank owning the element (index >> owner_shift),
// 2 = every rank
enum PushMode : u32 { PUSH_LOCAL = 0, PUSH_OWNER = 1, PUSH_ALL = 2 };
struct PushDst { PeerPtrs pp; u32 rank, world, mode, owner_shift; };
inline PushDst local_dst(u64* p) { PushDst d{}; d.pp.p[0] = p; d.rank = 0; d.world = 1; d.mode = PUSH_LOCAL; d.owner_shift = 0; return d; }

// Cross-GPU barrier on the stream: signal every peer's flag slot with `epoch` (release, system scope) and wait until
// every peer has signalled this rank (acquire).  flags.p[g] = rank g's array of MAX_RANKS slots (slot s written by
// rank s).  A wait longer than ~10 s raises bit 8 of *err instead of hanging the device.
void launch_barrier(const PeerPtrs& flags, u32 rank, u32 world, u64 epoch, u32* err, cudaStream_t st);
// src (local) -> the same words of every other rank's view dst.p[g]
void launch_push(const u64* src, const PeerPtrs& dst, u32 rank, u32 world, size_t n, cudaStream_t st);

// ---------------------------------------------------------------------------------------------
// NTT plan for one transform size N = 2^n = N1 * N2 (strided pass of size N1, contiguous pass N2)
// ---------------------------------------------------------------------------------------------
struct NttTables {
    u32 n, n1, n2, lo_bits;
    const u64* tw_n1;       // w_{N1}^i, i < N1/2       (forward)
    const u64* twi_n1;      // inverse roots
    const u64* twi_n2;
    const u64* w_lo;        // w_N^i,               i < 2^lo_bits
    const u64* w_hi;        // w_N^(i << lo_bits),  i < 2^(n - lo_bits)
    const u64* wi_lo;       // inverse
    const u64* wi_hi;
};
// Pre-multiplication tables for a coset base g: premul(j) = g^j / N with j = j2*N1 + j1, one pair per base:
//   tab_b[j1] = g^j1 / N (j1 < N1);
//   tab_c[(1 << s) - 1 + j] = (g^N1)^(N2 / 2^(s+1)) * w_{2^(s+1)}^j: per-stage twiddles of the contiguous pass with
//   the coset shift (g^N1)^j2 folded in (ntt2.cuh); built by ntt_tables.hpp.
struct PremulTables {
    const u64* tab_b;   // n_bases x N1
    const u64* tab_c;   // n_bases x N2 (N2 - 1 used)
};

// d_bad_flag (optional): set to 1 if any value is not a canonical field element (>= p)
void launch_transpose_rm_to_cm(const u64* src_rm, u64* dst_cm, u32 n_rows, u32 width, u32* d_bad_flag, cudaStream_t st);
// Rows [row0, row0 + n_rows_slice) (src_slice points at row row0) -> the same rows of the column-major matrix on EVERY
// rank (dst_cm.p[g], columns of height n_rows_total); a non-canonical value raises bit 0 of every rank's bad.p[g].
void launch_transpose_slice_push(const u64* src_slice, const PeerPtrs& dst_cm, const PeerPtrs& bad, u32 world, u32 row0, u32 n_rows_slice,
                                 u32 n_rows_total, u32 width, cudaStream_t st);
// n words of a column-major device matrix -> the same words of dst_cm, with 16-byte accesses where both pointers allow;
// a non-canonical value raises bit 0 of *d_bad_flag.  src_cm == dst_cm: check only, nothing is stored.
void launch_ingest_cm(const u64* src_cm, u64* dst_cm, size_t n, u32* d_bad_flag, cudaStream_t st);

// In-place inverse NTT of `n_cols` columns (stride col_stride): natural evaluations over H ->
// coefficients (unscaled by 1/N; the forward premul tables carry it), stored bit-reversed.
void launch_intt(u64* cols, size_t col_stride, u32 n_cols, const NttTables& T, cudaStream_t st);

// Forward coset NTTs.  Work item w (0 <= w < n_items): src column items[w].src (bit-reversed
// coefficients, length N), destination items[w].dst (length N, natural order), base id items[w].base.
struct FwdItem { const u64* src; u64* dst; u32 base; u32 pad; };
void launch_fwd_ntt(const FwdItem* d_items, u32 n_items, const NttTables& T, const PremulTables& Pm, cudaStream_t st);

// ---------------------------------------------------------------------------------------------
// Poseidon2 hashing
// ---------------------------------------------------------------------------------------------
struct LeafMat { const u64* base; u32 width; u32 pad; };   // LDE matrix of the group's height
struct LeafArgs { LeafMat m[8]; int n_mats; };
// Absorb one height-group of matrices into the per-leaf sponge states.
//   log_n        : log trace height of this group (leaves handled: B << log_n)
//   prev_states  : SoA [12][B << prev_log_n] states of the previous (shorter) group, or NULL
//   states_out   : SoA [12][B << log_n] if more groups follow, else NULL
//   digests_out  : tree leaf layer (4 u64 per leaf, indexed by DOMAIN index r*B + t), or NULL
//   t0, nt       : only cosets t0 .. t0 + nt are hashed (all rows of each); leaf r*B + t goes to dig (PushDst:
//                  local layer, the rank owning the leaf's sub-tree, or every rank); dig == NULL: no digests
// `perm` selects the permutation of the algebraic configurations: 0 Poseidon2, 3 RPO, 4 RPX (= mdn_hash_kind; rescue.cuh)
void launch_leaf_hash(const LeafArgs& a, u32 log_n, u32 log_blowup, const u64* prev_states, u32 prev_log_n,
                      u64* states_out, const PushDst* dig, u32 t0, u32 nt, cudaStream_t st, int perm = 0);
// parent[i] = perm(child[2i] | child[2i+1] | 0000)[0..4]
void launch_compress_layer(const u64* children, u64* parents, size_t n_parents, cudaStream_t st, int perm = 0);
// FRI round leaves: leaf i' (< quarter) = sponge([f[i'], f[i'+2q], f[i'+q], f[i'+3q]]) (8 felts, one block).
// Only leaves i' with (i' mod 2^log_b) in [t0, t0 + nt) are hashed (t0 = 0, nt = 2^log_b: all).
void launch_fri_leaf_hash(const u64* evals /* EF interleaved */, size_t rows, u32 log_arity, const PushDst& digests,
                          u32 log_b, u32 t0, u32 nt, cudaStream_t st, int perm = 0);
void launch_poseidon2_batch(u64* states, size_t n, cudaStream_t st);
// layers d_from-1 ... lg of the sub-tree of `rank` (heap-ordered tree, 4 u64 per node) in one block; hash_kind = mdn_hash_kind
void launch_compress_top(u64* tree, u32 d_from, u32 lg, u32 rank, int hash_kind, cudaStream_t st);
// The same three tree kernels and the proof-of-work search for the Blake3_256 configuration (air/src/config.rs:276-307):
// chaining leaf hasher (4-lane SoA states), blake3(left || right) nodes, hash-challenger PoW over the challenger's input
// buffer (d_input_words, whole 32-bit words).
void launch_leaf_hash_b3(const LeafArgs& a, u32 log_n, u32 log_blowup, const u64* prev_states, u32 prev_log_n,
                         u64* states_out, const PushDst* dig, u32 t0, u32 nt, cudaStream_t st);
void launch_compress_layer_b3(const u64* children, u64* parents, size_t n_parents, cudaStream_t st);
void launch_fri_leaf_hash_b3(const u64* evals, size_t rows, u32 log_arity, const PushDst& digests, u32 log_b, u32 t0, u32 nt, cudaStream_t st);
void launch_grind_b3(const u32* d_input_words, u32 n_words, u32 bits, u64 start, u64 count, u64* d_result, cudaStream_t st);
// the Keccak configuration: same contracts; the states between height groups are SoA [25][B << log_n]
void launch_leaf_hash_kk(const LeafArgs& a, u32 log_n, u32 log_blowup, const u64* prev_states, u32 prev_log_n,
                         u64* states_out, const PushDst* dig, u32 t0, u32 nt, cudaStream_t st);
void launch_compress_layer_kk(const u64* children, u64* parents, size_t n_parents, cudaStream_t st);
void launch_fri_leaf_hash_kk(const u64* evals, size_t rows, u32 log_arity, const PushDst& digests, u32 log_b, u32 t0, u32 nt, cudaStream_t st);
void launch_grind_kk(const u64* d_input_words, u32 n_words, u32 bits, u64 start, u64 count, u64* d_result, cudaStream_t st);

// ---------------------------------------------------------------------------------------------
// Constraints / quotient
// ---------------------------------------------------------------------------------------------
// Compiled constraint program: 4 words per instruction {op | ext << 8, dst slot, a, b}.  Ops 0..14 as in
// include/miden_b200.h (operands of ADD/SUB/MUL/NEG are SLOTS), 15 = FOLD slot a into the accumulator
// (acc <- acc * alpha + slot), 16 = PREPROCESSED (a = row offset, b = column).  `ext` = 1 selects extension-field arithmetic for ADD/SUB/MUL/NEG.
// Slots are assigned by liveness on the host, so the interpreter's register file is the program's
// maximum number of simultaneously live values, not its node count.
struct AirDev {
    const u32* code;         // 4 words per instruction
    const u64* consts;
    const u64* periodic;     // [col][(r mod max_period) * B + t], or NULL
    u32 n_instr, n_slots;
    u32 uses_selectors;
    u32 log_max_period, n_periodic;
};
struct ConstraintArgs {
    const u64* main_lde; u32 main_width;
    const u64* aux_lde; u32 aux_width_base;
    const u64* prep_lde;     // preprocessed LDE of this AIR (same height as main), or NULL
    u32 log_n, log_blowup;
    AirDev air;
    const u64* publics;      // device
    const u64* challenges;   // device, EF pairs
    const u64* aux_values;   // device, EF pairs
    E2 alpha, beta;
    const u64* acc_in; u32 acc_in_log_n;   // previous accumulator planes [2][B << acc_in_log_n], or NULL
    u64* acc_out;                          // planes [2][B << log_n]
    const NttTables* T;                    // for w_H powers (selectors)
    u32 t0, nt;                            // cosets evaluated: [t0, t0 + nt); nt == 0: all
};
int launch_constraints(const ConstraintArgs& a, cudaStream_t st);   // returns 0 or -1 (program too large)

// ---------------------------------------------------------------------------------------------
// LogUp aux trace on the device (build_logup_aux_trace, reference air/src/lookup/aux_builder.rs:49-97)
// ---------------------------------------------------------------------------------------------
// Compiled lookup program: the constraint instruction format with MAIN/PERIODIC reading the TRACE domain and
// op 17 = EMIT {op, column, flag slot | multiplicity slot << 16, denominator slot} (flag slot 0xffff = none).
// One thread per trace row keeps a rational (V_c, U_c) per aux column (V/U = sum of m/d over the row's
// active interactions), inverts once per column, writes the fraction columns c > 0 and the row total.
struct LogupArgs {
    const u64* main_cm;      // raw main trace, column-major [col][row]
    u32 log_n, n_cols;       // trace height, LookupAir::num_columns
    AirDev prog;             // periodic = RAW periodic matrix, row-major (max_period x n_periodic)
    const u64* publics; const u64* challenges;
    u64* aux_cm;             // aux trace, column-major planes [2c + coord][row]; column 0 is written by the scan
    u64* totals;             // EF interleaved row totals t(r)
    u32* bad_flag;           // set to 2 on a zero denominator
};
int launch_logup_rows(const LogupArgs& a, cudaStream_t st);   // 0, or -1 when the program needs too many slots/columns
// Exclusive prefix sum over EF row totals: acc[r] = sum_{r' < r} t(r') into planes acc0/acc1, grand total into
// final2 (device, 2 u64).  `scratch` needs 2 * ceil(n / 2048) + 2 u64.
void launch_ef_exclusive_scan(const u64* totals, size_t n, u64* acc0, u64* acc1, u64* final2, u64* scratch, cudaStream_t st);
static constexpr u32 LOGUP_MAX_COLS = 16;

// ---------------------------------------------------------------------------------------------
// Constraint check without proving (mdn_check_constraints; reference crates/lifted-stark/src/debug.rs:70-214)
// ---------------------------------------------------------------------------------------------
// The compiled constraint program evaluated on the TRACE domain, one thread per row r of [row0, row0 + n_rows):
// MAIN / AUX / PREPROCESSED read rows r and (r + 1) mod N of the raw column-major buffers, PERIODIC reads row
// r mod max_period of the raw periodic matrix, the selectors are exactly 0 or 1.  FOLD k (op 15) tests constraint k
// instead of folding it: a row where some constraint is non-zero does atomicMin(first, row << 32 | k) with its lowest
// such k and atomicAdd(failing_rows, 1).  With probe_value set, the thread of a row stores constraint probe_k's value.
struct CheckArgs {
    const u64* main_cm;      // raw main trace, column-major [col][row]
    const u64* aux_cm;       // aux trace, column-major planes [2c + coord][row], or NULL (aux_width 0)
    const u64* prep_cm;      // raw preprocessed trace, column-major, or NULL
    u32 log_n;
    AirDev prog;             // periodic = RAW periodic matrix, row-major (max_period x n_periodic)
    const u64* publics; const u64* challenges; const u64* aux_values;   // device; EF pairs for the last two
    size_t row0, n_rows;
    unsigned long long* first;          // init ~0
    unsigned long long* failing_rows;   // init 0
    u32 probe_k; u64* probe_value;      // EF pair, or NULL
};
int launch_check_rows(const CheckArgs& a, cudaStream_t st);   // 0, or -1 when the program needs too many slots

// ---------------------------------------------------------------------------------------------
// DEEP / FRI / misc
// ---------------------------------------------------------------------------------------------
// wvec[i] = y^(bitrev_n(p0 + i)) for i < cnt  (EF interleaved; p0 = 0, cnt = 2^n: the whole vector);
// scratch: 2 * (2^(n - n/2) + 2^(n/2)) u64
void launch_pow_bitrev(E2 y, u32 n, u64* wvec, u64* scratch, size_t p0, size_t cnt, cudaStream_t st);
// partial dot products: out[(col * n_chunks + chunk) * 4 + {0,1}] (point 0), {2,3} (point 1)
void launch_ood_dot(const u64* coef, size_t col_stride, u32 n_cols, u32 n, const u64* w0, const u64* w1,
                    u64* partial, u32 n_chunks, cudaStream_t st);
void launch_ood_reduce(const u64* partial, u32 n_cols, u32 n_chunks, u64* out /* n_cols x 4 */, cudaStream_t st);

struct DeepMat { const u64* base; u32 width; u32 log_n; u32 alpha_off; u32 pad; };
struct DeepArgs {
    const DeepMat* m; int n_mats;   // device array
    u32 log_n_max, log_blowup;
    const u64* apow;         // device: W EF pairs, alpha^(W-1-i)
    u32 total_w;
    E2 z0, z1, fz0, fz1, beta;
    PushDst out;             // EF interleaved, indexed by domain index (local, or stored into every rank)
    const NttTables* T;      // tables of the max height (w_H powers)
    u32 t0, nt;              // cosets evaluated: [t0, t0 + nt); nt == 0: all
};
void launch_deep(const DeepArgs& a, cudaStream_t st);

// next[i'] = fold4([f[i'], f[i'+2q], f[i'+q], f[i'+3q]], s_inv = w_dom^(-i'), beta) for the i' with
// (i' mod 2^log_b) in [t0, t0 + nt)
void launch_fri_fold(const u64* evals, u32 log_dom, u32 log_arity, E2 beta, const PushDst& next, u32 log_b, u32 t0, u32 nt,
                     cudaStream_t st);

// Proof-of-work: smallest w such that the duplexed state has (st[7] & mask) == 0.
//   base_state: 12 u64 with the pending inputs already written at rate[0..in_len) and the rest of
//   the rate holding whatever the sponge holds; the kernel writes w at rate[in_len], zero-fills
//   rate[in_len+1..8), adds (in_len+1) to st[8] and permutes.
void launch_grind(const u64* d_state12, u32 in_len, u32 bits, u64 start, u64 count, u64* d_result /* init ~0 */,
                  cudaStream_t st, int perm = 0);

// sets *flag |= 4 when a[i] != b[i] for some i < n (self-check of the NVRTC constraint kernels)
void launch_compare(const u64* a, const u64* b, size_t n, u32* flag, cudaStream_t st);
void launch_gather(const u64* const* d_ptrs, u64* d_out, size_t n, cudaStream_t st);
// sharded openings: owner[i] < 0: out.p[rank][i] = *ptrs[i]; owner[i] == rank: the value is stored into every rank's
// out.p[g][i]; otherwise rank owner[i] provides it
void launch_gather_push(const u64* const* d_ptrs, const int* d_owner, const PeerPtrs& out, u32 rank, u32 world, size_t n, cudaStream_t st);

// test/export helper: LDE (coset-major columns) -> row-major with bit-reversed rows
void launch_export_lde_bitrev_rm(const u64* lde, u32 log_n, u32 log_blowup, u32 width, u64* out_rm, cudaStream_t st);

void upload_constants();   // Poseidon2 round constants -> __constant__
unsigned long long launch_count();
void count_launch();   // for kernels launched outside kernels.cu (the NVRTC constraint kernels)
void reset_launch_count();

}  // namespace mk
