// Host orchestration of the proving path + the C ABI (include/miden_b200.h).
//
// This file mirrors `miden_lifted_stark::prover::prove` (reference
// crates/lifted-stark/src/prover/mod.rs:230-578) phase by phase; each phase names the reference
// lines it replaces.  Everything data-parallel runs in the kernels of kernels.cu; the host keeps
// the Fiat-Shamir transcript (sequential) exactly like the reference's host does.
#include "../../include/miden_b200.h"
#include "host_transcript.hpp"
#include "kernels.cuh"
#include "ntt_tables.hpp"
#include "jit.hpp"
#include <array>
#include <cstddef>

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

using gl::E2;
using gl::u32;
using gl::u64;
using hostfs::Duplex;
using hostfs::Indices;
using hostfs::Transcript;

namespace {

struct MdnError : std::runtime_error {
    int code;
    MdnError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
[[noreturn]] void fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    throw MdnError(code, buf);
}
#define CUDA_OK(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) fail(MDN_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

// MDN_FLAG_COLUMN_MAJOR is set; it is only valid together with MDN_FLAG_DEVICE_TRACES
bool column_major(uint32_t flags) {
    if (!(flags & MDN_FLAG_COLUMN_MAJOR)) return false;
    if (!(flags & MDN_FLAG_DEVICE_TRACES)) fail(MDN_ERR_INVALID_ARG, "MDN_FLAG_COLUMN_MAJOR is only valid together with MDN_FLAG_DEVICE_TRACES");
    return true;
}
// a column-major device matrix with cells has a 16-byte aligned base pointer (the ingest reads it in 16-byte words)
void check_column_major(const mdn_matrix& m, const char* what, uint32_t i) {
    if (!m.width) return;
    if (!m.values) fail(MDN_ERR_INVALID_ARG, "%s %u is NULL", what, i);
    if ((uintptr_t)m.values & 15) fail(MDN_ERR_INVALID_ARG, "%s %u: a column-major device matrix must be 16-byte aligned", what, i);
}

std::string g_create_error;

// Proof-lifetime device memory.  Every buffer a proof allocates is gone when the proof ends, and a prover proves
// the same shapes over and over, so the session owns slabs obtained once with cudaMalloc and hands out blocks by
// bumping (plus size-keyed reuse of blocks released mid-proof); at the end of a proof the bump pointers go back
// to zero.  After the first proof of a shape no allocation reaches the driver.  The stream-ordered pool this
// replaces had to re-map physical memory whenever its free space was fragmented when a 1 GB request arrived --
// a driver call that can stall for tens of milliseconds under a loaded neighbour.
// Blocks are used on the session's stream only (the copy stream is ordered behind it by events), so handing a
// released block to the next request is safe in stream order.
struct Arena {
    struct Slab { char* base; size_t size, used; };
    std::vector<Slab> slabs;
    std::multimap<size_t, char*> free_blocks;
    size_t live = 0, grow_events = 0;
    // One proof on several GPUs: every rank runs the same allocation sequence, so a block has the same slab index and
    // offset on every rank; the hooks map a new slab into the peers (CUDA IPC) and unmap before slabs are freed.
    std::function<void(char*, size_t)> on_new_slab;
    std::function<void()> before_drop_slabs;
    static size_t round_up(size_t b) { return (b + 511) & ~(size_t)511; }
    void* alloc(size_t bytes) {
        bytes = round_up(bytes);
        auto it = free_blocks.lower_bound(bytes);
        if (it != free_blocks.end() && it->first <= bytes + bytes / 4) { void* p = it->second; free_blocks.erase(it); live++; return p; }
        for (Slab& sl : slabs) if (sl.size - sl.used >= bytes) { void* p = sl.base + sl.used; sl.used += bytes; live++; return p; }
        size_t sz = std::max(bytes, (size_t)1 << 30);
        char* base = nullptr;
        CUDA_OK(cudaMalloc((void**)&base, sz));
        slabs.push_back(Slab{base, sz, bytes});
        grow_events++; live++;
        if (on_new_slab) on_new_slab(base, sz);
        return base;
    }
    void free(void* p, size_t bytes) { free_blocks.emplace(round_up(bytes), (char*)p); live--; }
    // end of a proof: everything must have been released; several slabs are merged into one of the total size
    void reset() {
        if (live) return;
        free_blocks.clear();
        for (Slab& sl : slabs) sl.used = 0;
        if (slabs.size() > 1) {
            size_t total = 0;
            for (Slab& sl : slabs) total += sl.size;
            if (before_drop_slabs) before_drop_slabs();
            for (Slab& sl : slabs) cudaFree(sl.base);
            slabs.clear();
            char* base = nullptr;
            if (cudaMalloc((void**)&base, total) == cudaSuccess) { slabs.push_back(Slab{base, total, 0}); if (on_new_slab) on_new_slab(base, total); }
            else cudaGetLastError();   // the next proof grows again
        }
    }
    void destroy() { if (before_drop_slabs && !slabs.empty()) before_drop_slabs(); for (Slab& sl : slabs) cudaFree(sl.base); slabs.clear(); free_blocks.clear(); live = 0; }
};
thread_local Arena* tl_arena = nullptr;   // set while an API call works on a proof
struct ArenaScope { Arena* prev; explicit ArenaScope(Arena* a) : prev(tl_arena) { tl_arena = a; } ~ArenaScope() { tl_arena = prev; } };

// device buffer: from the proof arena when one is active, else stream-ordered (persistent tables, tools)
struct DevBuf {
    u64* p = nullptr; size_t n = 0; cudaStream_t st = nullptr; Arena* owner = nullptr;
    DevBuf() {}
    DevBuf(const DevBuf&) = delete; DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept { p = o.p; n = o.n; st = o.st; owner = o.owner; o.p = nullptr; o.n = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept { release(); p = o.p; n = o.n; st = o.st; owner = o.owner; o.p = nullptr; o.n = 0; return *this; }
    void alloc(size_t count, cudaStream_t s) {
        release(); st = s; n = count; owner = tl_arena;
        if (!count) return;
        if (owner) p = (u64*)owner->alloc(count * sizeof(u64));
        else CUDA_OK(cudaMallocAsync((void**)&p, count * sizeof(u64), s));
    }
    void release() {
        if (!p) return;
        if (owner) owner->free(p, n * sizeof(u64)); else cudaFreeAsync(p, st);
        p = nullptr; n = 0;
    }
    ~DevBuf() { release(); }
};

struct NttPlan {
    mk::NttTables T;
    DevBuf store;
};
struct PremulPlan {
    mk::PremulTables P;
    DevBuf store;
    u32 n_bases;
};

enum ProfCat { PC_TRANSPOSE = 0, PC_NTT, PC_LEAF, PC_COMPRESS, PC_CONSTRAINTS, PC_OOD, PC_DEEP, PC_FRI, PC_GRIND, PC_GATHER, PC_COUNT };
struct Prof {
    std::vector<cudaEvent_t> pool;
    struct Region { int cat; size_t e0, e1; };
    std::vector<Region> regions;
    size_t used = 0;
    cudaStream_t st = nullptr;
    size_t ev() { if (used == pool.size()) { cudaEvent_t e; cudaEventCreate(&e); pool.push_back(e); } return used++; }
    size_t begin(int cat) { size_t a = ev(); cudaEventRecord(pool[a], st); regions.push_back({cat, a, a}); return regions.size() - 1; }
    void end(size_t r) { size_t b = ev(); cudaEventRecord(pool[b], st); regions[r].e1 = b; }
    void reset() { used = 0; regions.clear(); }
    void resolve(float* ms, unsigned* counts) {
        for (int i = 0; i < PC_COUNT; i++) { ms[i] = 0; counts[i] = 0; }
        for (auto& r : regions) { float t = 0; cudaEventElapsedTime(&t, pool[r.e0], pool[r.e1]); ms[r.cat] += t; counts[r.cat]++; }
    }
    ~Prof() { for (auto e : pool) cudaEventDestroy(e); }
};
struct ProfScope { Prof& p; size_t r; ProfScope(Prof& p_, int cat) : p(p_), r(p_.begin(cat)) {} ~ProfScope() { p.end(r); } };

struct Tree {
    DevBuf nodes;   // heap layout: layer d at ((1<<d)-1)*4, 4 u64 per digest
    u32 depth = 0;
    u64* layer(u32 d) { return nodes.p + (((size_t)1 << d) - 1) * 4; }
};

struct CommittedMat { u64* lde; u64* coef; u32 log_n, width; };
struct Committed {
    DevBuf lde_buf, coef_buf;
    std::vector<CommittedMat> mats;   // proof order (ascending height)
    Tree tree;
    u64 root[4];
};

// The row passes that can run on an NVRTC-specialised kernel (jit.hpp) instead of the op-list interpreter, and the note
// each leaves in jit_note when its kernel disagrees with the interpreter on its first use in a session.
enum JitPass : u32 { JIT_PROOF, JIT_LOGUP, JIT_CHECK, JIT_CENSUS, JIT_BALANCE, JIT_FOLD, JIT_FOLD_CENSUS, JIT_PASSES };
const char CHECK_DISAGREED[] = "NVRTC check kernel disagreed with the interpreter on its first use; interpreter kept";
const char LOOKUP_CHECK_DISAGREED[] = "NVRTC lookup-check kernel disagreed with the interpreter on its first use; interpreter kept";
const char* const JIT_DISAGREED[JIT_PASSES] = {
    "NVRTC kernel disagreed with the interpreter on its first use; interpreter kept",          // constraint evaluation
    "NVRTC lookup kernel disagreed with the interpreter on its first use; interpreter kept",   // LogUp aux build
    CHECK_DISAGREED, CHECK_DISAGREED,                                                          // check and guard, census
    LOOKUP_CHECK_DISAGREED, LOOKUP_CHECK_DISAGREED, LOOKUP_CHECK_DISAGREED};                   // balance, folds, fold census

struct AirHost {
    mdn_air desc;
    DevBuf program;   // nodes | constraints | consts(lo,hi pairs as u64)
    mk::AirDev dev;
    // lowered LookupAir (mdn_air.lookup): compiled program, raw periodic matrix, and the raw column-major main
    // trace kept from before the in-place inverse NTT (the LogUp fractions are evaluated on the trace domain):
    // raw_main_cm points at the copy in raw_main, or at the caller's column-major device trace (MDN_FLAG_COLUMN_MAJOR).
    // Under the constraint guard every AIR keeps its raw main trace, and raw_periodic holds its raw periodic matrix.
    bool has_lookup = false;
    DevBuf lookup_program, raw_main, raw_periodic;
    const u64* raw_main_cm = nullptr;
    mk::AirDev lookup_dev;
    // lookup_prep: the lookup program's interaction part reads preprocessed columns (op 15); reg_prep: its register
    // updates do (a proof's LogUp build then needs the rows; the lookup checks, which build no registers, do not).  raw_prep: the raw column-major rows of the
    // installed bundle's preprocessed trace of this AIR, derived once per proof or check (mdn_session::bundle_prep_rows)
    bool lookup_prep = false, reg_prep = false;
    DevBuf raw_prep;
    // lookup_v1: the lookup program's interaction part as a version-1 program, which the LogUp build and the three
    // lookup checks run (the caller's words for a version-1 program, lookup_words for a version-2 one).
    // lookup_cols: its LogUp columns.  A version-2 program's n_regs register columns follow them, built from the
    // compiled register program reg_dev (kernels.cuh RegisterArgs; it shares lookup_dev's periodic matrix).
    mdn_lookup lookup_v1{};
    std::vector<u32> lookup_words;
    u32 lookup_cols = 0, n_regs = 0;
    DevBuf reg_program;
    mk::AirDev reg_dev{};
    // per row pass, the NVRTC kernel of a large program (mdn_session::load_jit); NULL = interpreter.  The proof's
    // kernels are loaded for a proof, the check and census kernels for the checks and a guarded proof, the three
    // lookup-check kernels by the lookup checks only (load_lookup_check_jit).
    std::array<std::shared_ptr<jit::Kernel>, JIT_PASSES> jit;
    u32 n_constraints = 0;
};

}  // namespace

struct mdn_session {
    mdn_pcs_params params;
    int device = 0;
    cudaStream_t stream = nullptr;
    std::string error;
    // ONE proof on G ranks (mdn_session_set_shard; kernels.cuh "One proof on G GPUs"): rank g computes LDE cosets
    // [g*B/G, (g+1)*B/G) of every column -- forward NTTs, leaf sponge, constraints, DEEP, FRI folds -- and the Merkle
    // sub-tree over leaves [g*L/G, (g+1)*L/G).  Results cross ranks as peer-memory stores ordered by a device-side
    // barrier; the host callback is only the bootstrap transport for the CUDA IPC handles.
    u32 shard_rank = 0, shard_world = 1, shard_log_g = 0;
    mdn_allgather_fn allgather = nullptr; void* allgather_ctx = nullptr;
    bool shard_active = false;                     // inside a proof that is split over the ranks
    u32 shard_min_log = 10;                        // FRI layers below 2^shard_min_log leaves are replicated (MDN_SHARD_MIN_LOG)
    struct SlabView { char* base[mk::MAX_RANKS]; size_t size; };
    std::vector<SlabView> slab_views;              // every rank's mapping of arena slab i
    u64* sync_local = nullptr; mk::PeerPtrs sync_flags{}; u64 sync_epoch = 0;
    bool sharded() const { return shard_active && shard_world > 1; }
    bool tree_sharded(u32 depth) const { return sharded() && depth >= shard_log_g + 6; }
    bool fri_layer_sharded(u32 log_dom) const {    // domain 2^log_dom split by coset: folds and leaves stay rank-local
        const u32 la = params.log_folding_arity, lb = params.log_blowup;
        return sharded() && log_dom >= la + lb && log_dom >= la + shard_min_log;
    }
    u32 nt() const { return sharded() ? (1u << params.log_blowup) >> shard_log_g : (1u << params.log_blowup); }   // cosets of this rank
    u32 t0() const { return sharded() ? shard_rank * nt() : 0; }
    int coset_owner(u32 t) const { return sharded() ? (int)(t / nt()) : -1; }
    // STARK hash configuration (mdn_session_set_hash): Poseidon2 sponge + duplex challenger (default) or Blake3 chaining
    // hasher + hash challenger (air/src/config.rs:276-307).  `align` = LMCS alignment: 8 (sponge rate) or 1 (chaining).
    int hash_kind = MDN_HASH_POSEIDON2;
    u32 align() const { return hash_kind == MDN_HASH_BLAKE3 ? 1u : hash_kind == MDN_HASH_KECCAK ? 17u : 8u; }
    bool byte_hash() const { return hash_kind == MDN_HASH_BLAKE3 || hash_kind == MDN_HASH_KECCAK; }     // hash challenger, not the duplex one
    int perm() const { return byte_hash() ? 0 : hash_kind; }                                             // rescue.cuh permutations share the Poseidon2 kernels
    // Compression layers d_from-1 ... lg of the sub-tree of `rank` (the whole tree: lg = 0, rank = 0): one launch per layer while a
    // layer has more than 512 nodes, then ONE single-block launch for the rest (mk::launch_compress_top).  Returns the permutations.
    size_t compress_subtree(Tree& t, u32 d_from, u32 lg, u32 rank) {
        static constexpr u32 TOP = 10;
        size_t n_perm = 0;
        u32 d = d_from;
        for (; d > lg && d - 1 - lg >= TOP; d--) {
            size_t cnt = (size_t)1 << (d - 1 - lg), start = (size_t)rank << (d - 1 - lg);
            n_perm += cnt;
            compress_layer(t.layer(d) + 2 * start * 4, t.layer(d - 1) + start * 4, cnt);
        }
        if (d > lg) { n_perm += ((size_t)1 << (d - lg)) - 1; mk::launch_compress_top(t.nodes.p, d, lg, rank, hash_kind, stream); }
        return n_perm;
    }
    u32 state_words() const { return hash_kind == MDN_HASH_KECCAK ? 25u : 12u; }      // leaf state handed on between height groups
    std::vector<uint8_t> hash_ch_in, hash_ch_out;          // pre-bound HashChallenger state (mdn_session_set_hash_challenger)
    void hash_leaves(const mk::LeafArgs& a, u32 ln, u32 lb, const u64* prev, u32 prev_log, u64* states_out, const mk::PushDst* dig, u32 tb, u32 tn) {
        if (hash_kind == MDN_HASH_BLAKE3) mk::launch_leaf_hash_b3(a, ln, lb, prev, prev_log, states_out, dig, tb, tn, stream);
        else if (hash_kind == MDN_HASH_KECCAK) mk::launch_leaf_hash_kk(a, ln, lb, prev, prev_log, states_out, dig, tb, tn, stream);
        else mk::launch_leaf_hash(a, ln, lb, prev, prev_log, states_out, dig, tb, tn, stream, perm());
    }
    void compress_layer(const u64* children, u64* parents, size_t n) {
        if (hash_kind == MDN_HASH_BLAKE3) mk::launch_compress_layer_b3(children, parents, n, stream);
        else if (hash_kind == MDN_HASH_KECCAK) mk::launch_compress_layer_kk(children, parents, n, stream);
        else mk::launch_compress_layer(children, parents, n, stream, perm());
    }
    mdn_external_check external_check = nullptr; void* external_ctx = nullptr;   // Statement::eval_external (mdn_session_set_external_check)
    mdn_aux_builder_device dev_aux = nullptr; void* dev_aux_ctx = nullptr;        // mdn_session_set_device_aux_builder
    // mdn_session_set_constraint_guard: every proof checks its rows before the aux commitment; guard_report is the
    // report of the last guard run (mdn_last_constraint_report)
    bool constraint_guard = false;
    mdn_constraint_report guard_report{1, 0, 0, 0, 0, {0, 0}, 0};
    void shard_map_slab(char* base, size_t size);
    void shard_unmap_slabs();
    void shard_teardown();
    void shard_barrier();
    void shard_check(const char* where);
    // the same check folded into a stream synchronisation the caller performs anyway: enqueue the copy of the barrier
    // flag before that synchronisation, evaluate it after (one host round trip less per commitment of a split proof)
    u32 shard_flag_host = 0;
    void shard_check_enqueue();
    void shard_check_finish(const char* where);
    mk::PeerPtrs peers_of(const u64* p) const;
    mk::PushDst push_dst(u64* p, u32 mode, u32 owner_shift = 0) const;
    std::map<u32, std::unique_ptr<NttPlan>> ntt_plans;
    std::map<std::pair<u32, u32>, std::unique_ptr<PremulPlan>> premul_plans;   // (n, kind)

    // ---- per-proof state ----
    Arena arena;
    bool use_arena = getenv("MDN_NO_ARENA") == nullptr;   // off: every buffer is its own allocation (compute-sanitizer memcheck)
    void release_proof_memory();
    bool in_proof = false;
    bool col_major = false;                 // the proof's traces (and staged aux matrices) are column-major device buffers
    std::vector<AirHost> airs;              // instance order
    std::vector<u32> log_heights;           // instance order
    std::vector<u32> order;                 // proof position -> instance
    std::vector<u64> publics;
    u32 log_max_n = 0;
    u32 log_qd = 0;                         // max log_quotient_degree over the AIRs (number of quotient chunks)
    Transcript tr;
    std::vector<E2> randomness;
    Committed main_c, aux_c, quot_c;
    // Preprocessed bundle (mdn_session_set_preprocessed): persists across proofs like the reference's borrowed
    // `Preprocessed` (preprocessed.rs:49-61).  prep_air[q] = instance of committed preprocessed trace q.
    // constraint JIT: programs with at least jit_min_nodes nodes are compiled with NVRTC (0 = never)
    u32 jit_min_nodes = 256;
    std::map<u64, std::shared_ptr<jit::Kernel>> jit_kernels;   // loaded modules by program hash
    std::vector<u64> jit_used;       // per AIR of the last proof: 1 = JIT kernel, 0 = interpreter
    std::vector<u64> jit_check_used; // per AIR (instance order) of the last constraint check, census or guard run: the same
    std::vector<u64> jit_lookup_check_used;   // per AIR (instance order) of the last lookup check: the same
    struct JitEntry { JitPass pass; const char* name; u64 salt; };
    void load_jit(AirHost& h, const u32* w, u32 n_words, jit::Mode mode, u32 n_cols, std::initializer_list<JitEntry> entries);
    void load_lookup_check_jit();
    // The first-use self-check shared by every NVRTC row pass.  row_kernel: AIR h's kernel for pass p, or NULL for the
    // interpreter (a kernel that disagreed earlier in the session is dropped); launch_jit: one thread per row in
    // 128-thread blocks; unchecked: its first use, when the caller runs the interpreter into twin buffers as well.
    static jit::Kernel* row_kernel(AirHost& h, JitPass p) {
        std::shared_ptr<jit::Kernel>& kn = h.jit[p];
        if (kn && kn->checked < 0) kn.reset();
        return kn.get();
    }
    static bool unchecked(const jit::Kernel& kn) { return kn.checked == 0; }
    template <class Args> void launch_jit(const jit::Kernel& kn, const Args& a, size_t rows) {
        try { kn.launch(a, (unsigned)((rows + 127) / 128), 128, stream); }
        catch (const std::exception& e) { fail(MDN_ERR_CUDA, "%s", e.what()); }
        mk::count_launch();
    }
    bool settle_jit(jit::Kernel& kn, JitPass p, bool differs, u64* used, bool promote = true);
    struct Twin { u64* kernel; const u64* interp; size_t n; };   // n words the kernel and the interpreter wrote
    bool compare_jit(jit::Kernel& kn, JitPass p, u64* used, std::initializer_list<Twin> twins, bool all_ranks = false);
    bool alloc_if_free(std::initializer_list<std::pair<DevBuf*, size_t>> bufs);
    std::string jit_note;            // why the JIT was not used, if it was wanted
    Committed prep_c; bool has_prep = false;
    std::vector<u32> prep_air, prep_log_h;
    void set_preprocessed(const mdn_statement* st, const mdn_matrix* mats);
    std::vector<std::vector<u64>> aux_values_p;   // proof order, EF pairs
    DevBuf d_publics, d_randomness, d_aux_values, d_flag;
    void check_input_flag(const char* what);
    std::vector<size_t> aux_values_off;           // proof order offsets (in u64) into d_aux_values
    // outputs
    std::vector<uint8_t> out_heights;
    std::vector<u64> out_fields, out_commitments;
    // introspection
    E2 ood_z{0, 0};
    u64 dbg_roots[3][4] = {};
    std::vector<u64> dbg_quot_acc, dbg_deep, dbg_fri_roots, dbg_queries;
    bool keep_debug = false;
    mdn_timings timings{};
    cudaEvent_t ev[16];
    Prof prof;
    double leaf_bytes = 0, ntt_bytes = 0; unsigned long long perms = 0;

    NttPlan& ntt(u32 n);
    PremulPlan& premul_trace(u32 n);
    PremulPlan& premul_quotient(u32 n, u32 log_d);
    PremulPlan& premul_unshifted(u32 n);
    void build_tree(Committed& c);
    void lde_matrix(CommittedMat& m);
    void keep_raw_main(u32 j, const u64* caller_cm);
    const u64* bundle_prep_rows(u32 i);
    void check_bundle_prep(u32 i);
    // registers == false: the LogUp columns only (the lookup checks, which compare no register column)
    void build_logup_aux(u32 j, const u64* main_cm, const u64* prep_cm, u64* aux_cm, u64 final_out[2], bool registers = true);
    void lde_and_commit(Committed& c, float* t_lde, float* t_hash, bool lde_done = false);
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t copy_ev[8];
    // pinned bounce buffers for pageable host inputs (a Rust Vec<Felt> is pageable)
    u64* bounce[2] = {nullptr, nullptr}; cudaEvent_t bounce_ev[2]; bool bounce_busy[2] = {false, false};
    static constexpr size_t BOUNCE_WORDS = (size_t)4 << 20;   // 32 MiB each
    void host_to_device(u64* dst, const u64* src, size_t n);
    void upload_matrix(const mdn_matrix& m, bool on_device, u64* dst_cm, bool col_major = false);
    void prove_begin(const mdn_statement* st, const mdn_matrix* traces, const mdn_challenger* ch, u32 flags);
    void validate_statement(const mdn_statement* st, const mdn_matrix* traces, const mdn_challenger* ch);
    void bind_airs(const mdn_statement* st, const mdn_matrix* traces, bool jit, bool check_jit);
    void bind_order(const mdn_statement* st, bool tables);
    void bind_challenger(const mdn_challenger* ch);
    void upload_and_commit_main(const mdn_matrix* traces, bool on_device);
    int eval_external(u32* failed);
    // what every trace check starts with (start_check) and the pieces its callers share
    struct CheckStart { bool cm, on_device; u32 k; };
    CheckStart start_check(const mdn_statement* st, const mdn_matrix* traces, const mdn_challenger* ch, u32 flags, const void* out, bool check_jit = false);
    std::vector<u64*> stage_main(const mdn_matrix* traces, const std::vector<u32>& insts, bool cm, bool on_device);
    u32 check_randomness(const u64* rnd);
    void upload_leaves(const u64* rnd, size_t n_words);
    void alloc_checked(const std::string& what, std::initializer_list<std::pair<DevBuf*, size_t>> bufs);
    bool lookup_air(u32 i, const char* given, u32& skipped);
    // the row program's inputs of AIR i (proof position j) for k_check_rows and k_census_rows, whose argument structs
    // name them alike; `values`: the aux values in proof order
    template <class Args> Args row_args(u32 i, u32 j, const u64* main_cm, const u64* prep_cm, const u64* periodic, const u64* values) const {
        const AirHost& h = airs[i];
        Args c{};
        c.main_cm = main_cm;
        c.aux_cm = h.desc.aux_width ? aux_c.mats[j].coef : nullptr;
        c.prep_cm = prep_cm;
        c.log_n = log_heights[i];
        c.prog = h.dev;
        c.prog.periodic = periodic;
        c.publics = d_publics.p; c.challenges = d_randomness.p; c.aux_values = values + aux_values_off[j];
        return c;
    }
    // the same inputs for the NVRTC trace-check kernels (jit.hpp CheckJitArgs); the result pointers are the caller's
    static_assert(jit::CENSUS_SHARED_K == mk::CENSUS_SHARED_K, "k_jit_census tallies in shared memory as k_census_rows does");
    template <class Args> static jit::CheckJitArgs check_jit_args(const Args& c) {
        jit::CheckJitArgs ja{};
        ja.main_lde = c.main_cm; ja.aux_lde = c.aux_cm; ja.prep_lde = c.prep_cm;
        ja.publics = c.publics; ja.challenges = c.challenges; ja.aux_values = c.aux_values; ja.periodic = c.prog.periodic;
        ja.log_n = c.log_n; ja.n_periodic = c.prog.n_periodic; ja.log_max_period = c.prog.log_max_period;
        return ja;
    }
    // the same inputs for the NVRTC lookup-check kernels (jit.hpp LookupCheckJitArgs), one per interpreter struct
    template <class Args> static jit::LookupCheckJitArgs lookup_check_args(const Args& b) {
        jit::LookupCheckJitArgs ja{};
        ja.main_lde = b.main_cm; ja.prep_lde = b.prep_cm; ja.publics = b.publics; ja.challenges = b.challenges;
        ja.periodic = b.prog.periodic; ja.log_n = b.log_n; ja.n_periodic = b.prog.n_periodic; ja.log_max_period = b.prog.log_max_period;
        return ja;
    }
    static jit::LookupCheckJitArgs balance_jit_args(const mk::BalanceArgs& b) {
        jit::LookupCheckJitArgs ja = lookup_check_args(b);
        ja.mutex_pos = b.mutex_pos; ja.mutex_group = b.mutex_group; ja.mutex_site = b.mutex_site; ja.n_mutex = b.n_mutex;
        ja.t_keys = b.t.keys; ja.t_sums = b.t.sums; ja.t_count = b.t.count; ja.t_first = b.t.first; ja.t_mask = b.t.mask;
        ja.counters = b.counters; ja.mutex_out = b.mutex_out; ja.contrib_out = b.contrib_out;
        ja.instance = b.instance; ja.mode = b.mode;
        return ja;
    }
    template <class Args> static jit::LookupCheckJitArgs fold_jit_args(const Args& f) {   // LookupFoldArgs, FoldCensusArgs
        jit::LookupCheckJitArgs ja = lookup_check_args(f);
        ja.n_cols = f.n_cols; ja.marks = f.marks; ja.aux_cm = f.aux_cm; ja.final_a = f.final.a; ja.final_b = f.final.b;
        ja.failing_rows = f.failing_rows;
        return ja;
    }
    void check_constraints(const mdn_statement* st, const mdn_matrix* traces, const mdn_matrix* prep, const mdn_challenger* ch,
                           mdn_aux_builder build_aux, void* aux_ctx, u32 flags, mdn_constraint_report* out);
    // what prepare_check leaves per instance for the row pass of check_constraints / constraint_census
    struct CheckSetup {
        std::vector<u32> pos;                    // proof position of each instance (main_c / aux_c index)
        std::vector<DevBuf> prep_cm, periodic;   // raw preprocessed trace and periodic matrix, or empty
        int ext_rc = 0; u32 ext_failed = 0;      // the external check: > 0 with ext_failed = the failing assertion
    };
    void prepare_check(const mdn_statement* st, const mdn_matrix* traces, const mdn_matrix* prep, const mdn_challenger* ch,
                       mdn_aux_builder build_aux, void* aux_ctx, u32 flags, const void* out, CheckSetup& cs);
    void check_rows(std::vector<mk::CheckArgs>& ca, bool locate, mdn_constraint_report* out);
    void guard_constraints(const std::vector<u64>& flat_values);
    void constraint_census(const mdn_statement* st, const mdn_matrix* traces, const mdn_matrix* prep, const mdn_challenger* ch,
                           mdn_aux_builder build_aux, void* aux_ctx, u32 flags, mdn_constraint_failure* failures, u64 max_failures,
                           mdn_constraint_tally* tallies, u64 max_tallies, mdn_constraint_census_report* out);
    void check_trace_balance(const mdn_statement* st, const mdn_matrix* traces, const u64* rnd, const u64* boundary, size_t n_boundary,
                             const uint32_t* const* mutex_sites, u64 max_contrib, u32 flags, mdn_balance_report* out);
    // what prepare_folds leaves for the row passes of check_lookup_folds / lookup_fold_census
    struct FoldSetup {
        bool on_device = false, cm = false; u32 k = 0;
        u32 skipped = 0;                        // AIRs without a lookup program
        size_t staging_words = 0;               // the largest host fold buffer
        std::vector<u64*> main_cm, aux_cm;      // raw column-major main and aux traces of the lookup AIRs
        std::vector<DevBuf> marks;              // device fold marks, or empty
        std::vector<E2> finals;                 // the value aux[N][0] would hold
    };
    void prepare_folds(const mdn_statement* st, const mdn_matrix* traces, const u64* rnd, const uint32_t* const* fold_marks,
                       const mdn_matrix* aux, const u64* const* aux_finals, u64* const* folds_out, u32 flags, const void* out, FoldSetup& fs);
    // the fold kernels' inputs of lookup AIR i (kernels.cuh LookupFoldArgs, FoldCensusArgs name them alike)
    template <class Args> Args fold_args(u32 i, const FoldSetup& fs) const {
        Args f{};
        f.main_cm = fs.main_cm[i]; f.prep_cm = airs[i].raw_prep.p; f.log_n = log_heights[i]; f.n_cols = airs[i].lookup_cols; f.prog = airs[i].lookup_dev;
        f.publics = d_publics.p; f.challenges = d_randomness.p; f.marks = (const u32*)fs.marks[i].p;
        f.aux_cm = fs.aux_cm[i]; f.final = fs.finals[i];
        return f;
    }
    void check_lookup_folds(const mdn_statement* st, const mdn_matrix* traces, const u64* rnd, const uint32_t* const* fold_marks,
                            const mdn_matrix* aux, const u64* const* aux_finals, u64* const* folds_out, u32 flags, mdn_fold_report* out);
    void lookup_fold_census(const mdn_statement* st, const mdn_matrix* traces, const u64* rnd, const uint32_t* const* fold_marks,
                            const mdn_matrix* aux, const u64* const* aux_finals, u32 flags, mdn_fold_failure* failures, u64 max_failures,
                            mdn_fold_tally* tallies, u64 max_tallies, mdn_fold_census_report* out);
    // the last balance report's lists (mdn_balance_report points into them)
    std::vector<mdn_unmatched> bal_unmatched;
    std::vector<mdn_balance_push> bal_contrib;
    std::vector<mdn_mutex_violation> bal_mutex;
    void commit_aux(const mdn_matrix* aux, const u64* const* aux_values, bool zero_aux, const mdn_matrix* builder_main = nullptr);
    void call_device_aux_builder(u32 inst, const mdn_matrix& main, u64* aux_slot, std::vector<u64>& values);
    void finish();
    u64 grind(u32 bits);
    void reset_proof();
};

namespace {

// ---------------------------------------------------------------------------------------------
// table construction (host, tiny): ntt_tables.hpp ------------------------------------------------
// ---------------------------------------------------------------------------------------------
using ntt_tables::split_n;

}  // namespace

NttPlan& mdn_session::ntt(u32 n) {
    auto it = ntt_plans.find(n);
    if (it != ntt_plans.end()) return *it->second;
    if (n > 22) fail(MDN_ERR_UNSUPPORTED, "trace height 2^%u exceeds the supported 2^22", n);
    auto plan = std::make_unique<NttPlan>();
    ntt_tables::NttHost host = ntt_tables::build_ntt(n);
    { ArenaScope persistent(nullptr); plan->store.alloc(host.data.size(), stream); }
    CUDA_OK(cudaMemcpyAsync(plan->store.p, host.data.data(), host.data.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    plan->T = host.view(plan->store.p);
    auto& ref = *plan;
    ntt_plans[n] = std::move(plan);
    return ref;
}

namespace {
std::unique_ptr<PremulPlan> make_premul(const std::vector<u64>& bases, u32 n, cudaStream_t stream) {
    ntt_tables::PremulHost host = ntt_tables::build_premul(bases, n);
    auto plan = std::make_unique<PremulPlan>();
    { ArenaScope persistent(nullptr); plan->store.alloc(host.data.size(), stream); }
    CUDA_OK(cudaMemcpyAsync(plan->store.p, host.data.data(), host.data.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    plan->P = host.view(plan->store.p);
    plan->n_bases = (u32)bases.size();
    return plan;
}
}  // namespace

// bases g_t = shift * w_L^t: coset t of the LDE of a height-2^n trace (commit.rs:137-141, domain.rs:358-361)
PremulPlan& mdn_session::premul_trace(u32 n) {
    auto key = std::make_pair(n, 0u);
    auto it = premul_plans.find(key);
    if (it != premul_plans.end()) return *it->second;
    u32 lb = params.log_blowup, B = 1u << lb;
    u64 s = gl::lde_shift(n + lb), wl = gl::two_adic_generator(n + lb);
    std::vector<u64> bases(B);
    u64 x = s;
    for (u32 t = 0; t < B; t++) { bases[t] = x; x = gl::mul(x, wl); }
    auto plan = make_premul(bases, n, stream);
    auto& ref = *plan;
    premul_plans[key] = std::move(plan);
    return ref;
}
// bases w_J^(-t) * w_L^(t'), id = t*B + t' for chunk t < D and LDE coset t' < B, with J the quotient
// domain of order N*D (w_J = w_L^(B/D))  (quotient.rs:186-209: chunk t scaled by w_J^(-kt), then a
// plain DFT over K evaluates on g*K because the iDFT over H left g^k baked into the coefficients)
PremulPlan& mdn_session::premul_quotient(u32 n, u32 log_d) {
    auto key = std::make_pair(n, 1u + log_d);
    auto it = premul_plans.find(key);
    if (it != premul_plans.end()) return *it->second;
    u32 lb = params.log_blowup, B = 1u << lb, D = 1u << log_d;
    u64 wl = gl::two_adic_generator(n + lb), wji = gl::inv(gl::two_adic_generator(n + log_d));
    std::vector<u64> bases(D * B);
    for (u32 t = 0; t < D; t++)
        for (u32 t2 = 0; t2 < B; t2++) bases[t * B + t2] = gl::mul(gl::pow(wji, t), gl::pow(wl, t2));
    auto plan = make_premul(bases, n, stream);
    auto& ref = *plan;
    premul_plans[key] = std::move(plan);
    return ref;
}
// the one base 1: a forward NTT with it evaluates bit-reversed coefficients back on H, the rows of the trace
PremulPlan& mdn_session::premul_unshifted(u32 n) {
    auto key = std::make_pair(n, ~0u);
    auto it = premul_plans.find(key);
    if (it != premul_plans.end()) return *it->second;
    auto plan = make_premul(std::vector<u64>{1}, n, stream);
    auto& ref = *plan;
    premul_plans[key] = std::move(plan);
    return ref;
}

void mdn_session::reset_proof() {
    in_proof = false; shard_active = false; col_major = false;
    log_heights.clear(); order.clear(); publics.clear(); randomness.clear();
    aux_values_p.clear(); aux_values_off.clear();
    tr = Transcript();
    release_proof_memory();
}

// Called when no proof-lifetime buffer of a caller's frame is alive any more (API wrappers, error paths).
void mdn_session::release_proof_memory() {
    main_c = Committed(); aux_c = Committed(); quot_c = Committed();
    airs.clear();
    d_publics.release(); d_randomness.release(); d_aux_values.release();
    arena.reset();
}

// ---------------------------------------------------------------------------------------------
// One proof on G ranks: peer mappings of the arena, device barrier
// ---------------------------------------------------------------------------------------------
// Collective (every rank reaches it at the same point of the same allocation sequence): export the new slab, gather
// the G handles through the host callback, map the peers' slabs.
void mdn_session::shard_map_slab(char* base, size_t size) {
    if (shard_world <= 1) return;
    cudaIpcMemHandle_t h;
    CUDA_OK(cudaIpcGetMemHandle(&h, base));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
    const size_t W = 10;
    std::vector<u64> mine(W), all(W * shard_world);
    memcpy(mine.data(), &h, 64); mine[8] = size; mine[9] = slab_views.size();
    if (allgather(allgather_ctx, mine.data(), all.data(), W) != 0) fail(MDN_ERR_INVALID_ARG, "all-gather callback failed");
    SlabView v{}; v.size = size;
    for (u32 g = 0; g < shard_world; g++) {
        if (all[g * W + 8] != size || all[g * W + 9] != mine[9])
            fail(MDN_ERR_INVALID_ARG, "rank %u allocated a different proof arena (slab %llu of %llu bytes here, slab %llu of %llu bytes there): every rank must prove the same statement with the same flags",
                 g, (unsigned long long)mine[9], (unsigned long long)size, (unsigned long long)all[g * W + 9], (unsigned long long)all[g * W + 8]);
        if (g == shard_rank) { v.base[g] = base; continue; }
        cudaIpcMemHandle_t hg; memcpy(&hg, &all[g * W], 64);
        void* m = nullptr;
        CUDA_OK(cudaIpcOpenMemHandle(&m, hg, cudaIpcMemLazyEnablePeerAccess));
        v.base[g] = (char*)m;
    }
    slab_views.push_back(v);
    { std::vector<u64> one(1, 0), got(shard_world); if (allgather(allgather_ctx, one.data(), got.data(), 1) != 0) fail(MDN_ERR_INVALID_ARG, "all-gather callback failed"); }   // every rank has mapped it
}
// Collective: nobody frees a slab a peer still has mapped.
void mdn_session::shard_unmap_slabs() {
    if (slab_views.empty()) return;
    cudaStreamSynchronize(stream);
    for (auto& v : slab_views) for (u32 g = 0; g < shard_world; g++) if (g != shard_rank && v.base[g]) cudaIpcCloseMemHandle(v.base[g]);
    slab_views.clear();
    if (shard_world > 1 && allgather) { std::vector<u64> one(1, 0), all(shard_world); allgather(allgather_ctx, one.data(), all.data(), 1); }
}
void mdn_session::shard_teardown() {
    if (shard_world > 1) {
        release_proof_memory();
        arena.destroy();                    // unmaps the peers first (before_drop_slabs)
        if (sync_local) {
            for (u32 g = 0; g < shard_world; g++) if (g != shard_rank && sync_flags.p[g]) cudaIpcCloseMemHandle(sync_flags.p[g]);
            cudaFree(sync_local); sync_local = nullptr;
        }
    }
    arena.on_new_slab = nullptr; arena.before_drop_slabs = nullptr;
    sync_flags = mk::PeerPtrs{}; sync_epoch = 0;
    shard_rank = 0; shard_world = 1; shard_log_g = 0; allgather = nullptr; allgather_ctx = nullptr; shard_active = false;
}
mk::PeerPtrs mdn_session::peers_of(const u64* p) const {
    mk::PeerPtrs r{};
    if (shard_world <= 1) { r.p[0] = const_cast<u64*>(p); return r; }
    for (size_t i = 0; i < slab_views.size() && i < arena.slabs.size(); i++) {
        const char* b = arena.slabs[i].base;
        if ((const char*)p >= b && (const char*)p < b + arena.slabs[i].size) {
            size_t off = (const char*)p - b;
            for (u32 g = 0; g < shard_world; g++) r.p[g] = (u64*)(slab_views[i].base[g] + off);
            return r;
        }
    }
    fail(MDN_ERR_CUDA, "internal: buffer outside the shared proof arena");
}
mk::PushDst mdn_session::push_dst(u64* p, u32 mode, u32 owner_shift) const {
    if (!sharded() || mode == mk::PUSH_LOCAL) return mk::local_dst(p);
    mk::PushDst d{};
    d.pp = peers_of(p); d.rank = shard_rank; d.world = shard_world; d.mode = mode; d.owner_shift = owner_shift;
    return d;
}
void mdn_session::shard_barrier() {
    if (!sharded()) return;
    mk::launch_barrier(sync_flags, shard_rank, shard_world, ++sync_epoch, (u32*)d_flag.p, stream);
}
void mdn_session::shard_check(const char* where) {
    if (!sharded()) return;
    u32 flag = 0;
    CUDA_OK(cudaMemcpyAsync(&flag, d_flag.p, sizeof flag, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    if (flag & 8) { CUDA_OK(cudaMemsetAsync(d_flag.p, 0, 8, stream)); fail(MDN_ERR_CUDA, "cross-GPU barrier timed out (%s): a peer rank stopped or proves a different statement", where); }
}

void mdn_session::shard_check_enqueue() {
    shard_flag_host = 0;
    if (sharded()) CUDA_OK(cudaMemcpyAsync(&shard_flag_host, d_flag.p, sizeof shard_flag_host, cudaMemcpyDeviceToHost, stream));
}
void mdn_session::shard_check_finish(const char* where) {
    if (!sharded()) return;
    if (shard_flag_host & 8) { CUDA_OK(cudaMemsetAsync(d_flag.p, 0, 8, stream)); fail(MDN_ERR_CUDA, "cross-GPU barrier timed out (%s): a peer rank stopped or proves a different statement", where); }
}

void mdn_session::check_input_flag(const char* what) {
    u32 flag = 0;
    CUDA_OK(cudaMemcpyAsync(&flag, d_flag.p, sizeof flag, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    if (sharded()) {   // slices checked by the other ranks report into every rank's word (launch_transpose_slice_push)
        u32 peer_flag = 0;
        CUDA_OK(cudaMemcpyAsync(&peer_flag, sync_local + 16, sizeof peer_flag, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        if (peer_flag) { CUDA_OK(cudaMemsetAsync(sync_local + 16, 0, 8, stream)); flag |= peer_flag & 1u; }
    }
    if (flag) {
        CUDA_OK(cudaMemsetAsync(d_flag.p, 0, 8, stream));
        if (flag & 8) fail(MDN_ERR_CUDA, "cross-GPU barrier timed out: a peer rank stopped or proves a different statement");
        fail(MDN_ERR_INVALID_ARG, "%s contains a non-canonical field element (>= p)", what);
    }
}

// Host -> device copy on the copy stream.  Pinned (or registered) memory goes straight to the DMA engine;
// pageable memory is staged through two pinned 32 MiB bounce buffers filled by a few host threads, which
// sustains more throughput than a plain cudaMemcpyAsync from pageable memory.
void mdn_session::host_to_device(u64* dst, const u64* src, size_t n) {
    cudaPointerAttributes at{};
    bool pinned = cudaPointerGetAttributes(&at, src) == cudaSuccess && at.type == cudaMemoryTypeHost;
    cudaGetLastError();
    if (pinned) { CUDA_OK(cudaMemcpyAsync(dst, src, n * sizeof(u64), cudaMemcpyHostToDevice, copy_stream)); return; }
    for (int b = 0; b < 2; b++) if (!bounce[b]) { CUDA_OK(cudaHostAlloc((void**)&bounce[b], BOUNCE_WORDS * sizeof(u64), cudaHostAllocDefault)); CUDA_OK(cudaEventCreateWithFlags(&bounce_ev[b], cudaEventDisableTiming)); }
    unsigned nt = std::min(16u, std::max(1u, std::thread::hardware_concurrency() / 2));
    int b = 0;
    for (size_t off = 0; off < n; off += BOUNCE_WORDS, b ^= 1) {
        size_t cnt = std::min(BOUNCE_WORDS, n - off);
        if (bounce_busy[b]) CUDA_OK(cudaEventSynchronize(bounce_ev[b]));
        std::vector<std::thread> th;
        size_t per = (cnt + nt - 1) / nt;
        for (unsigned q = 0; q < nt; q++) {
            size_t a = (size_t)q * per, e = std::min(cnt, a + per);
            if (a >= e) break;
            th.emplace_back([=] { memcpy(bounce[b] + a, src + off + a, (e - a) * sizeof(u64)); });
        }
        for (auto& t : th) t.join();
        CUDA_OK(cudaMemcpyAsync(dst + off, bounce[b], cnt * sizeof(u64), cudaMemcpyHostToDevice, copy_stream));
        CUDA_OK(cudaEventRecord(bounce_ev[b], copy_stream));
        bounce_busy[b] = true;
    }
}

// row-major (host or device) or column-major (device) -> column-major device; a column-major matrix whose values are
// dst_cm already is only checked
void mdn_session::upload_matrix(const mdn_matrix& m, bool on_device, u64* dst_cm, bool col_major) {
    size_t N = (size_t)1 << m.log_height;
    if (m.width == 0) return;
    if (col_major) {
        ProfScope ps(prof, PC_TRANSPOSE);
        mk::launch_ingest_cm(m.values, dst_cm, N * m.width, (u32*)d_flag.p, stream);
        return;
    }
    if (on_device) {
        ProfScope ps(prof, PC_TRANSPOSE);
        mk::launch_transpose_rm_to_cm(m.values, dst_cm, (u32)N, m.width, (u32*)d_flag.p, stream);
        return;
    }
    DevBuf staging; staging.alloc(N * m.width, stream);
    CUDA_OK(cudaEventRecord(copy_ev[7], stream));
    CUDA_OK(cudaStreamWaitEvent(copy_stream, copy_ev[7], 0));
    host_to_device(staging.p, m.values, N * m.width);
    CUDA_OK(cudaEventRecord(copy_ev[6], copy_stream));
    CUDA_OK(cudaStreamWaitEvent(stream, copy_ev[6], 0));
    ProfScope ps(prof, PC_TRANSPOSE);
    mk::launch_transpose_rm_to_cm(staging.p, dst_cm, (u32)N, m.width, (u32*)d_flag.p, stream);
}

// a1 + a2 + a3: coset LDE of every matrix of `c` (coefficients already in c.coef as natural
// evaluations over H), leaf hashing and tree compression.
//   reference: commit_traces (prover/commit.rs:142-180) -> coset_lde_batch (:173) +
//   build_aligned_tree (:178; lmcs/lifted_tree.rs:202-284)
void mdn_session::lde_matrix(CommittedMat& m) {
    if (!m.width) return;
    u32 lb = params.log_blowup;
    size_t N = (size_t)1 << m.log_n, L = N << lb;
    NttPlan& plan = ntt(m.log_n);
    PremulPlan& pm = premul_trace(m.log_n);
    ProfScope ps(prof, PC_NTT);
    ntt_bytes += (double)(N + (size_t)nt() * N) * m.width * 8.0;   // read the trace column once, write this rank's cosets of the LDE once
    if (sharded() && m.log_n >= shard_log_g + shard_min_log) {
        // interpolation split by column: rank g transforms columns [g*w/G, (g+1)*w/G) and stores the coefficients into
        // every rank (the all-gather of coefficient columns of SURVEY 8(e), as peer stores)
        u32 c0 = (u32)((u64)m.width * shard_rank / shard_world), c1 = (u32)((u64)m.width * (shard_rank + 1) / shard_world);
        if (c1 > c0) mk::launch_intt(m.coef + (size_t)c0 * N, N, c1 - c0, plan.T, stream);
        shard_barrier();     // every rank is done with the raw columns (transposes, the copy kept for the LogUp build)
        if (c1 > c0) mk::launch_push(m.coef + (size_t)c0 * N, peers_of(m.coef + (size_t)c0 * N), shard_rank, shard_world, (size_t)(c1 - c0) * N, stream);
        shard_barrier();
    } else mk::launch_intt(m.coef, N, m.width, plan.T, stream);
    // this rank's cosets only (all B of them on one GPU); column groups sized so a group's LDE (the fwd passes'
    // working set) stays L2-resident: 20 MB leaves room in either 25 MB half of the H100's 50 MB L2
    const u32 tb = t0(), tn = nt();
    size_t col_bytes = (size_t)tn * N * sizeof(u64);
    u32 group = (u32)std::max<size_t>(1, (20u << 20) / col_bytes);
    std::vector<mk::FwdItem> items;
    for (u32 cc = 0; cc < m.width; cc++)
        for (u32 t = tb; t < tb + tn; t++)
            items.push_back(mk::FwdItem{m.coef + (size_t)cc * N, m.lde + (size_t)cc * L + (size_t)t * N, t, 0});
    DevBuf d_items;
    d_items.alloc(items.size() * sizeof(mk::FwdItem) / sizeof(u64), stream);
    CUDA_OK(cudaMemcpyAsync(d_items.p, items.data(), items.size() * sizeof(mk::FwdItem), cudaMemcpyHostToDevice, stream));
    for (u32 c0 = 0; c0 < m.width; c0 += group) {
        u32 cn = std::min(group, m.width - c0);
        mk::launch_fwd_ntt((const mk::FwdItem*)d_items.p + (size_t)c0 * tn, cn * tn, plan.T, pm.P, stream);
    }
}

void mdn_session::lde_and_commit(Committed& c, float* t_lde, float* t_hash, bool lde_done) {
    cudaEvent_t e0 = ev[12], e1 = ev[13], e2 = ev[14];
    CUDA_OK(cudaEventRecord(e0, stream));
    if (!lde_done) for (auto& m : c.mats) lde_matrix(m);
    CUDA_OK(cudaEventRecord(e1, stream));
    build_tree(c);
    CUDA_OK(cudaEventRecord(e2, stream));
    CUDA_OK(cudaEventSynchronize(e2));
    float a = 0, b = 0;
    cudaEventElapsedTime(&a, e0, e1); cudaEventElapsedTime(&b, e1, e2);
    if (t_lde) *t_lde += a;
    if (t_hash) *t_hash += b;
}

// leaf sponge states per height group (ascending), then the compression layers.
// Split over ranks: every rank hashes the leaves of its cosets and stores each digest into the rank that owns the
// leaf's sub-tree (leaf index = domain index r*B + t, owner = index >> (depth - log G)); after the barrier every rank
// compresses its own sub-tree, stores its sub-root into all ranks, and the top log G layers are recomputed everywhere.
// Trees too small to split are replicated: the digests go to every rank.
void mdn_session::build_tree(Committed& c) {
    u32 lb = params.log_blowup;
    u32 log_n_max = 0;
    for (auto& m : c.mats) log_n_max = std::max(log_n_max, m.log_n);
    u32 depth = log_n_max + lb;
    size_t L = (size_t)1 << depth;
    c.tree.depth = depth;
    c.tree.nodes.alloc((2 * L - 1) * 4, stream);
    const bool sh = sharded(), split = tree_sharded(depth);
    const u32 lg = shard_log_g, tb = t0(), tn = nt();
    mk::PushDst dig = push_dst(c.tree.layer(depth), sh ? (split ? mk::PUSH_OWNER : mk::PUSH_ALL) : mk::PUSH_LOCAL, depth - (split ? lg : 0));
    shard_barrier();   // the tree buffer is a fresh allocation: no rank may still be using the memory under its old identity
    DevBuf states_a, states_b;
    // One launch absorbs up to 8 matrices of one height (launch-argument space); a taller pile of equal-height matrices
    // is absorbed in several launches that hand the sponge states on through the SoA state buffers, exactly like the
    // hand-over between height groups.
    const u64* prev = nullptr; u32 prev_log = 0;
    size_t i = 0;
    while (i < c.mats.size()) {
        size_t j = i;
        mk::LeafArgs args; args.n_mats = 0;
        const u32 ln = c.mats[i].log_n;
        while (j < c.mats.size() && c.mats[j].log_n == ln && args.n_mats < 8) {
            // a zero-width matrix is a no-op for the sponge (an empty absorb leaves the state untouched) but not for the
            // chaining hasher, which re-hashes its state (crates/stateful-hasher/src/chaining.rs:43-46)
            if (c.mats[j].width || hash_kind == MDN_HASH_BLAKE3) args.m[args.n_mats++] = mk::LeafMat{c.mats[j].lde, c.mats[j].width, 0};
            j++;
        }
        bool last = (j == c.mats.size());
        DevBuf& out = (prev == states_a.p && prev) ? states_b : states_a;
        if (!last) out.alloc((size_t)state_words() << (ln + lb), stream);
        {
            ProfScope ps(prof, PC_LEAF);
            size_t Lg = (size_t)tn << ln;
            const u32 rate = hash_kind == MDN_HASH_KECCAK ? 17 : 8;
            for (int q = 0; q < args.n_mats; q++) { leaf_bytes += (double)Lg * args.m[q].width * 8.0; perms += Lg * ((args.m[q].width + rate - 1) / rate); }
            leaf_bytes += last ? (double)Lg * 32.0 : (double)Lg * 8.0 * state_words();
            hash_leaves(args, ln, lb, prev, prev_log, last ? nullptr : out.p, last ? &dig : nullptr, tb, tn);
        }
        prev = out.p; prev_log = ln;
        i = j;
    }
    shard_barrier();   // every digest of this rank's leaf range (or of the whole replicated tree) has arrived
    if (!split) {
        ProfScope ps(prof, PC_COMPRESS);
        perms += compress_subtree(c.tree, depth, 0, 0);
    } else {
        {
            ProfScope ps(prof, PC_COMPRESS);
            perms += compress_subtree(c.tree, depth, lg, shard_rank);
        }
        u64* mine = c.tree.layer(lg) + (size_t)shard_rank * 4;
        mk::launch_push(mine, peers_of(mine), shard_rank, shard_world, 4, stream);
        shard_barrier();
        ProfScope ps(prof, PC_COMPRESS);
        compress_subtree(c.tree, lg, 0, 0);
    }
    CUDA_OK(cudaMemcpyAsync(c.root, c.tree.layer(0), 4 * sizeof(u64), cudaMemcpyDeviceToHost, stream));
    shard_check_enqueue();
    CUDA_OK(cudaStreamSynchronize(stream));
    shard_check_finish("commitment");
}

// GrindingChallenger::grind on the device: smallest witness (sequential p3 order), then the
// challenger advances to the post-check state (random_coin.masm:929-966).
u64 mdn_session::grind(u32 bits) {
    if (bits == 0) { tr.fields.push_back(0); return 0; }
    Duplex& ch = tr.ch;
    if (ch.hashed) {
        // hash challenger: a candidate w is checked by hashing (input buffer || w as 8 little-endian bytes) and reading
        // the low bits of the first sampled u64; the buffer is whole 32-bit words (every observation is 8 or 32 bytes)
        if (ch.bin.size() % (ch.keccak ? 8 : 4)) fail(MDN_ERR_INVALID_ARG, "hash challenger input buffer is not a whole number of words");
        u32 nw = (u32)(ch.bin.size() / 4);
        DevBuf d; d.alloc((nw + 1) / 2 + 2, stream);
        u64 none = ~0ull;
        if (nw) CUDA_OK(cudaMemcpyAsync(d.p + 1, ch.bin.data(), ch.bin.size(), cudaMemcpyHostToDevice, stream));
        CUDA_OK(cudaMemcpyAsync(d.p, &none, sizeof none, cudaMemcpyHostToDevice, stream));
        u64 start = 0, found = ~0ull;
        u64 batch = std::max<u64>(1ull << 14, std::min<u64>(1ull << 20, 4ull << bits));
        ProfScope ps(prof, PC_GRIND);
        while (found == ~0ull) {
            if (start >= gl::P) fail(MDN_ERR_INVALID_ARG, "proof-of-work search exhausted");
            if (ch.keccak) mk::launch_grind_kk(d.p + 1, nw / 2, bits, start, batch, d.p, stream);
            else mk::launch_grind_b3((const u32*)(d.p + 1), nw, bits, start, batch, d.p, stream);
            CUDA_OK(cudaMemcpyAsync(&found, d.p, sizeof(u64), cudaMemcpyDeviceToHost, stream));
            CUDA_OK(cudaStreamSynchronize(stream));
            start += batch;
        }
        ch.observe(found);
        if (ch.sample_bits(bits) != 0) fail(MDN_ERR_CUDA, "device proof-of-work witness failed the host check");
        tr.fields.push_back(found);
        return found;
    }
    if (ch.in_len >= 8) fail(MDN_ERR_INVALID_ARG, "challenger buffer overflow");
    u64 base[12];
    for (int i = 0; i < 12; i++) base[i] = ch.st[i];
    for (u32 i = 0; i < ch.in_len; i++) base[i] = ch.in[i];
    DevBuf d; d.alloc(13, stream);
    u64 init[13];
    memcpy(init, base, sizeof base); init[12] = ~0ull;
    CUDA_OK(cudaMemcpyAsync(d.p, init, sizeof init, cudaMemcpyHostToDevice, stream));
    u64 start = 0, found = ~0ull;
    u64 batch = std::max<u64>(1ull << 14, std::min<u64>(1ull << 22, 4ull << bits));
    ProfScope ps(prof, PC_GRIND);
    while (found == ~0ull) {
        if (start >= gl::P) fail(MDN_ERR_INVALID_ARG, "proof-of-work search exhausted");
        mk::launch_grind(d.p, ch.in_len, bits, start, batch, d.p + 12, stream, perm());
        CUDA_OK(cudaMemcpyAsync(&found, d.p + 12, sizeof(u64), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        start += batch;
    }
    ch.observe(found);
    u64 chk = ch.sample_bits(bits);
    if (chk != 0) fail(MDN_ERR_CUDA, "device proof-of-work witness failed the host check");
    tr.fields.push_back(found);
    return found;
}

// ---------------------------------------------------------------------------------------------
// op-list compiler: validation, liveness, slot assignment (shared by constraint and lookup programs)
// ---------------------------------------------------------------------------------------------
struct Compiled { std::vector<u32> code; std::vector<u64> consts; u32 n_slots = 0; bool uses_sel = false; };
// node j = (op, x, y) of AIR i's program with nk constants: op and operands in range, operands defined before j
static void check_node(u32 i, const mdn_air& a, u32 n_publics, u32 nk, bool lookup, u32 j, u32 op, u32 x, u32 y) {
    if (op > 15) fail(MDN_ERR_INVALID_ARG, "AIR %u: unknown op %u", i, op);
    // a LookupBuilder exposes the main and preprocessed windows, periodic values, public values, challenges and
    // constants only
    if (lookup && (op == 1 || (op >= 4 && op <= 7))) fail(MDN_ERR_INVALID_ARG, "AIR %u: op %u is not available to a lookup program", i, op);
    if (op == 15 && (x > 1 || y >= a.preprocessed_width)) fail(MDN_ERR_INVALID_ARG, "AIR %u: preprocessed column out of range", i);
    if (op >= 10 && op <= 12 && (x >= j || y >= j)) fail(MDN_ERR_INVALID_ARG, "AIR %u: forward reference", i);
    if (op == 13 && x >= j) fail(MDN_ERR_INVALID_ARG, "AIR %u: forward reference", i);
    if (op == 0 && (x > 1 || y >= a.width)) fail(MDN_ERR_INVALID_ARG, "AIR %u: main column out of range", i);
    if (op == 1 && (x > 1 || y >= a.aux_width)) fail(MDN_ERR_INVALID_ARG, "AIR %u: aux column out of range", i);
    if (op == 2 && x >= n_publics) fail(MDN_ERR_INVALID_ARG, "AIR %u: public value out of range", i);
    if (op == 3 && x >= a.num_randomness) fail(MDN_ERR_INVALID_ARG, "AIR %u: challenge out of range", i);
    if (op == 4 && x >= a.num_aux_values) fail(MDN_ERR_INVALID_ARG, "AIR %u: aux value out of range", i);
    if (op == 8 && x >= nk) fail(MDN_ERR_INVALID_ARG, "AIR %u: constant out of range", i);
    if (op == 9 && x + 1 >= nk) fail(MDN_ERR_INVALID_ARG, "AIR %u: constant out of range", i);
    if (op == 14 && x >= a.num_periodic_columns) fail(MDN_ERR_INVALID_ARG, "AIR %u: periodic column out of range", i);
}
// lookup == false: words = [MAIR, 1, n_nodes, n_constraints, n_consts | nodes | constraint node ids | consts];
//                  a FOLD instruction (15) is placed right after the node it folds, in emission order.
// lookup == true : words = [MLKP, 1, n_nodes, n_interactions, n_consts | nodes | {column, flag, mult, denom} | consts];
//                  an EMIT instruction (17) is placed once its three operands are defined.
static Compiled compile_oplist(u32 i, const mdn_air& a, u32 n_publics, const u32* w, u32 n_words, bool lookup, u32 lookup_cols) {
    const char* what = lookup ? "lookup program" : "constraint program";
    const u32 magic = lookup ? 0x504B4C4Du : 0x5249414Du, item = lookup ? 4u : 1u;
    if (!w || n_words < 5 || w[0] != magic || w[1] != 1) fail(MDN_ERR_INVALID_ARG, "AIR %u: bad %s header", i, what);
    u32 nn = w[2], nc = w[3], nk = w[4];
    if ((size_t)n_words != 5 + 3 * (size_t)nn + (size_t)item * nc + 2 * (size_t)nk) fail(MDN_ERR_INVALID_ARG, "AIR %u: bad %s length", i, what);
    Compiled out;
    const u32* items = w + 5 + 3 * (size_t)nn;
    for (u32 j = 0; j < nn; j++) {
        u32 op = w[5 + 3 * j], x = w[6 + 3 * j], y = w[7 + 3 * j];
        check_node(i, a, n_publics, nk, lookup, j, op, x, y);
        if (op >= 5 && op <= 7) out.uses_sel = true;
    }
    // event stream: node definitions, each followed by the folds / emits that became ready
    struct Ev { u32 kind; u32 node; };   // kind 0: define node; 1: fold node / emit interaction `node`
    std::vector<Ev> evs; evs.reserve(nn + nc);
    auto ready_at = [&](u32 kk) -> u32 {
        if (!lookup) return items[kk];
        const u32* it = items + 4 * (size_t)kk;
        u32 m = std::max(it[2], it[3]);
        return it[1] == 0xFFFFFFFFu ? m : std::max(m, it[1]);
    };
    for (u32 kk = 0; kk < nc; kk++) {
        if (!lookup) { if (items[kk] >= nn) fail(MDN_ERR_INVALID_ARG, "AIR %u: bad constraint id", i); continue; }
        const u32* it = items + 4 * (size_t)kk;
        if (it[0] >= lookup_cols) fail(MDN_ERR_INVALID_ARG, "AIR %u: lookup column out of range", i);
        if ((it[1] != 0xFFFFFFFFu && it[1] >= nn) || it[2] >= nn || it[3] >= nn) fail(MDN_ERR_INVALID_ARG, "AIR %u: bad lookup interaction", i);
    }
    { u32 kk = 0;
      for (u32 j = 0; j < nn; j++) {
          evs.push_back({0, j});
          while (kk < nc && ready_at(kk) <= j) { evs.push_back({1, lookup ? kk : items[kk]}); kk++; }
      }
      if (kk != nc) fail(MDN_ERR_INVALID_ARG, "AIR %u: %s with no nodes", i, what); }
    std::vector<u32> last_use(nn, 0);
    std::vector<uint8_t> is_ext(nn, 0);
    for (u32 e = 0; e < evs.size(); e++) {
        if (evs[e].kind) {
            if (!lookup) { last_use[evs[e].node] = e; continue; }
            const u32* it = items + 4 * (size_t)evs[e].node;
            if (it[1] != 0xFFFFFFFFu) last_use[it[1]] = e;
            last_use[it[2]] = e; last_use[it[3]] = e;
            continue;
        }
        u32 j = evs[e].node, op = w[5 + 3 * j], x = w[6 + 3 * j], y = w[7 + 3 * j];
        last_use[j] = std::max(last_use[j], e);
        if (op >= 10 && op <= 12) { last_use[x] = e; last_use[y] = e; is_ext[j] = is_ext[x] | is_ext[y]; }
        else if (op == 13) { last_use[x] = e; is_ext[j] = is_ext[x]; }
        else is_ext[j] = (op == 1 || op == 3 || op == 4 || op == 9);
    }
    if (lookup) for (u32 kk = 0; kk < nc; kk++) {
        const u32* it = items + 4 * (size_t)kk;
        if ((it[1] != 0xFFFFFFFFu && is_ext[it[1]]) || is_ext[it[2]]) fail(MDN_ERR_INVALID_ARG, "AIR %u: lookup flag and multiplicity must be base-field expressions", i);
    }
    std::vector<u32> slot_of(nn, 0), free_slots;
    u32 n_slots = 0;
    std::vector<u32>& code = out.code; code.reserve(4 * evs.size());
    auto release = [&](u32 node, u32 e) { if (last_use[node] == e) free_slots.push_back(slot_of[node]); };
    for (u32 e = 0; e < evs.size(); e++) {
        if (evs[e].kind && !lookup) {
            code.insert(code.end(), {15u | ((u32)is_ext[evs[e].node] << 8), 0u, slot_of[evs[e].node], 0u});
            release(evs[e].node, e);
            continue;
        }
        if (evs[e].kind) {
            const u32* it = items + 4 * (size_t)evs[e].node;
            u32 fs = it[1] == 0xFFFFFFFFu ? 0xffffu : slot_of[it[1]];
            // bits 8..31: the interaction index (read by the balance check only; it keeps nc below 2^24)
            code.insert(code.end(), {17u | ((evs[e].node & 0xFFFFFFu) << 8), it[0], fs | (slot_of[it[2]] << 16), slot_of[it[3]]});
            // a node may serve several operands of one interaction: release each distinct node once
            u32 ops3[3] = {it[1], it[2], it[3]};
            for (int q = 0; q < 3; q++) {
                if (ops3[q] == 0xFFFFFFFFu) continue;
                bool dup = false;
                for (int q2 = 0; q2 < q; q2++) dup |= ops3[q2] == ops3[q];
                if (!dup) release(ops3[q], e);
            }
            continue;
        }
        u32 j = evs[e].node, op = w[5 + 3 * j], x = w[6 + 3 * j], y = w[7 + 3 * j];
        u32 ox = x, oy = y;
        if (op >= 10 && op <= 13) {
            ox = slot_of[x]; oy = (op == 13) ? 0 : slot_of[y];
            release(x, e);
            if (op != 13 && y != x) release(y, e);
        }
        u32 dst;
        if (!free_slots.empty()) { dst = free_slots.back(); free_slots.pop_back(); }
        else dst = n_slots++;
        slot_of[j] = dst;
        code.insert(code.end(), {(op == 15 ? 16u : op) | ((u32)is_ext[j] << 8), dst, ox, oy});   // compiled 15 = FOLD, 16 = PREPROCESSED
        if (last_use[j] == e) free_slots.push_back(dst);   // dead value
    }
    if (n_slots > 1024) fail(MDN_ERR_UNSUPPORTED, "AIR %u: %s needs %u live values (interpreter limit 1024)", i, what, n_slots);
    out.n_slots = n_slots;
    const u32* kw = items + (size_t)item * nc;
    for (u32 j = 0; j < nk; j++) {
        u64 v = (u64)kw[2 * j] | ((u64)kw[2 * j + 1] << 32);
        if (v >= gl::P) fail(MDN_ERR_INVALID_ARG, "AIR %u: non-canonical constant", i);
        out.consts.push_back(v);
    }
    return out;
}

// A version-2 lookup program of AIR i (words = [MLKP, 2, n_nodes, n_interactions, n_consts, n_registers | nodes |
// {column, flag, mult, denom} | update node per register | consts]), validated and split in two:
//   v1   : the interaction part, a version-1 program of the nodes the interactions reach (renumbered in order), which
//          every consumer of version-1 programs takes as it is;
//   regs : the register part in the constraint-program format, its "constraints" being the update nodes, over the nodes
//          the updates reach; AUX(0, num_columns + i) reads register i.
struct LookupSplit { std::vector<u32> v1, regs; u32 n_regs = 0; };
static LookupSplit split_lookup_v2(u32 i, const mdn_air& a, u32 n_publics, const mdn_lookup& lk) {
    const u32* w = lk.program;
    const u32 n_words = lk.program_words;
    if (n_words < 6) fail(MDN_ERR_INVALID_ARG, "AIR %u: bad lookup program header", i);
    const u32 nn = w[2], nc = w[3], nk = w[4], nr = w[5];
    if ((size_t)n_words != 6 + 3 * (size_t)nn + 4 * (size_t)nc + nr + 2 * (size_t)nk) fail(MDN_ERR_INVALID_ARG, "AIR %u: bad lookup program length", i);
    if (nr < 1 || nr > mk::REG_MAX) fail(MDN_ERR_INVALID_ARG, "AIR %u: a version-2 lookup program has 1..=%u registers, not %u", i, mk::REG_MAX, nr);
    if (a.aux_width != lk.num_columns + nr || a.num_aux_values != 1)
        fail(MDN_ERR_INVALID_ARG, "AIR %u: a lookup program with registers needs aux_width == num_columns + n_registers and num_aux_values == 1", i);
    const u32* nodes = w + 6;
    const u32* items = nodes + 3 * (size_t)nn;
    const u32* upd = items + 4 * (size_t)nc;
    const u32* kw = upd + nr;
    // vocabulary and ranges; the AUX leaf is a register's row-r value; register degree of every node
    std::vector<uint8_t> deg(nn, 0);
    for (u32 j = 0; j < nn; j++) {
        const u32 op = nodes[3 * j], x = nodes[3 * j + 1], y = nodes[3 * j + 2];
        if (op == 1) {
            if (x != 0 || y < lk.num_columns || y >= a.aux_width) fail(MDN_ERR_INVALID_ARG, "AIR %u: node %u: an AUX leaf must read a register column at offset 0", i, j);
            deg[j] = 1;
            continue;
        }
        check_node(i, a, n_publics, nk, true, j, op, x, y);
        if (op == 10 || op == 11) deg[j] = std::max(deg[x], deg[y]);
        else if (op == 12) deg[j] = (uint8_t)std::min(2, deg[x] + deg[y]);
        else if (op == 13) deg[j] = deg[x];
    }
    for (u32 q = 0; q < nr; q++) {
        if (upd[q] >= nn) fail(MDN_ERR_INVALID_ARG, "AIR %u: bad register update node", i);
        if (deg[upd[q]] > 1) fail(MDN_ERR_INVALID_ARG, "AIR %u: the update of register %u is not affine in the registers", i, q);
    }
    for (u32 q = 0; q < nc; q++) {
        const u32* it = items + 4 * (size_t)q;
        if ((it[1] != 0xFFFFFFFFu && it[1] >= nn) || it[2] >= nn || it[3] >= nn) fail(MDN_ERR_INVALID_ARG, "AIR %u: bad lookup interaction", i);
    }
    // the nodes each part reaches (operands precede their node, so one backward pass)
    auto reach = [&](std::vector<uint8_t>& m) {
        for (u32 j = nn; j-- > 0;) {
            if (!m[j]) continue;
            const u32 op = nodes[3 * j];
            if (op >= 10 && op <= 12) { m[nodes[3 * j + 1]] = 1; m[nodes[3 * j + 2]] = 1; }
            else if (op == 13) m[nodes[3 * j + 1]] = 1;
        }
    };
    std::vector<uint8_t> in_v1(nn, 0), in_regs(nn, 0);
    for (u32 q = 0; q < nc; q++) {
        const u32* it = items + 4 * (size_t)q;
        if (it[1] != 0xFFFFFFFFu) in_v1[it[1]] = 1;
        in_v1[it[2]] = 1; in_v1[it[3]] = 1;
    }
    for (u32 q = 0; q < nr; q++) in_regs[upd[q]] = 1;
    reach(in_v1); reach(in_regs);
    for (u32 j = 0; j < nn; j++)
        if (in_v1[j] && deg[j]) fail(MDN_ERR_INVALID_ARG, "AIR %u: a lookup interaction reads a register (node %u); registers are read by register updates only", i, j);
    // one part: the kept nodes renumbered, then its items, then every constant
    auto part = [&](const std::vector<uint8_t>& keep, u32 magic, u32 n_items, auto&& emit_items) {
        std::vector<u32> id(nn, 0), out = {magic, 1, 0, n_items, nk};
        u32 m = 0;
        for (u32 j = 0; j < nn; j++) {
            if (!keep[j]) continue;
            u32 op = nodes[3 * j], x = nodes[3 * j + 1], y = nodes[3 * j + 2];
            if (op >= 10 && op <= 12) { x = id[x]; y = id[y]; }
            else if (op == 13) x = id[x];
            out.insert(out.end(), {op, x, y});
            id[j] = m++;
        }
        out[2] = m;
        emit_items(out, id);
        out.insert(out.end(), kw, kw + 2 * (size_t)nk);
        return out;
    };
    LookupSplit s;
    s.n_regs = nr;
    s.v1 = part(in_v1, 0x504B4C4Du, nc, [&](std::vector<u32>& out, const std::vector<u32>& id) {
        for (u32 q = 0; q < nc; q++) {
            const u32* it = items + 4 * (size_t)q;
            out.insert(out.end(), {it[0], it[1] == 0xFFFFFFFFu ? it[1] : id[it[1]], id[it[2]], id[it[3]]});
        }
    });
    s.regs = part(in_regs, 0x5249414Du, nr, [&](std::vector<u32>& out, const std::vector<u32>& id) {
        for (u32 q = 0; q < nr; q++) out.push_back(id[upd[q]]);
    });
    return s;
}


// ---------------------------------------------------------------------------------------------
// prove_begin: validation, statement/shape binding, main commit, randomness  (mod.rs:240-349)
// ---------------------------------------------------------------------------------------------
void mdn_session::prove_begin(const mdn_statement* st, const mdn_matrix* traces, const mdn_challenger* chal, u32 flags) {
    const bool cm = column_major(flags);
    reset_proof();
    log_qd = 0;
    memset(&timings, 0, sizeof timings);
    mk::reset_launch_count();
    prof.st = stream; prof.reset(); leaf_bytes = ntt_bytes = 0; perms = 0;
    validate_statement(st, traces, chal);
    if (cm) for (u32 i = 0; i < st->n_airs; i++) check_column_major(traces[i], "trace", i);
    col_major = cm;
    bool on_device = (flags & MDN_FLAG_DEVICE_TRACES) != 0;
    u32 lb = params.log_blowup;
    if (shard_world > 1) {
        if (!use_arena) fail(MDN_ERR_UNSUPPORTED, "a proof split over several ranks needs the proof arena (unset MDN_NO_ARENA)");
        if (lb < shard_log_g) fail(MDN_ERR_UNSUPPORTED, "a proof can be split over at most 2^log_blowup = %u ranks (one LDE coset each)", 1u << lb);
        shard_active = true;
        shard_barrier();   // no rank stores into a peer's arena for this proof before every rank has left the previous one
    }
    CUDA_OK(cudaEventRecord(ev[0], stream));

    u32 k = st->n_airs;
    bind_airs(st, traces, true, constraint_guard);
    if (constraint_guard) for (u32 i = 0; i < k; i++) {   // the guard's raw periodic matrices (canonical: checked by bind_airs)
        const mdn_air& a = st->airs[i];
        if (!a.num_periodic_columns) continue;
        size_t n = ((size_t)1 << a.log_max_period) * a.num_periodic_columns;
        airs[i].raw_periodic.alloc(n, stream);
        CUDA_OK(cudaMemcpyAsync(airs[i].raw_periodic.p, a.periodic_values, n * sizeof(u64), cudaMemcpyHostToDevice, stream));
    }
    // preprocessed presence / shape parity (ProverInstance::new, prover/mod.rs:139-153; validate_preprocessed,
    // preprocessed.rs:147-260): a bundle must be installed exactly when some AIR declares preprocessed columns,
    // and each committed trace must have its AIR's declared width and its main trace's height
    {
        bool expected = false;
        for (u32 i = 0; i < k; i++) expected |= st->airs[i].preprocessed_width > 0;
        if (expected != has_prep) fail(MDN_ERR_INVALID_ARG, "preprocessed presence mismatch: AIRs %s preprocessed columns but %s bundle is installed", expected ? "declare" : "declare no", has_prep ? "a" : "no");
        if (has_prep) {
            std::vector<int> idx(k, -1);
            for (size_t q = 0; q < prep_air.size(); q++) { if (prep_air[q] >= k) fail(MDN_ERR_INVALID_ARG, "preprocessed bundle was built for a different AIR list"); idx[prep_air[q]] = (int)q; }
            for (u32 i = 0; i < k; i++) {
                bool want = st->airs[i].preprocessed_width > 0;
                if (want != (idx[i] >= 0)) fail(MDN_ERR_INVALID_ARG, "AIR %u: preprocessed trace presence mismatch", i);
                if (!want) continue;
                if (prep_c.mats[idx[i]].width != st->airs[i].preprocessed_width) fail(MDN_ERR_INVALID_ARG, "AIR %u: preprocessed width %u does not match the declared %u", i, prep_c.mats[idx[i]].width, st->airs[i].preprocessed_width);
                if (prep_log_h[idx[i]] != traces[i].log_height) fail(MDN_ERR_INVALID_ARG, "AIR %u: preprocessed height 2^%u differs from the main trace height 2^%u", i, prep_log_h[idx[i]], traces[i].log_height);
            }
        }
    }
    bind_order(st, true);

    // challenger: caller's pre-bound state, then Statement::observe + observe_shape (mod.rs:290-291)
    bind_challenger(chal);
    Duplex& ch = tr.ch;
    if (has_prep) ch.observe_digest(prep_c.root);   // preprocessed commitment first (mod.rs:282-286)
    for (u32 i = 0; i < st->n_observe_felts; i++) ch.observe(st->observe_felts[i]);
    ch.observe(k);
    for (u32 i = 0; i < k; i++) ch.observe(log_heights[i]);
    upload_and_commit_main(traces, on_device);
}

// argument checks of prove_begin, shared with check_constraints
void mdn_session::validate_statement(const mdn_statement* st, const mdn_matrix* traces, const mdn_challenger* chal) {
    if (!st || !traces || (!chal && !byte_hash())) fail(MDN_ERR_INVALID_ARG, "null argument");
    if (st->n_airs == 0 || st->n_airs > 256) fail(MDN_ERR_INVALID_ARG, "AIR count must be in 1..=256");
    if (params.log_folding_arity < 1 || params.log_folding_arity > 3) fail(MDN_ERR_INVALID_ARG, "invalid folding arity: log_arity %u (must be 1, 2, or 3)", params.log_folding_arity);
    u32 lb = params.log_blowup;
    if (lb == 0 || lb > 4) fail(MDN_ERR_UNSUPPORTED, "log_blowup must be in 1..=4");
    if (st->n_public_values && !st->public_values) fail(MDN_ERR_INVALID_ARG, "public_values is NULL");
    if (st->n_observe_felts && !st->observe_felts) fail(MDN_ERR_INVALID_ARG, "observe_felts is NULL");
    for (u32 i = 0; i < st->n_public_values; i++) if (st->public_values[i] >= gl::P) fail(MDN_ERR_INVALID_ARG, "public value %u is not a canonical field element (>= p)", i);
    for (u32 i = 0; i < st->n_observe_felts; i++) if (st->observe_felts[i] >= gl::P) fail(MDN_ERR_INVALID_ARG, "observed statement felt %u is not a canonical field element (>= p)", i);
}

// per-AIR shape checks, constraint program compilation and upload, lowered lookup programs.  `jit`: also load the
// NVRTC kernels of large programs for the proof (its constraint evaluation and LogUp row build); `check_jit`: the
// trace-check kernels of large constraint programs (the constraint check and census, the constraint guard)
void mdn_session::bind_airs(const mdn_statement* st, const mdn_matrix* traces, bool jit, bool check_jit) {
    u32 k = st->n_airs, lb = params.log_blowup;
    airs.resize(k); log_heights.resize(k);
    for (u32 i = 0; i < k; i++) {
        const mdn_air& a = st->airs[i];
        if (traces[i].width != a.width) fail(MDN_ERR_INVALID_ARG, "trace %u width %u does not match AIR width %u", i, traces[i].width, a.width);
        if (a.log_quotient_degree > lb)
            fail(MDN_ERR_DOMAIN, "log_quotient_degree %u > log_blowup %u", a.log_quotient_degree, lb);
        log_qd = std::max(log_qd, a.log_quotient_degree);
        if (traces[i].log_height + lb > 32) fail(MDN_ERR_DOMAIN, "LDE log order %u exceeds two-adicity 32", traces[i].log_height + lb);
        if (a.width == 0) fail(MDN_ERR_INVALID_ARG, "AIR %u has zero width", i);
        log_heights[i] = traces[i].log_height;
        // parse + upload the constraint program
        AirHost& h = airs[i];
        h.desc = a;
        Compiled cp = compile_oplist(i, a, st->n_public_values, a.program, a.program_words, false, 0);
        bool uses_sel = cp.uses_sel;
        u32 n_slots = cp.n_slots;
        std::vector<u32>& code = cp.code;
        u32 nk = (u32)cp.consts.size();
        std::vector<u64> hostp((code.size() + 1) / 2 + nk + 2, 0);
        memcpy(hostp.data(), code.data(), code.size() * sizeof(u32));
        size_t const_off = (code.size() + 1) / 2;
        for (u32 j = 0; j < nk; j++) hostp[const_off + j] = cp.consts[j];
        // periodic columns: table[col][m] = P_col(s^(n/maxp) * w_{maxp*B}^m), m < maxp*B
        // (prover/periodic.rs:49-98; the column is interpolated over the size-maxp subgroup)
        size_t per_off = hostp.size();
        if (a.num_periodic_columns) {
            if (!a.periodic_values) fail(MDN_ERR_INVALID_ARG, "AIR %u: periodic_values is NULL", i);
            if (a.log_max_period > traces[i].log_height) fail(MDN_ERR_INVALID_ARG, "AIR %u: periodic column period exceeds the trace height", i);
            size_t mp = (size_t)1 << a.log_max_period, np = a.num_periodic_columns, tl = mp << lb;
            u64 wp_inv = gl::inv(gl::two_adic_generator(a.log_max_period)), mp_inv = gl::inv((u64)mp);
            u64 sh = gl::exp_pow2(gl::lde_shift(traces[i].log_height + lb), traces[i].log_height - a.log_max_period);
            u64 wq = gl::two_adic_generator(a.log_max_period + lb);
            hostp.resize(per_off + np * tl);
            std::vector<u64> coef(mp);
            for (size_t c = 0; c < np; c++) {
                for (size_t kq = 0; kq < mp; kq++) {        // naive inverse DFT (periods are tiny)
                    u64 acc = 0, wk = gl::pow(wp_inv, kq), xx = 1;
                    for (size_t rr = 0; rr < mp; rr++) {
                        u64 v = a.periodic_values[rr * np + c];
                        if (v >= gl::P) fail(MDN_ERR_INVALID_ARG, "AIR %u: non-canonical periodic value", i);
                        acc = gl::add(acc, gl::mul(v, xx)); xx = gl::mul(xx, wk);
                    }
                    coef[kq] = gl::mul(acc, mp_inv);
                }
                u64 pt = sh;
                for (size_t m2 = 0; m2 < tl; m2++) {
                    u64 acc = 0;
                    for (size_t kq = mp; kq-- > 0;) acc = gl::add(gl::mul(acc, pt), coef[kq]);
                    hostp[per_off + c * tl + m2] = acc;
                    pt = gl::mul(pt, wq);
                }
            }
        }
        h.program.alloc(hostp.size(), stream);
        CUDA_OK(cudaMemcpyAsync(h.program.p, hostp.data(), hostp.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        h.dev.code = (const u32*)h.program.p;
        h.dev.consts = h.program.p + const_off;
        h.dev.periodic = a.num_periodic_columns ? h.program.p + per_off : nullptr;
        h.dev.n_instr = (u32)(code.size() / 4); h.dev.n_slots = std::max(1u, n_slots); h.dev.uses_selectors = uses_sel;
        h.dev.log_max_period = a.log_max_period; h.dev.n_periodic = a.num_periodic_columns;
        // large programs: straight-line kernels compiled once per program (jit.hpp); the interpreter stays the fallback
        h.jit = {}; h.n_constraints = a.program[3];
        if (jit) load_jit(h, a.program, a.program_words, jit::MODE_CONSTRAINTS, 0, {{JIT_PROOF, "k_jit", 0}});
        if (check_jit)   // the keys carry the mode as the lookup kernel's carries "LKUP"
            load_jit(h, a.program, a.program_words, jit::MODE_CHECK, 0,
                     {{JIT_CHECK, "k_jit_check", 0x4348454Bull}, {JIT_CENSUS, "k_jit_census", 0x43454E53ull}});   // "CHEK", "CENS"
        // lowered LookupAir -> the aux trace of this AIR is built on the device (commit_aux)
        h.has_lookup = a.lookup != nullptr;
        if (h.has_lookup) {
            const bool v2 = a.lookup->program && a.lookup->program_words >= 2 && a.lookup->program[0] == 0x504B4C4Du && a.lookup->program[1] == 2;
            h.lookup_words.clear(); h.n_regs = 0;
            LookupSplit split;
            if (v2) {
                split = split_lookup_v2(i, a, st->n_public_values, *a.lookup);
                h.lookup_words = std::move(split.v1); h.n_regs = split.n_regs;
                h.lookup_v1 = mdn_lookup{a.lookup->num_columns, (u32)h.lookup_words.size(), h.lookup_words.data()};
            } else h.lookup_v1 = *a.lookup;
            const mdn_lookup& lk = h.lookup_v1;
            h.lookup_cols = lk.num_columns;
            if (!v2 && (lk.num_columns != a.aux_width || a.num_aux_values != 1)) fail(MDN_ERR_INVALID_ARG, "AIR %u: a lookup program needs aux_width == num_columns and num_aux_values == 1", i);
            if (lk.num_columns == 0 || lk.num_columns > mk::LOGUP_MAX_COLS) fail(MDN_ERR_UNSUPPORTED, "AIR %u: at most %u lookup columns", i, mk::LOGUP_MAX_COLS);
            Compiled lc = compile_oplist(i, a, st->n_public_values, lk.program, lk.program_words, true, lk.num_columns);
            // code | consts | raw periodic matrix, on the device
            auto upload = [&](const Compiled& c, DevBuf& buf, mk::AirDev& d) {
                size_t c_off = (c.code.size() + 1) / 2, p_off = c_off + c.consts.size() + 2;
                size_t np = a.num_periodic_columns, mp = (size_t)1 << a.log_max_period;
                std::vector<u64> hp(p_off + np * mp, 0);
                memcpy(hp.data(), c.code.data(), c.code.size() * sizeof(u32));
                for (size_t j = 0; j < c.consts.size(); j++) hp[c_off + j] = c.consts[j];
                for (size_t q = 0; q < np * mp; q++) hp[p_off + q] = a.periodic_values[q];   // canonical: checked above
                buf.alloc(hp.size(), stream);
                CUDA_OK(cudaMemcpyAsync(buf.p, hp.data(), hp.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
                CUDA_OK(cudaStreamSynchronize(stream));
                d = mk::AirDev{};
                d.code = (const u32*)buf.p; d.consts = buf.p + c_off;
                d.periodic = np ? buf.p + p_off : nullptr;
                d.n_instr = (u32)(c.code.size() / 4); d.n_slots = std::max(1u, c.n_slots);
                d.log_max_period = a.log_max_period; d.n_periodic = a.num_periodic_columns;
            };
            upload(lc, h.lookup_program, h.lookup_dev);
            if (v2) {
                // the register updates as constraints: the m-th FOLD (emitted in constraint order) becomes STORE m, and
                // AUX(0, num_columns + q) becomes REGISTER q
                Compiled rc = compile_oplist(i, a, st->n_public_values, split.regs.data(), (u32)split.regs.size(), false, 0);
                u32 m = 0;
                for (size_t q = 0; q < rc.code.size(); q += 4) {
                    const u32 op = rc.code[q] & 0xff;
                    if (op == 15) rc.code[q + 1] = m++;
                    else if (op == 1) rc.code[q + 3] -= lk.num_columns;
                }
                upload(rc, h.reg_program, h.reg_dev);
            }
            h.lookup_prep = h.reg_prep = false;
            for (u32 j = 0; j < lk.program[2]; j++) h.lookup_prep |= lk.program[5 + 3 * (size_t)j] == 15;
            for (u32 j = 0; v2 && j < split.regs[2]; j++) h.reg_prep |= split.regs[5 + 3 * (size_t)j] == 15;
            if (jit) load_jit(h, lk.program, lk.program_words, jit::MODE_LOOKUP, lk.num_columns, {{JIT_LOGUP, "k_jit", 0x4C4B5550ull}});   // "LKUP"
        }
    }
}

// The entry points `entries` of the cubin of program w (n_words words, compiled in `mode` for n_cols columns) into AIR
// h's kernel slots, when the program has at least jit_min_nodes nodes.  The session caches each entry point in
// jit_kernels under the program's hash salted with the entry's salt, so AIRs with the same program share one kernel
// and its first-use state.  A compile or load failure leaves the AIR on the interpreter and says why in jit_note.
void mdn_session::load_jit(AirHost& h, const u32* w, u32 n_words, jit::Mode mode, u32 n_cols, std::initializer_list<JitEntry> entries) {
    if (!jit_min_nodes || w[2] < jit_min_nodes) return;
    try {
        const u64 key = jit::fnv1a(w, n_words) ^ ((u64)n_words << 40);
        bool cached = true;
        for (const JitEntry& e : entries) cached &= jit_kernels.count(key ^ e.salt) != 0;
        if (!cached) {
            std::string file;
            const std::vector<char>& cubin = jit::cubin_for(w, n_words, nullptr, mode, n_cols, &file);
            std::vector<std::shared_ptr<jit::Kernel>> kns;
            try {
                for (const JitEntry& e : entries) {
                    kns.push_back(std::make_shared<jit::Kernel>());
                    if (kns.size() == 1) kns[0]->load(cubin, e.name);
                    else kns.back()->load(*kns[0], e.name);
                }
            } catch (const std::exception& e) {
                if (file.empty()) throw;
                throw std::runtime_error(std::string(e.what()) + " (cubin read from " + file + ")");
            }
            size_t q = 0;
            for (const JitEntry& e : entries) jit_kernels[key ^ e.salt] = kns[q++];
        }
        for (const JitEntry& e : entries) h.jit[e.pass] = jit_kernels[key ^ e.salt];
    } catch (const std::exception& e) { jit_note = e.what(); }
}

// The verdict of kernel kn's first use in pass p: whether the interpreter's results stand.  A disagreement -- or any
// comparison while MDN_JIT_FORCE_DISAGREE=1, which lets tests run every fallback -- retires the kernel for the rest of
// the session, clears the caller's used flag and sets the pass's note; it wins over an agreement of an AIR sharing the
// kernel.  An agreement marks a kernel on its first use as checked, unless `promote` is false (a pass with more
// comparisons to come).
bool mdn_session::settle_jit(jit::Kernel& kn, JitPass p, bool differs, u64* used, bool promote) {
    const char* force = getenv("MDN_JIT_FORCE_DISAGREE");
    if (differs || (force && !strcmp(force, "1"))) {
        kn.checked = -1;
        if (used) *used = 0;
        jit_note = JIT_DISAGREED[p];
        return true;
    }
    if (promote && kn.checked == 0) kn.checked = 1;
    return false;
}

// The first-use comparison of pass p on the device: every twin's kernel words against its interpreter words (`all_ranks`:
// the verdict of every rank of a split proof, which must all take the same branch), settled by settle_jit.  When the
// interpreter's results stand they are copied over the kernel's, for exactly the words compared.
bool mdn_session::compare_jit(jit::Kernel& kn, JitPass p, u64* used, std::initializer_list<Twin> twins, bool all_ranks) {
    DevBuf word; word.alloc(1, stream);
    CUDA_OK(cudaMemsetAsync(word.p, 0, sizeof(u64), stream));
    for (const Twin& t : twins) if (t.n) mk::launch_compare(t.kernel, t.interp, t.n, (u32*)word.p, stream);
    u64 differs = 0;
    CUDA_OK(cudaMemcpyAsync(&differs, word.p, sizeof differs, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaGetLastError());
    if (all_ranks && sharded()) {
        std::vector<u64> all(shard_world);
        if (allgather(allgather_ctx, &differs, all.data(), 1) != 0) fail(MDN_ERR_INVALID_ARG, "all-gather callback failed");
        for (u64 f : all) differs |= f;
    }
    if (!settle_jit(kn, p, differs != 0, used)) return false;
    for (const Twin& t : twins) if (t.n) CUDA_OK(cudaMemcpyAsync(t.kernel, t.interp, t.n * sizeof(u64), cudaMemcpyDeviceToDevice, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    return true;
}

// public values, TraceOrder and the NTT tables of every height (`tables` false: the height limit only, for a check)
void mdn_session::bind_order(const mdn_statement* st, bool tables) {
    u32 k = st->n_airs;
    publics.assign(st->public_values, st->public_values + st->n_public_values);
    // TraceOrder: stable sort on (log_height, instance)  (order.rs)
    order.resize(k);
    for (u32 i = 0; i < k; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](u32 a, u32 b) { return log_heights[a] < log_heights[b]; });
    log_max_n = log_heights[order.back()];
    for (u32 i = 0; i < k; i++) {
        if (tables) ntt(log_heights[i]);   // validates the supported range early
        else if (log_heights[i] > 22) fail(MDN_ERR_UNSUPPORTED, "trace height 2^%u exceeds the supported 2^22", log_heights[i]);
    }
}

// the transcript starts from the caller's pre-bound challenger (duplex) or the installed hash challenger
void mdn_session::bind_challenger(const mdn_challenger* chal) {
    Duplex& ch = tr.ch;
    ch.perm = perm();
    if (byte_hash()) {
        ch.hashed = true; ch.keccak = (hash_kind == MDN_HASH_KECCAK); ch.bin = hash_ch_in; ch.bout = hash_ch_out;      // mdn_session_set_hash_challenger
        if (ch.keccak && ch.bin.size() % 8) fail(MDN_ERR_INVALID_ARG, "Keccak hash challenger: the input buffer must be whole 64-bit words");
    } else {
        if (!chal) fail(MDN_ERR_INVALID_ARG, "null challenger");
        for (int i = 0; i < 12; i++) ch.st[i] = chal->sponge_state[i];
        if (chal->input_len > 7 || chal->output_len > 8) fail(MDN_ERR_INVALID_ARG, "malformed challenger state");
        for (u32 i = 0; i < chal->input_len; i++) ch.in[i] = chal->input_buffer[i];
        ch.in_len = chal->input_len; ch.out_len = chal->output_len;
    }
}

// the rest of prove_begin: main traces committed, randomness sampled
void mdn_session::upload_and_commit_main(const mdn_matrix* traces, bool on_device) {
    u32 k = (u32)airs.size(), lb = params.log_blowup;
    // 1. upload + transpose main traces (proof order), LDE, LMCS  (mod.rs:326-341)
    size_t coef_total = 0, lde_total = 0;
    for (u32 j = 0; j < k; j++) {
        u32 inst = order[j];
        size_t N = (size_t)1 << log_heights[inst];
        coef_total += N * airs[inst].desc.width; lde_total += (N << lb) * airs[inst].desc.width;
    }
    main_c.coef_buf.alloc(coef_total, stream);
    main_c.lde_buf.alloc(lde_total, stream);
    size_t co = 0, lo = 0;
    for (u32 j = 0; j < k; j++) {
        u32 inst = order[j];
        size_t N = (size_t)1 << log_heights[inst];
        u32 w = airs[inst].desc.width;
        main_c.mats.push_back(CommittedMat{main_c.lde_buf.p + lo, main_c.coef_buf.p + co, log_heights[inst], w});
        co += N * w; lo += (N << lb) * w;
    }
    // H2D copies run on a second stream, so the LDE of matrix j overlaps the copy of matrix j+1
    // (copies of pinned buffers are asynchronous; pageable buffers degrade to a staged copy).
    std::vector<DevBuf> staging(k);
    if (!on_device && sharded()) {
        // A proof split over G ranks: every rank copies 1/G of the rows of every trace to its GPU, transposes that slice
        // and stores it into the column-major trace of EVERY rank over NVLink, so each PCIe link carries 1/G of the
        // trace instead of all of it.  Traces too short to split are copied whole by every rank.
        const u32 lg = shard_log_g;
        auto slice_rows = [&](u32 ln) -> size_t { return ln >= lg + 5 ? ((size_t)1 << (ln - lg)) : ((size_t)1 << ln); };
        for (u32 j = 0; j < k; j++) staging[j].alloc(slice_rows(main_c.mats[j].log_n) * main_c.mats[j].width, stream);
        shard_barrier();                       // the coefficient buffer is a fresh allocation on every rank
        CUDA_OK(cudaEventRecord(copy_ev[7], stream));
        CUDA_OK(cudaStreamWaitEvent(copy_stream, copy_ev[7], 0));
        mk::PeerPtrs bad{};
        for (u32 g = 0; g < shard_world; g++) bad.p[g] = sync_flags.p[g] + 16;
        // smallest matrix first, and the LDE of a matrix is queued as soon as every rank's slice of it has arrived, so
        // the copies of the later matrices (copy stream) hide behind the LDE of the earlier ones, as on one GPU
        std::vector<u32> by_size(k);
        for (u32 j = 0; j < k; j++) by_size[j] = j;
        std::stable_sort(by_size.begin(), by_size.end(), [&](u32 a, u32 b) { return staging[a].n < staging[b].n; });
        for (u32 q = 0; q < k; q++) {
            const u32 j = by_size[q];
            const mdn_matrix& m = traces[order[j]];
            CommittedMat& cm = main_c.mats[j];
            const bool whole = cm.log_n < lg + 5;
            size_t rows = slice_rows(cm.log_n), row0 = whole ? 0 : rows * shard_rank;
            host_to_device(staging[j].p, m.values + row0 * cm.width, rows * cm.width);
            CUDA_OK(cudaEventRecord(copy_ev[q % 7], copy_stream));
            CUDA_OK(cudaStreamWaitEvent(stream, copy_ev[q % 7], 0));
            {
                ProfScope ps(prof, PC_TRANSPOSE);
                if (whole) mk::launch_transpose_rm_to_cm(staging[j].p, cm.coef, 1u << cm.log_n, cm.width, (u32*)d_flag.p, stream);
                else mk::launch_transpose_slice_push(staging[j].p, peers_of(cm.coef), bad, shard_world, (u32)row0, (u32)rows, 1u << cm.log_n, cm.width, stream);
            }
            shard_barrier();                   // every rank's slice of this matrix has arrived everywhere
            if (q + 1 == k) CUDA_OK(cudaEventRecord(ev[1], stream));
            keep_raw_main(j, nullptr);
            lde_matrix(cm);
        }
    } else if (!on_device) {
        for (u32 j = 0; j < k; j++) staging[j].alloc(((size_t)1 << main_c.mats[j].log_n) * main_c.mats[j].width, stream);
        CUDA_OK(cudaEventRecord(copy_ev[7], stream));
        CUDA_OK(cudaStreamWaitEvent(copy_stream, copy_ev[7], 0));
        // smallest matrix first: only its copy is exposed, every later copy hides behind the LDE of its predecessors
        // (the committed order of the matrices does not depend on the order in which they are prepared)
        std::vector<u32> by_size(k);
        for (u32 j = 0; j < k; j++) by_size[j] = j;
        std::stable_sort(by_size.begin(), by_size.end(), [&](u32 a, u32 b) { return staging[a].n < staging[b].n; });
        for (u32 q = 0; q < k; q++) {
            u32 j = by_size[q];
            const mdn_matrix& m = traces[order[j]];
            host_to_device(staging[j].p, m.values, staging[j].n);
            CUDA_OK(cudaEventRecord(copy_ev[q % 7], copy_stream));
            CUDA_OK(cudaStreamWaitEvent(stream, copy_ev[q % 7], 0));
            {
                ProfScope ps(prof, PC_TRANSPOSE);
                mk::launch_transpose_rm_to_cm(staging[j].p, main_c.mats[j].coef, 1u << main_c.mats[j].log_n, main_c.mats[j].width, (u32*)d_flag.p, stream);
            }
            if (q + 1 == k) CUDA_OK(cudaEventRecord(ev[1], stream));
            keep_raw_main(j, nullptr);
            lde_matrix(main_c.mats[j]);   // queued behind the copy of this matrix; overlaps the copy of the next one
        }
    } else {
        // device traces: a transpose (row-major) or an ingest (column-major) per matrix; a split proof does the same on
        // every rank, each from its own whole copy.  A LogUp build reads a column-major trace where the caller keeps it.
        for (u32 j = 0; j < k; j++) upload_matrix(traces[order[j]], true, main_c.mats[j].coef, col_major);
        CUDA_OK(cudaEventRecord(ev[1], stream));
        for (u32 j = 0; j < k; j++) { keep_raw_main(j, col_major ? traces[order[j]].values : nullptr); lde_matrix(main_c.mats[j]); }
    }
    staging.clear();
    check_input_flag("a main trace");
    lde_and_commit(main_c, &timings.lde_main, &timings.hash_main, true);
    CUDA_OK(cudaEventRecord(ev[2], stream));
    tr.send_commitment(main_c.root);
    memcpy(dbg_roots[0], main_c.root, 32);
    // 2. randomness (mod.rs:344-349)
    u32 max_rand = 0;
    for (auto& a : airs) max_rand = std::max(max_rand, a.desc.num_randomness);
    for (u32 i = 0; i < max_rand; i++) randomness.push_back(tr.ch.sample_ext());
    in_proof = true;
}

// Preprocessed::build (preprocessed.rs:63-131): the declared matrices sorted by (height, AIR index), coset LDE on
// the canonical shift of their own height, one aligned LMCS tree.  Kept on the device until replaced.
void mdn_session::set_preprocessed(const mdn_statement* st, const mdn_matrix* mats) {
    if (in_proof) fail(MDN_ERR_INVALID_ARG, "set_preprocessed called inside a proof");
    prep_c = Committed(); has_prep = false; prep_air.clear(); prep_log_h.clear();
    if (!mats) return;
    if (!st) fail(MDN_ERR_INVALID_ARG, "null argument");
    u32 lb = params.log_blowup;
    if (lb == 0 || lb > 4) fail(MDN_ERR_UNSUPPORTED, "log_blowup must be in 1..=4");
    std::vector<u32> ids;
    for (u32 i = 0; i < st->n_airs; i++) {
        if (mats[i].width != st->airs[i].preprocessed_width) fail(MDN_ERR_INVALID_ARG, "AIR %u: preprocessed matrix width %u does not match the declared %u", i, mats[i].width, st->airs[i].preprocessed_width);
        if (!mats[i].width) continue;
        if (!mats[i].values) fail(MDN_ERR_INVALID_ARG, "AIR %u: preprocessed matrix is NULL", i);
        if (mats[i].log_height + lb > 32) fail(MDN_ERR_DOMAIN, "LDE log order %u exceeds two-adicity 32", mats[i].log_height + lb);
        ntt(mats[i].log_height);
        ids.push_back(i);
    }
    if (ids.empty()) return;
    std::stable_sort(ids.begin(), ids.end(), [&](u32 a, u32 b) { return mats[a].log_height < mats[b].log_height; });
    size_t coef_total = 0, lde_total = 0;
    for (u32 i : ids) { size_t N = (size_t)1 << mats[i].log_height; coef_total += N * mats[i].width; lde_total += (N << lb) * mats[i].width; }
    prep_c.coef_buf.alloc(coef_total, stream); prep_c.lde_buf.alloc(lde_total, stream);
    size_t co = 0, lo = 0;
    for (u32 i : ids) {
        size_t N = (size_t)1 << mats[i].log_height;
        prep_c.mats.push_back(CommittedMat{prep_c.lde_buf.p + lo, prep_c.coef_buf.p + co, mats[i].log_height, mats[i].width});
        co += N * mats[i].width; lo += (N << lb) * mats[i].width;
        upload_matrix(mats[i], false, prep_c.mats.back().coef);
    }
    check_input_flag("a preprocessed trace");
    lde_and_commit(prep_c, nullptr, nullptr);
    prep_air = ids;
    for (u32 i : ids) prep_log_h.push_back(mats[i].log_height);
    has_prep = true;
}

// the raw main trace of a LogUp AIR for its aux build, and of every AIR for the constraint guard: the caller's
// column-major device trace when there is one (read in place: the caller keeps it unchanged until the aux commit),
// otherwise a copy made before the in-place inverse NTT
void mdn_session::keep_raw_main(u32 j, const u64* caller_cm) {
    AirHost& h = airs[order[j]];
    if (!h.has_lookup && !constraint_guard) return;
    if (caller_cm) { h.raw_main_cm = caller_cm; return; }
    CommittedMat& m = main_c.mats[j];
    size_t n = ((size_t)1 << m.log_n) * m.width;
    h.raw_main.alloc(n, stream);
    CUDA_OK(cudaMemcpyAsync(h.raw_main.p, m.coef, n * sizeof(u64), cudaMemcpyDeviceToDevice, stream));
    h.raw_main_cm = h.raw_main.p;
}

// The raw rows of AIR i's preprocessed trace in the installed bundle, column-major on the trace domain: re-derived from
// the bundle's coefficients by a forward NTT with shift 1 (exact), once per proof or check, into airs[i].raw_prep, so
// the bundle needs no raw copy.  The LogUp build and the constraint guard of one proof share the derivation.  The
// bundle holds AIR i at its height and width (checked by prove_begin, or by check_bundle_prep for a lookup check).
const u64* mdn_session::bundle_prep_rows(u32 i) {
    AirHost& h = airs[i];
    if (h.raw_prep.p) return h.raw_prep.p;
    const u32 q = (u32)(std::find(prep_air.begin(), prep_air.end(), i) - prep_air.begin());
    const CommittedMat& pm = prep_c.mats[q];
    const size_t N = (size_t)1 << pm.log_n;
    h.raw_prep.alloc(N * pm.width, stream);
    std::vector<mk::FwdItem> items;
    for (u32 c = 0; c < pm.width; c++) items.push_back(mk::FwdItem{pm.coef + (size_t)c * N, h.raw_prep.p + (size_t)c * N, 0, 0});
    DevBuf d_items; d_items.alloc(items.size() * sizeof(mk::FwdItem) / sizeof(u64), stream);
    CUDA_OK(cudaMemcpyAsync(d_items.p, items.data(), items.size() * sizeof(mk::FwdItem), cudaMemcpyHostToDevice, stream));
    mk::launch_fwd_ntt((const mk::FwdItem*)d_items.p, pm.width, ntt(pm.log_n).T, premul_unshifted(pm.log_n).P, stream);
    return h.raw_prep.p;
}

// The lookup checks take no preprocessed argument: an AIR whose lookup program reads preprocessed columns reads the
// installed bundle, which must hold that AIR at its height and width.  Refused before any device work.
void mdn_session::check_bundle_prep(u32 i) {
    if (!airs[i].has_lookup || !airs[i].lookup_prep) return;
    const u32 q = (u32)(std::find(prep_air.begin(), prep_air.end(), i) - prep_air.begin());
    if (!has_prep || q == prep_air.size())
        fail(MDN_ERR_INVALID_ARG, "AIR %u: its lookup program reads preprocessed columns, but the installed preprocessed bundle does not hold AIR %u (mdn_session_set_preprocessed)", i, i);
    const CommittedMat& pm = prep_c.mats[q];
    if (pm.log_n != log_heights[i] || pm.width != airs[i].desc.preprocessed_width)
        fail(MDN_ERR_INVALID_ARG, "AIR %u: the installed preprocessed bundle holds it as 2^%u rows of %u columns, the call needs 2^%u rows of %u", i, pm.log_n, pm.width, log_heights[i], airs[i].desc.preprocessed_width);
}

// build_logup_aux_trace (air/src/lookup/aux_builder.rs:49-97) for proof position j: fraction collection and
// per-row sums on the trace domain, exclusive EF prefix sum into column 0, committed final = the grand total.
// prep_cm: the raw column-major preprocessed rows the lookup program reads, or NULL when it reads none.
void mdn_session::build_logup_aux(u32 j, const u64* main_cm, const u64* prep_cm, u64* aux_cm, u64 final_out[2], bool registers) {
    AirHost& h = airs[order[j]];
    u32 ln = log_heights[order[j]];
    size_t N = (size_t)1 << ln;
    DevBuf totals, scratch, fin;
    totals.alloc(2 * N, stream); scratch.alloc(2 * ((N + 2047) / 2048) + 2, stream); fin.alloc(2, stream);
    mk::LogupArgs la;
    la.main_cm = main_cm; la.prep_cm = prep_cm; la.log_n = ln; la.n_cols = h.lookup_cols; la.prog = h.lookup_dev;
    la.publics = d_publics.p; la.challenges = d_randomness.p; la.aux_cm = aux_cm; la.totals = totals.p; la.bad_flag = (u32*)d_flag.p;
    {
        ProfScope ps(prof, PC_CONSTRAINTS);
        if (jit::Kernel* kn = row_kernel(h, JIT_LOGUP)) {
            jit::LookupJitArgs ja{};
            ja.main_lde = la.main_cm; ja.prep_lde = prep_cm; ja.publics = la.publics; ja.challenges = la.challenges;
            ja.periodic = h.lookup_dev.periodic; ja.aux_cm = aux_cm; ja.totals = totals.p; ja.bad_flag = la.bad_flag;
            ja.log_n = ln; ja.n_periodic = h.lookup_dev.n_periodic; ja.log_max_period = h.lookup_dev.log_max_period;
            launch_jit(*kn, ja, N);
            if (unchecked(*kn)) {
                // the interpreter builds the same rows into scratch buffers: fraction columns and row totals are compared
                DevBuf aux2, tot2;
                const size_t C = h.lookup_cols;
                aux2.alloc(2 * C * N, stream); tot2.alloc(2 * N, stream);
                mk::LogupArgs lb2 = la; lb2.aux_cm = aux2.p; lb2.totals = tot2.p;
                if (mk::launch_logup_rows(lb2, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "lookup program too large for the interpreter");
                compare_jit(*kn, JIT_LOGUP, nullptr, {{aux_cm + 2 * N, aux2.p + 2 * N, 2 * (C - 1) * N}, {totals.p, tot2.p, 2 * N}});
            }
        } else if (mk::launch_logup_rows(la, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "lookup program too large for the interpreter");
        mk::launch_ef_exclusive_scan(totals.p, N, aux_cm, aux_cm + N, fin.p, scratch.p, stream);
        if (h.n_regs && registers) {   // a version-2 program's register columns, after the LogUp columns
            DevBuf reg_scratch;
            reg_scratch.alloc(mk::register_scratch_words(ln, h.n_regs), stream);
            mk::RegisterArgs ra{};
            ra.main_cm = main_cm; ra.prep_cm = prep_cm; ra.log_n = ln; ra.n_regs = h.n_regs; ra.col0 = h.lookup_cols; ra.prog = h.reg_dev;
            ra.publics = d_publics.p; ra.challenges = d_randomness.p; ra.aux_cm = aux_cm; ra.scratch = reg_scratch.p; ra.bad_flag = (u32*)d_flag.p;
            const int rc = mk::launch_register_columns(ra, stream);
            if (rc < 0) fail(MDN_ERR_UNSUPPORTED, "register program too large for the interpreter");
            if (rc > 0) fail(MDN_ERR_CUDA, "AIR %u: register column kernels: %s", order[j], cudaGetErrorString((cudaError_t)rc));
        }
    }
    CUDA_OK(cudaMemcpyAsync(final_out, fin.p, 2 * sizeof(u64), cudaMemcpyDeviceToHost, stream));
    u32 flag = 0;
    CUDA_OK(cudaMemcpyAsync(&flag, d_flag.p, sizeof flag, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    if (!constraint_guard) h.raw_main.release();   // the guard reads it after the build (commit_aux releases it)
    if (flag) {
        CUDA_OK(cudaMemsetAsync(d_flag.p, 0, 8, stream));
        if (flag & 2) fail(MDN_ERR_INVALID_ARG, "AIR %u: LogUp denominator must be non-zero", order[j]);   // aux_builder.rs:240-243
        fail(MDN_ERR_INVALID_ARG, "an aux trace contains a non-canonical field element (>= p)");
    }
}

// Statement::eval_external (statement.rs:94-110) on the current aux values, instance order: 0 when every assertion is
// zero or no callback is installed, > 0 with *failed = the non-zero assertion, < 0 for a ReductionError
int mdn_session::eval_external(u32* failed) {
    if (!external_check) return 0;
    u32 k = (u32)airs.size();
    std::vector<std::vector<u64>> by_inst(k);
    for (u32 j = 0; j < k; j++) by_inst[order[j]] = aux_values_p[j];
    std::vector<const u64*> vp(k); std::vector<u32> vn(k); std::vector<uint8_t> lh(k);
    for (u32 i = 0; i < k; i++) { vp[i] = by_inst[i].data(); vn[i] = (u32)by_inst[i].size() / 2; lh[i] = (uint8_t)log_heights[i]; }
    return external_check(external_ctx, (const u64*)randomness.data(), (u32)randomness.size(), vp.data(), vn.data(), lh.data(), k, failed);
}

// ---------------------------------------------------------------------------------------------
// the trace checks' shared host steps
// ---------------------------------------------------------------------------------------------
namespace {
const mdn_challenger no_challenger{};   // for the checks that take their challenges as an argument: nothing is observed

// the interaction items {column, flag node, multiplicity, denominator} of a lowered lookup program (compiled by
// bind_airs, so the header and the items are in range)
struct LookupItems {
    const u32* items; u32 n;
    explicit LookupItems(const mdn_lookup& lk) : items(lk.program + 5 + 3 * (size_t)lk.program[2]), n(lk.program[3]) {}
    u32 column(u32 q) const { return items[4 * (size_t)q]; }
    u32 flag(u32 q) const { return items[4 * (size_t)q + 1]; }
};
}  // namespace

// The start of a trace check: a fresh proof state, the statement validated (`chal` NULL-checked as mdn_prove does;
// &no_challenger when nothing is observed) and its AIRs compiled (`check_jit`: with the trace-check kernels of large
// constraint programs).  The caller validates what it takes besides and then calls bind_order, in that order: the order
// of the errors a call reports is part of its behaviour.
mdn_session::CheckStart mdn_session::start_check(const mdn_statement* st, const mdn_matrix* traces, const mdn_challenger* chal, u32 flags, const void* out, bool check_jit) {
    const bool cm = column_major(flags);
    reset_proof();
    prof.st = stream; prof.reset();
    if (!out) fail(MDN_ERR_INVALID_ARG, "null argument");
    validate_statement(st, traces, chal);
    if (cm) for (u32 i = 0; i < st->n_airs; i++) check_column_major(traces[i], "trace", i);
    bind_airs(st, traces, false, check_jit);
    return CheckStart{cm, (flags & MDN_FLAG_DEVICE_TRACES) != 0, st->n_airs};
}

// Raw main traces of the instances `insts`, column-major, laid out in that order in main_c.coef_buf; column-major
// device traces are read where the caller keeps them (only read: the const_cast feeds the common pointer type).
// Returns each instance's trace, NULL for the instances not staged.
std::vector<u64*> mdn_session::stage_main(const mdn_matrix* traces, const std::vector<u32>& insts, bool cm, bool on_device) {
    std::vector<u64*> main_cm(airs.size(), nullptr);
    size_t total = 0;
    if (!cm) for (u32 i : insts) total += ((size_t)1 << log_heights[i]) * airs[i].desc.width;
    main_c.coef_buf.alloc(total, stream);
    size_t co = 0;
    for (u32 i : insts) {
        main_cm[i] = cm ? const_cast<u64*>(traces[i].values) : main_c.coef_buf.p + co;
        if (!cm) co += ((size_t)1 << log_heights[i]) * airs[i].desc.width;
    }
    for (u32 i : insts) upload_matrix(traces[i], on_device, main_cm[i], cm);   // column-major: check only
    check_input_flag("a main trace");
    return main_cm;
}

// challenges given as an argument (2 words per extension element): as many as the AIRs draw, canonical
u32 mdn_session::check_randomness(const u64* rnd) {
    u32 max_rand = 0;
    for (auto& a : airs) max_rand = std::max(max_rand, a.desc.num_randomness);
    if (max_rand && !rnd) fail(MDN_ERR_INVALID_ARG, "randomness is NULL");
    for (u32 i = 0; i < 2 * max_rand; i++) if (rnd[i] >= gl::P) fail(MDN_ERR_INVALID_ARG, "randomness word %u is not a canonical field element (>= p)", i);
    return max_rand;
}

// device copies of the public values and of the challenges (n_words words), read by the lookup and constraint kernels
void mdn_session::upload_leaves(const u64* rnd, size_t n_words) {
    d_publics.alloc(std::max<size_t>(1, publics.size()), stream);
    if (!publics.empty()) CUDA_OK(cudaMemcpyAsync(d_publics.p, publics.data(), publics.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
    d_randomness.alloc(std::max<size_t>(1, n_words), stream);
    if (n_words) CUDA_OK(cudaMemcpyAsync(d_randomness.p, rnd, n_words * sizeof(u64), cudaMemcpyHostToDevice, stream));
}

// Allocates buffers whose size depends on the data (each with its word count), refusing with MDN_ERR_UNSUPPORTED and
// "<what> <GiB> of device memory: <why>" when the device's and the arena's free memory cannot hold them, or when an
// allocation fails.
void mdn_session::alloc_checked(const std::string& what, std::initializer_list<std::pair<DevBuf*, size_t>> bufs) {
    size_t need = 0;
    for (auto& b : bufs) need += b.second * sizeof(u64);
    auto too_large = [&](const char* why) {
        fail(MDN_ERR_UNSUPPORTED, "%s %.1f GiB of device memory: %s", what.c_str(), need / 1073741824.0, why);
    };
#ifndef MDN_EMULATED   // tests/emu has no device memory of its own: only the failed allocation below is reported there
    size_t arena_b = 0, free_b = 0, total_b = 0;
    for (auto& sl : arena.slabs) arena_b += sl.size - sl.used;
    CUDA_OK(cudaMemGetInfo(&free_b, &total_b));
    char msg[64];
    snprintf(msg, sizeof msg, "%.1f GiB are free", (free_b + arena_b) / 1073741824.0);
    if (need > free_b + arena_b) too_large(msg);
#endif
    try {
        for (auto& b : bufs) b.first->alloc(b.second, stream);
    } catch (const MdnError&) {   // an out-of-memory allocation leaves no error behind; nothing has been launched on them yet
        cudaGetLastError();
        too_large("the allocation failed");
    }
}

// Whether AIR i has a lowered lookup program, which the lookup checks run.  An AIR without one counts in `skipped`,
// and `given` -- a per-AIR argument of the check given for it, or NULL -- is refused.
bool mdn_session::lookup_air(u32 i, const char* given, u32& skipped) {
    if (airs[i].has_lookup) return true;
    skipped++;
    if (given) fail(MDN_ERR_INVALID_ARG, "AIR %u: %s given for an AIR without a lookup program", i, given);
    return false;
}

// The lookup checks' NVRTC kernels (jit.hpp MODE_LOOKUP_CHECK) of every AIR whose lookup program -- its interaction
// part, for a version-2 program -- has at least jit_min_nodes nodes: one cubin per program and column count, cached in
// jit_kernels with the keys "LKCB" / "LKCF" / "LKCC" (one per entry point, each with its own first-use state).  Proofs
// and the constraint checks never call this; the emulator build never specialises.
void mdn_session::load_lookup_check_jit() {
    jit_lookup_check_used.assign(airs.size(), 0);
    for (AirHost& h : airs) {
        for (JitPass p : {JIT_BALANCE, JIT_FOLD, JIT_FOLD_CENSUS}) h.jit[p].reset();
#ifndef MDN_EMULATED
        const mdn_lookup& lk = h.lookup_v1;
        const u64 c = (u64)lk.num_columns << 32;
        if (h.has_lookup)
            load_jit(h, lk.program, lk.program_words, jit::MODE_LOOKUP_CHECK, lk.num_columns,
                     {{JIT_BALANCE, "k_jit_balance", c ^ 0x4C4B4342ull}, {JIT_FOLD, "k_jit_fold", c ^ 0x4C4B4346ull},
                      {JIT_FOLD_CENSUS, "k_jit_fold_census", c ^ 0x4C4B4343ull}});
#endif
    }
}

// Allocates buffers that are optional to the caller: false, with nothing allocated, when the device's and the arena's
// free memory cannot hold them or an allocation fails.
bool mdn_session::alloc_if_free(std::initializer_list<std::pair<DevBuf*, size_t>> bufs) {
    size_t need = 0;
    for (auto& b : bufs) need += b.second * sizeof(u64);
#ifndef MDN_EMULATED
    size_t arena_b = 0, free_b = 0, total_b = 0;
    for (auto& sl : arena.slabs) arena_b += sl.size - sl.used;
    CUDA_OK(cudaMemGetInfo(&free_b, &total_b));
    if (need > free_b + arena_b) return false;
#endif
    try {
        for (auto& b : bufs) b.first->alloc(b.second, stream);
    } catch (const MdnError&) {
        cudaGetLastError();
        for (auto& b : bufs) b.first->release();
        return false;
    }
    return true;
}

// ---------------------------------------------------------------------------------------------
// check_constraints: every constraint of every AIR on every trace row, without a proof  (debug.rs:70-214)
// ---------------------------------------------------------------------------------------------
// The validation, program compilation and main-trace upload of prove_begin; challenges from the statement felts and
// the instance shape only (no commitment is observed); aux traces from the device LogUp build, the host callback or
// zeros; the session's external check; then k_check_rows per AIR in instance order.  Nothing of the last proof's
// outputs, timings or introspection is touched; the caller releases the proof arena afterwards.
// prepare_check is everything before the row pass, shared with constraint_census.
void mdn_session::check_constraints(const mdn_statement* st, const mdn_matrix* traces, const mdn_matrix* prep, const mdn_challenger* chal,
                                    mdn_aux_builder build_aux, void* aux_ctx, u32 flags, mdn_constraint_report* out) {
    if (!out) fail(MDN_ERR_INVALID_ARG, "null argument");
    CheckSetup cs;
    prepare_check(st, traces, prep, chal, build_aux, aux_ctx, flags, out, cs);
    const u32 k = st->n_airs;
    std::vector<mk::CheckArgs> ca(k);
    for (u32 i = 0; i < k; i++) {
        const u32 j = cs.pos[i];
        ca[i] = row_args<mk::CheckArgs>(i, j, main_c.mats[j].coef, cs.prep_cm[i].p, cs.periodic[i].p, d_aux_values.p);
    }
    check_rows(ca, cs.ext_rc == 0, out);
    if (cs.ext_rc > 0) { out->kind = 2; out->constraint = cs.ext_failed; }
    out->holds = cs.ext_rc == 0 && out->failing_rows == 0;
}

// The row pass (debug.rs:120-214) of check_constraints and of the constraint guard: k_jit_check when AIR i has the
// NVRTC check kernel, else k_check_rows, on every row of every AIR, instance order (ca[i]: AIR i's traces, program and
// leaves; the rows and result words are set here).  `out` gets the failing-row total over all AIRs and, when `locate`,
// kind 1 with the least failing (instance, row, constraint) and that constraint's value, from a one-row relaunch of
// k_check_rows; every other field is zero.
void mdn_session::check_rows(std::vector<mk::CheckArgs>& ca, bool locate, mdn_constraint_report* out) {
    const u32 k = (u32)ca.size();
    // per AIR the lowest (row, constraint) that is non-zero and the failing-row count; 4 scratch words for the probe;
    // then per AIR the interpreter's two words of a check kernel's first-use comparison
    const size_t twin = 2 * (size_t)k + 4;
    DevBuf res; res.alloc(twin + 2 * (size_t)k, stream);
    std::vector<u64> host_res(twin + 2 * (size_t)k, 0);
    for (u32 i = 0; i < k; i++) host_res[2 * i] = host_res[twin + 2 * i] = ~0ull;
    CUDA_OK(cudaMemcpyAsync(res.p, host_res.data(), host_res.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
    jit_check_used.assign(k, 0);
    std::vector<u32> first_use;
    for (u32 i = 0; i < k; i++) {
        mk::CheckArgs& c = ca[i];
        c.row0 = 0; c.n_rows = (size_t)1 << c.log_n;
        c.first = (unsigned long long*)(res.p + 2 * i); c.failing_rows = (unsigned long long*)(res.p + 2 * i + 1);
        jit::Kernel* kn = row_kernel(airs[i], JIT_CHECK);
        if (!kn) {
            if (mk::launch_check_rows(c, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: constraint program too large for the interpreter", i);
            continue;
        }
        jit::CheckJitArgs ja = check_jit_args(c);
        ja.first = c.first; ja.failing_rows = c.failing_rows; ja.row0 = c.row0; ja.n_rows = c.n_rows;
        launch_jit(*kn, ja, c.n_rows);
        jit_check_used[i] = 1;
        if (unchecked(*kn)) {
            // first use of this kernel in the session: the interpreter checks the same rows into its own two words
            mk::CheckArgs t = c;
            t.first = (unsigned long long*)(res.p + twin + 2 * i); t.failing_rows = (unsigned long long*)(res.p + twin + 2 * i + 1);
            if (mk::launch_check_rows(t, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: constraint program too large for the interpreter", i);
            first_use.push_back(i);
        }
    }
    CUDA_OK(cudaMemcpyAsync(host_res.data(), res.p, host_res.size() * sizeof(u64), cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaGetLastError());
    for (u32 i : first_use) {
        const bool differs = host_res[2 * i] != host_res[twin + 2 * i] || host_res[2 * i + 1] != host_res[twin + 2 * i + 1];
        if (settle_jit(*airs[i].jit[JIT_CHECK], JIT_CHECK, differs, &jit_check_used[i])) {
            host_res[2 * i] = host_res[twin + 2 * i]; host_res[2 * i + 1] = host_res[twin + 2 * i + 1];
        }
    }

    memset(out, 0, sizeof *out);
    for (u32 i = 0; i < k; i++) out->failing_rows += host_res[2 * i + 1];
    if (locate) for (u32 i = 0; i < k; i++) {
        u64 f = host_res[2 * i];
        if (f == ~0ull) continue;
        out->kind = 1; out->instance = i; out->row = f >> 32; out->constraint = (u32)f;
        // the value: the same kernel on that one row, recording constraint K (its own atomics go to scratch words)
        mk::CheckArgs c = ca[i];
        c.row0 = out->row; c.n_rows = 1; c.probe_k = out->constraint; c.probe_value = res.p + 2 * (size_t)k;
        c.first = (unsigned long long*)(res.p + 2 * (size_t)k + 2); c.failing_rows = (unsigned long long*)(res.p + 2 * (size_t)k + 3);
        if (mk::launch_check_rows(c, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: constraint program too large for the interpreter", i);
        CUDA_OK(cudaMemcpyAsync(out->value, res.p + 2 * (size_t)k, 2 * sizeof(u64), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        break;
    }
}

// The constraint guard (mdn_session_set_constraint_guard), from commit_aux once the aux traces and values are final and
// the external assertions hold, before the aux commitment: the row pass of check_constraints on what this proof is about
// to commit.  Main rows: the raw copies of keep_raw_main (or the caller's column-major traces); aux rows: aux_c's
// coefficient slots, still raw; `flat_values`: the aux values in proof order; challenges and publics: the proof's own.
// Preprocessed rows: bundle_prep_rows, shared with the proof's LogUp build.  Every rank of a split proof runs the whole
// check on its own whole copies.  A non-zero constraint fails the proof with MDN_ERR_CONSTRAINT_VIOLATED.
void mdn_session::guard_constraints(const std::vector<u64>& flat_values) {
    const u32 k = (u32)airs.size();
    ProfScope ps(prof, PC_CONSTRAINTS);
    DevBuf values; values.alloc(std::max<size_t>(1, flat_values.size()), stream);
    if (!flat_values.empty()) CUDA_OK(cudaMemcpyAsync(values.p, flat_values.data(), flat_values.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
    std::vector<mk::CheckArgs> ca(k);
    for (u32 j = 0; j < k; j++) {
        const u32 i = order[j];
        AirHost& h = airs[i];
        const u64* prep = h.desc.preprocessed_width ? bundle_prep_rows(i) : nullptr;   // present: checked by prove_begin
        ca[i] = row_args<mk::CheckArgs>(i, j, h.raw_main_cm, prep, h.raw_periodic.p, values.p);
    }
    mdn_constraint_report rep;
    check_rows(ca, true, &rep);
    rep.holds = rep.failing_rows == 0;
    guard_report = rep;
    if (!rep.holds)
        fail(MDN_ERR_CONSTRAINT_VIOLATED, "constraint %u of AIR %u is non-zero at row %llu (%llu failing rows): the statement does not hold, nothing was committed",
             rep.constraint, rep.instance, (unsigned long long)rep.row, (unsigned long long)rep.failing_rows);
}

// Validation, challenges, main / preprocessed / periodic upload, aux traces and the external check of a constraint
// check (debug.rs:70-118): after it, main_c / aux_c hold the raw column-major traces in proof order (cs.pos[instance]),
// d_publics / d_randomness / d_aux_values the leaves, and cs the per-instance preprocessed and periodic buffers and
// the external check's outcome.
void mdn_session::prepare_check(const mdn_statement* st, const mdn_matrix* traces, const mdn_matrix* prep, const mdn_challenger* chal,
                                mdn_aux_builder build_aux, void* aux_ctx, u32 flags, const void* out, CheckSetup& cs) {
    const auto [cm, on_device, k] = start_check(st, traces, chal, flags, out, true);
    const bool dev_built = cm && dev_aux;   // aux traces from the device aux builder
    // the preprocessed traces come with the call (debug.rs re-materialises BaseAir::preprocessed_trace), not from the
    // session's committed bundle
    bool expected = false;
    for (u32 i = 0; i < k; i++) expected |= st->airs[i].preprocessed_width > 0;
    if (expected && !prep) fail(MDN_ERR_INVALID_ARG, "preprocessed presence mismatch: AIRs declare preprocessed columns but no preprocessed traces are given");
    if (prep) for (u32 i = 0; i < k; i++) {
        if (prep[i].width != st->airs[i].preprocessed_width) fail(MDN_ERR_INVALID_ARG, "AIR %u: preprocessed width %u does not match the declared %u", i, prep[i].width, st->airs[i].preprocessed_width);
        if (!prep[i].width) continue;
        if (!prep[i].values) fail(MDN_ERR_INVALID_ARG, "AIR %u: preprocessed matrix is NULL", i);
        if (prep[i].log_height != traces[i].log_height) fail(MDN_ERR_INVALID_ARG, "AIR %u: preprocessed height 2^%u differs from the main trace height 2^%u", i, prep[i].log_height, traces[i].log_height);
    }
    if (build_aux && cm) fail(MDN_ERR_INVALID_ARG, "with MDN_FLAG_COLUMN_MAJOR the aux traces come from the device aux builder (mdn_session_set_device_aux_builder): build_aux must be NULL");
    if (build_aux && on_device) fail(MDN_ERR_UNSUPPORTED, "an aux builder needs host-resident main traces");
    bind_order(st, false);

    // challenges: Statement::observe + observe_shape, no commitment (debug.rs:87-97)
    bind_challenger(chal);
    for (u32 i = 0; i < st->n_observe_felts; i++) tr.ch.observe(st->observe_felts[i]);
    tr.ch.observe(k);
    for (u32 i = 0; i < k; i++) tr.ch.observe(log_heights[i]);
    u32 max_rand = 0;
    for (auto& a : airs) max_rand = std::max(max_rand, a.desc.num_randomness);
    for (u32 i = 0; i < max_rand; i++) randomness.push_back(tr.ch.sample_ext());

    // raw main and aux traces, column-major, proof order (the layout build_logup_aux reads)
    std::vector<u32>& pos = cs.pos;
    pos.assign(k, 0);
    for (u32 j = 0; j < k; j++) pos[order[j]] = j;
    const std::vector<u64*> main_cm = stage_main(traces, order, cm, on_device);
    size_t aux_total = 0;
    for (u32 i = 0; i < k; i++) aux_total += ((size_t)1 << log_heights[i]) * 2 * airs[i].desc.aux_width;
    aux_c.coef_buf.alloc(aux_total, stream);
    size_t ao = 0;
    for (u32 j = 0; j < k; j++) {
        u32 inst = order[j];
        main_c.mats.push_back(CommittedMat{nullptr, main_cm[inst], log_heights[inst], airs[inst].desc.width});
        aux_c.mats.push_back(CommittedMat{nullptr, aux_c.coef_buf.p + ao, log_heights[inst], 2 * airs[inst].desc.aux_width});
        ao += ((size_t)1 << log_heights[inst]) * 2 * airs[inst].desc.aux_width;
    }
    std::vector<DevBuf>& prep_cm = cs.prep_cm;
    std::vector<DevBuf>& periodic = cs.periodic;
    prep_cm.clear(); prep_cm.resize(k);
    periodic.clear(); periodic.resize(k);
    if (prep) {
        for (u32 i = 0; i < k; i++) if (prep[i].width) {
            prep_cm[i].alloc(((size_t)1 << prep[i].log_height) * prep[i].width, stream);
            upload_matrix(prep[i], false, prep_cm[i].p);
        }
        check_input_flag("a preprocessed trace");
    }
    for (u32 i = 0; i < k; i++) {
        const mdn_air& a = st->airs[i];
        if (!a.num_periodic_columns) continue;
        size_t n = ((size_t)1 << a.log_max_period) * a.num_periodic_columns;   // canonical: checked by bind_airs
        periodic[i].alloc(n, stream);
        CUDA_OK(cudaMemcpyAsync(periodic[i].p, a.periodic_values, n * sizeof(u64), cudaMemcpyHostToDevice, stream));
    }

    // aux traces built with those challenges (debug.rs:99-106), as mdn_prove builds them
    std::vector<std::vector<u64>> aux_host(k), val_host(k);
    if (build_aux) for (u32 i = 0; i < k; i++) {
        const mdn_air& a = st->airs[i];
        if (a.lookup) continue;   // built on the device
        aux_host[i].assign(((size_t)1 << traces[i].log_height) * 2 * a.aux_width, 0);
        val_host[i].assign(2 * (size_t)a.num_aux_values + 1, 0);
        std::vector<u64> r;
        for (u32 q = 0; q < a.num_randomness; q++) { r.push_back(randomness[q].a); r.push_back(randomness[q].b); }
        r.push_back(0);
        if (build_aux(aux_ctx, i, &traces[i], r.data(), aux_host[i].data(), val_host[i].data()) != 0)
            fail(MDN_ERR_AUX_BUILDER, "aux builder failed for instance %u", i);
    }
    if (dev_built) for (u32 i = 0; i < k; i++)
        if (!st->airs[i].lookup) call_device_aux_builder(i, traces[i], aux_c.mats[pos[i]].coef, val_host[i]);
    upload_leaves((const u64*)randomness.data(), 2 * randomness.size());
    std::vector<u64> flat_values;
    aux_values_p.assign(k, {}); aux_values_off.assign(k, 0);
    for (u32 j = 0; j < k; j++) {
        u32 inst = order[j];
        AirHost& h = airs[inst];
        u32 w = 2 * h.desc.aux_width;
        size_t N = (size_t)1 << log_heights[inst];
        u64 logup_final[2] = {0, 0};
        if (h.has_lookup) build_logup_aux(j, main_c.mats[j].coef, cs.prep_cm[inst].p, aux_c.mats[j].coef, logup_final);   // no LDE: the buffer is raw
        else if (w && dev_built) upload_matrix(mdn_matrix{aux_c.mats[j].coef, log_heights[inst], w}, true, aux_c.mats[j].coef, true);   // check only
        else if (w && build_aux) upload_matrix(mdn_matrix{aux_host[inst].data(), log_heights[inst], w}, false, aux_c.mats[j].coef);
        else if (w) CUDA_OK(cudaMemsetAsync(aux_c.mats[j].coef, 0, N * w * sizeof(u64), stream));
        aux_values_off[j] = flat_values.size();
        for (u32 v = 0; v < 2 * h.desc.num_aux_values; v++) {
            u64 x = h.has_lookup ? logup_final[v] : (build_aux || dev_built ? val_host[inst][v] : 0);
            if (x >= gl::P) fail(MDN_ERR_INVALID_ARG, "non-canonical aux value");
            aux_values_p[j].push_back(x); flat_values.push_back(x);
        }
    }
    if (build_aux || dev_built) check_input_flag("an aux trace");
    d_aux_values.alloc(std::max<size_t>(1, flat_values.size()), stream);
    if (!flat_values.empty()) CUDA_OK(cudaMemcpyAsync(d_aux_values.p, flat_values.data(), flat_values.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));

    // external assertions before the row checks (debug.rs:108-118); a failing one is reported, the rows still run
    cs.ext_failed = 0;
    cs.ext_rc = eval_external(&cs.ext_failed);
    if (cs.ext_rc < 0) fail(MDN_ERR_EXTERNAL_ASSERTION, "eval_external reported a reduction error");
}

// ---------------------------------------------------------------------------------------------
// constraint_census: every violated constraint of every AIR, per constraint and in row order, without a proof
// ---------------------------------------------------------------------------------------------
// prepare_check as check_constraints; then per AIR (instance order) k_census_rows fills that AIR's slice of one
// per-row count array, concatenated in instance order, and its per-constraint tally; one exclusive scan of the counts
// gives every failing row its first failure slot and the total.  k_census_list then writes the first max_failures
// records in (instance, row, constraint) order, and in probe mode the values at the reported tallies' first rows (plus
// the least failure's, when truncation drops it).  Counts, minima, maxima and the scan do not depend on the order
// the atomics ran in, so neither does anything reported.
void mdn_session::constraint_census(const mdn_statement* st, const mdn_matrix* traces, const mdn_matrix* prep, const mdn_challenger* chal,
                                    mdn_aux_builder build_aux, void* aux_ctx, u32 flags, mdn_constraint_failure* failures, u64 max_failures,
                                    mdn_constraint_tally* tallies, u64 max_tallies, mdn_constraint_census_report* out) {
    CheckSetup cs;
    prepare_check(st, traces, prep, chal, build_aux, aux_ctx, flags, out, cs);
    const u32 k = st->n_airs;

    // per-row counts of all AIRs (u32, instance order), their offsets, one tally table per AIR, two counters
    std::vector<size_t> row_base(k + 1, 0), tally_base(k + 1, 0);
    for (u32 i = 0; i < k; i++) {
        row_base[i + 1] = row_base[i] + ((size_t)1 << log_heights[i]);
        tally_base[i + 1] = tally_base[i] + 3 * (size_t)airs[i].n_constraints;
    }
    const size_t rows = row_base[k];
    DevBuf counts, offsets, tally, words, scratch;
    counts.alloc((rows + 1) / 2, stream);
    offsets.alloc(rows, stream);
    tally.alloc(std::max<size_t>(1, tally_base[k]), stream);
    words.alloc(2, stream);                       // rows with a failure, violations
    scratch.alloc((rows + 2047) / 2048, stream);  // block sums of the scan
    std::vector<u64> host_tally(std::max<size_t>(1, tally_base[k]), 0);
    for (size_t q = 0; q < tally_base[k]; q += 3) host_tally[q + 1] = ~0ull;
    CUDA_OK(cudaMemcpyAsync(tally.p, host_tally.data(), host_tally.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
    CUDA_OK(cudaMemsetAsync(words.p, 0, 2 * sizeof(u64), stream));
    u32* d_counts = reinterpret_cast<u32*>(counts.p);
    std::vector<mk::CensusArgs> ca(k);
    jit_check_used.assign(k, 0);
    u64 checked_rows = 0;   // failing rows of AIRs whose row pass was compared on first use (not in words[0])
    for (u32 i = 0; i < k; i++) {
        const u32 j = cs.pos[i];
        mk::CensusArgs& c = ca[i];
        c = row_args<mk::CensusArgs>(i, j, main_c.mats[j].coef, cs.prep_cm[i].p, cs.periodic[i].p, d_aux_values.p);
        c.n_cons = airs[i].n_constraints;
        c.instance = i;
        c.row_count = d_counts + row_base[i];
        c.tally = (unsigned long long*)(tally.p + tally_base[i]);
        c.failing_rows = (unsigned long long*)words.p;
        c.offsets = offsets.p + row_base[i];
        jit::Kernel* kn = row_kernel(airs[i], JIT_CENSUS);
        if (!kn) {
            if (mk::launch_census_rows(c, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: constraint program too large for the interpreter", i);
            continue;
        }
        const size_t N = (size_t)1 << c.log_n, nt = 3 * (size_t)c.n_cons;
        jit::CheckJitArgs ja = check_jit_args(c);
        ja.failing_rows = c.failing_rows; ja.row_count = c.row_count; ja.tally = c.tally; ja.n_cons = c.n_cons;
        // first use of this kernel in the session: the kernel's failing rows go to a word of their own, and the
        // interpreter runs the same rows into its own counts, tally and word; all three must agree word for word
        const bool first_use = unchecked(*kn);
        DevBuf twin;
        if (first_use) {
            twin.alloc((N + 1) / 2 + nt + 2, stream);
            CUDA_OK(cudaMemcpyAsync(twin.p + (N + 1) / 2, host_tally.data() + tally_base[i], nt * sizeof(u64), cudaMemcpyHostToDevice, stream));
            CUDA_OK(cudaMemsetAsync(twin.p + (N + 1) / 2 + nt, 0, 2 * sizeof(u64), stream));
            ja.failing_rows = (unsigned long long*)(twin.p + (N + 1) / 2 + nt);
        }
        launch_jit(*kn, ja, N);
        jit_check_used[i] = 1;
        if (!first_use) continue;
        mk::CensusArgs t = c;
        t.row_count = reinterpret_cast<u32*>(twin.p); t.tally = (unsigned long long*)(twin.p + (N + 1) / 2);
        t.failing_rows = (unsigned long long*)(twin.p + (N + 1) / 2 + nt + 1);
        if (mk::launch_census_rows(t, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: constraint program too large for the interpreter", i);
        std::vector<u32> cnt_j(N), cnt_i(N);
        std::vector<u64> tw(nt + 2), tj(std::max<size_t>(1, nt));
        CUDA_OK(cudaMemcpyAsync(cnt_j.data(), c.row_count, N * sizeof(u32), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaMemcpyAsync(cnt_i.data(), twin.p, N * sizeof(u32), cudaMemcpyDeviceToHost, stream));
        if (nt) CUDA_OK(cudaMemcpyAsync(tj.data(), c.tally, nt * sizeof(u64), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaMemcpyAsync(tw.data(), twin.p + (N + 1) / 2, (nt + 2) * sizeof(u64), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        CUDA_OK(cudaGetLastError());
        const bool differs = cnt_j != cnt_i || !std::equal(tj.begin(), tj.begin() + nt, tw.begin()) || tw[nt] != tw[nt + 1];
        if (settle_jit(*kn, JIT_CENSUS, differs, &jit_check_used[i])) {   // the interpreter's counts and tally stand
            CUDA_OK(cudaMemcpyAsync(c.row_count, twin.p, N * sizeof(u32), cudaMemcpyDeviceToDevice, stream));
            if (nt) CUDA_OK(cudaMemcpyAsync(c.tally, twin.p + (N + 1) / 2, nt * sizeof(u64), cudaMemcpyDeviceToDevice, stream));
        }
        checked_rows += tw[nt + 1];
    }
    mk::launch_count_exclusive_scan(d_counts, rows, offsets.p, words.p + 1, scratch.p, stream);
    u64 host_words[2];
    CUDA_OK(cudaMemcpyAsync(host_tally.data(), tally.p, host_tally.size() * sizeof(u64), cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaMemcpyAsync(host_words, words.p, sizeof host_words, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaGetLastError());
    host_words[0] += checked_rows;

    // the failing (instance, constraint) pairs in order, and the least failure: the first failing instance's least
    // (first_row, constraint)
    std::vector<mdn_constraint_tally> all;
    size_t least = SIZE_MAX;
    for (u32 i = 0; i < k; i++)
        for (u32 c = 0; c < airs[i].n_constraints; c++) {
            const u64* t = host_tally.data() + tally_base[i] + 3 * (size_t)c;
            if (!t[0]) continue;
            all.push_back(mdn_constraint_tally{i, c, t[0], t[1], t[2], {0, 0}});
            if (least == SIZE_MAX || (all[least].instance == i && t[1] < all[least].first_row)) least = all.size() - 1;
        }
    memset(out, 0, sizeof *out);
    out->violations = host_words[1];
    out->n_failures = std::min<u64>(out->violations, max_failures);
    out->failing_constraints = all.size();
    out->n_tallies = std::min<u64>(all.size(), max_tallies);

    // values at the first rows of the reported tallies and of the least failure: probe mode, one launch per instance
    std::vector<size_t> probed;
    for (size_t q = 0; q < out->n_tallies; q++) probed.push_back(q);
    if (least != SIZE_MAX && least >= out->n_tallies) probed.push_back(least);   // `all` is in instance order: still sorted
    DevBuf d_probes, d_records, d_failures;
    if (!probed.empty()) {
        std::vector<u64> pr;
        for (size_t q : probed) { pr.push_back(all[q].first_row); pr.push_back(all[q].constraint); }
        d_probes.alloc(pr.size(), stream);
        d_records.alloc(4 * probed.size(), stream);
        CUDA_OK(cudaMemcpyAsync(d_probes.p, pr.data(), pr.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
        for (size_t b = 0; b < probed.size();) {
            u32 i = all[probed[b]].instance;
            size_t e = b;
            while (e < probed.size() && all[probed[e]].instance == i) e++;
            mk::CensusArgs c = ca[i];
            c.probes = d_probes.p + 2 * b; c.n_probes = e - b; c.failures = d_records.p + 4 * b;
            if (mk::launch_census_list(c, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: constraint program too large for the interpreter", i);
            b = e;
        }
    }
    // the first n_failures records, every AIR with a failing constraint writing its own slots
    if (out->n_failures) {
        d_failures.alloc(4 * out->n_failures, stream);
        for (u32 i = 0; i < k; i++) {
            bool any = false;
            for (u32 c = 0; c < airs[i].n_constraints && !any; c++) any = host_tally[tally_base[i] + 3 * (size_t)c] != 0;
            if (!any) continue;
            mk::CensusArgs c = ca[i];
            c.max_failures = out->n_failures; c.failures = d_failures.p;
            if (mk::launch_census_list(c, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: constraint program too large for the interpreter", i);
        }
    }
    std::vector<u64> records(4 * probed.size());
    if (!probed.empty()) CUDA_OK(cudaMemcpyAsync(records.data(), d_records.p, records.size() * sizeof(u64), cudaMemcpyDeviceToHost, stream));
    static_assert(sizeof(mdn_constraint_failure) == 4 * sizeof(u64), "mdn_constraint_failure is the kernel's record");
    if (out->n_failures) CUDA_OK(cudaMemcpyAsync(failures, d_failures.p, out->n_failures * sizeof(mdn_constraint_failure), cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaGetLastError());
    for (size_t q = 0; q < probed.size(); q++) { all[probed[q]].first_value[0] = records[4 * q + 2]; all[probed[q]].first_value[1] = records[4 * q + 3]; }
    for (size_t q = 0; q < out->n_tallies; q++) tallies[q] = all[q];

    // `first`: what check_constraints reports for the same call
    mdn_constraint_report& f = out->first;
    f.failing_rows = host_words[0];
    if (cs.ext_rc > 0) { f.kind = 2; f.constraint = cs.ext_failed; }
    else if (least != SIZE_MAX) {
        const mdn_constraint_tally& t = all[least];
        f.kind = 1; f.instance = t.instance; f.row = t.first_row; f.constraint = t.constraint;
        f.value[0] = t.first_value[0]; f.value[1] = t.first_value[1];
    }
    f.holds = cs.ext_rc == 0 && f.failing_rows == 0;
}

// ---------------------------------------------------------------------------------------------
// check_trace_balance: every active LogUp push keyed by its denominator, without a proof  (debug/trace/mod.rs:169-309)
// ---------------------------------------------------------------------------------------------
// start_check, then the main traces of the lookup AIRs staged; the challenges are an argument.  Per AIR with a lowered
// lookup program, k_balance_rows counts the pushes (which sizes the table), then inserts them; the boundary triples
// follow; k_balance_finish reduces every sum and compacts the unmatched denominators; when the report can hold them, a
// third row pass collects their pushes.  The host sorts what is reported.
void mdn_session::check_trace_balance(const mdn_statement* st, const mdn_matrix* traces, const u64* rnd, const u64* boundary, size_t n_boundary,
                                      const uint32_t* const* mutex_sites, u64 max_contrib, u32 flags, mdn_balance_report* out) {
    const CheckStart start = start_check(st, traces, &no_challenger, flags, out);
    const u32 k = start.k;
    bind_order(st, false);

    // arguments: challenges, boundary emissions, interaction counts, mutex annotations
    const u32 max_rand = check_randomness(rnd);
    if (n_boundary && !boundary) fail(MDN_ERR_INVALID_ARG, "boundary is NULL");
    if (n_boundary >= (1u << 24)) fail(MDN_ERR_UNSUPPORTED, "at most 2^24 - 1 boundary emissions");
    for (size_t q = 0; q < 3 * n_boundary; q++)
        if (boundary[q] >= gl::P) fail(MDN_ERR_INVALID_ARG, "boundary emission %zu: %s is not a canonical field element (>= p)", q / 3, q % 3 == 2 ? "the multiplicity" : "the denominator");
    struct Mutex { std::vector<u32> pos, group, site; };
    std::vector<Mutex> mx(k);
    u32 skipped = 0;
    for (u32 i = 0; i < k; i++) {
        const uint32_t* ann = mutex_sites ? mutex_sites[i] : nullptr;
        if (!lookup_air(i, ann ? "mutex sites" : nullptr, skipped)) continue;
        const LookupItems items(airs[i].lookup_v1);
        if (items.n >= (1u << 24)) fail(MDN_ERR_UNSUPPORTED, "AIR %u: at most 2^24 - 1 lookup interactions", i);
        if (!ann) continue;
        std::vector<u32> ids;
        for (u32 q = 0; q < items.n; q++) if (ann[q] != 0xFFFFFFFFu) ids.push_back(q);
        if (ids.size() > mk::BALANCE_MUTEX_MAX) fail(MDN_ERR_UNSUPPORTED, "AIR %u: %zu interactions in cached-encoding groups (at most %u)", i, ids.size(), mk::BALANCE_MUTEX_MAX);
        auto group_of = [&](u32 q) { return (items.column(q) << 16) | (ann[q] >> 16); };
        std::stable_sort(ids.begin(), ids.end(), [&](u32 a, u32 b) {
            return std::make_pair(group_of(a), ann[a] & 0xFFFFu) < std::make_pair(group_of(b), ann[b] & 0xFFFFu); });
        Mutex& m = mx[i];
        m.pos.assign(items.n, 0xFFFFFFFFu);
        for (size_t b = 0; b < ids.size(); b++) {
            u32 q = ids[b];
            if (b && group_of(ids[b - 1]) == group_of(q) && (ann[ids[b - 1]] & 0xFFFFu) == (ann[q] & 0xFFFFu) && items.flag(ids[b - 1]) != items.flag(q))
                fail(MDN_ERR_INVALID_ARG, "AIR %u: interactions %u and %u share mutex site %u of group %u but not a flag node (one site is one insert or batch call)", i, ids[b - 1], q, ann[q] & 0xFFFFu, ann[q] >> 16);
            m.pos[q] = (u32)b; m.group.push_back(group_of(q)); m.site.push_back(ann[q] & 0xFFFFu);
        }
    }

    for (u32 i = 0; i < k; i++) check_bundle_prep(i);
    std::vector<u32> lookups;
    for (u32 i = 0; i < k; i++) if (airs[i].has_lookup) lookups.push_back(i);
    const std::vector<u64*> main_cm = stage_main(traces, lookups, start.cm, start.on_device);
    upload_leaves(rnd, 2 * (size_t)max_rand);
    std::vector<DevBuf> d_mx(k);
    for (u32 i = 0; i < k; i++) {
        const Mutex& m = mx[i];
        if (m.group.empty()) continue;
        std::vector<u32> words(m.pos);
        words.insert(words.end(), m.group.begin(), m.group.end());
        words.insert(words.end(), m.site.begin(), m.site.end());
        d_mx[i].alloc((words.size() + 1) / 2, stream);
        CUDA_OK(cudaMemcpyAsync(d_mx[i].p, words.data(), words.size() * sizeof(u32), cudaMemcpyHostToDevice, stream));
    }
    DevBuf ctr; ctr.alloc(5, stream);
    CUDA_OK(cudaMemsetAsync(ctr.p, 0, 5 * sizeof(u64), stream));
    unsigned long long* counters = (unsigned long long*)ctr.p;
    std::vector<mk::BalanceArgs> ba(k);
    // k_jit_balance where the AIR has it.  `twin`: one of them is on its first use in the session, so every pass runs
    // the interpreter a second time, on every lookup AIR, into a table, counters and lists of its own (tw); the passes
    // compare the two and, on a disagreement, keep the interpreter's and retire the kernels on their first use.
    load_lookup_check_jit();
    std::vector<jit::Kernel*> bk(k);
    std::vector<u32> first_use;   // the AIRs whose kernel is on its first use
    for (u32 i = 0; i < k; i++) {
        bk[i] = row_kernel(airs[i], JIT_BALANCE);
        if (bk[i]) jit_lookup_check_used[i] = 1;
        if (bk[i] && unchecked(*bk[i])) first_use.push_back(i);
    }
    bool twin = !first_use.empty();
    DevBuf tw_ctr, tw_table, tw_mut, tw_con;
    mk::BalanceTable tw_t{};
    if (twin) { tw_ctr.alloc(5, stream); CUDA_OK(cudaMemsetAsync(tw_ctr.p, 0, 5 * sizeof(u64), stream)); }
    auto drop_jit = [&] {   // the interpreter's results stand from here on
        for (u32 i = 0; i < k; i++) if (bk[i]) { bk[i] = nullptr; jit_lookup_check_used[i] = 0; }
        twin = false;
    };
    // the verdict of a pass the twin compared: a disagreement retires the kernels on their first use and drops them all;
    // the kernels count as checked when the last pass of the call agrees
    auto settle = [&](bool differs, bool last) {
        bool fallback = false;
        for (u32 i : first_use) fallback |= settle_jit(*bk[i], JIT_BALANCE, differs, &jit_lookup_check_used[i], last);
        if (fallback) drop_jit();
        return fallback;
    };
    auto run_rows = [&](u32 mode) {
        for (u32 i = 0; i < k; i++) {
            if (!airs[i].has_lookup) continue;
            mk::BalanceArgs& b = ba[i];
            b.mode = mode;
            if (bk[i]) launch_jit(*bk[i], balance_jit_args(b), (size_t)1 << b.log_n);
            else if (mk::launch_balance_rows(b, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: lookup program too large for the interpreter", i);
            if (!twin) continue;
            mk::BalanceArgs c = b;
            c.t = tw_t; c.counters = (unsigned long long*)tw_ctr.p; c.mutex_out = tw_mut.p; c.contrib_out = tw_con.p;
            if (mk::launch_balance_rows(c, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: lookup program too large for the interpreter", i);
        }
    };
    // the twin's counters (after the stream's work so far)
    auto twin_counters = [&](u64 c2[5]) {
        CUDA_OK(cudaMemcpyAsync(c2, tw_ctr.p, 5 * sizeof(u64), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
    };
    // n triples of a list, sorted: the lists are written in the order the atomics ran
    auto sorted_triples = [&](const u64* d, u64 n) {
        std::vector<std::array<u64, 3>> v(n);
        if (n) CUDA_OK(cudaMemcpyAsync(v.data(), d, 3 * n * sizeof(u64), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        std::sort(v.begin(), v.end());
        return v;
    };
    for (u32 i = 0; i < k; i++) {
        if (!airs[i].has_lookup) continue;
        mk::BalanceArgs& b = ba[i];
        b = mk::BalanceArgs{};
        b.main_cm = main_cm[i]; b.prep_cm = airs[i].lookup_prep ? bundle_prep_rows(i) : nullptr; b.log_n = log_heights[i]; b.prog = airs[i].lookup_dev;
        b.publics = d_publics.p; b.challenges = d_randomness.p; b.instance = i;
        const u32 nc = LookupItems(airs[i].lookup_v1).n, na = (u32)mx[i].group.size();
        if (na) {
            const u32* w = (const u32*)d_mx[i].p;
            b.mutex_pos = w; b.mutex_group = w + nc; b.mutex_site = w + nc + na; b.n_mutex = na;
        }
        b.counters = counters;
    }

    // 1. count: the table holds at most every push, so 2x the pushes in slots keeps it at most half full
    run_rows(0);
    u64 cnt[5];
    CUDA_OK(cudaMemcpyAsync(cnt, ctr.p, sizeof cnt, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    if (twin) {
        u64 c2[5];
        twin_counters(c2);
        if (settle(c2[0] != cnt[0] || c2[1] != cnt[1], false)) { cnt[0] = c2[0]; cnt[1] = c2[1]; }
    }
    const u64 n_push = cnt[0] + n_boundary, n_mutex = cnt[1];
    u64 slots = 1024;
    while (slots < 2 * n_push) slots <<= 1;
    DevBuf table, unm, mut;
    alloc_checked("the balance table for " + std::to_string(n_push) + " pushes needs",
                  {{&table, 6 * slots}, {&unm, 6 * std::max<u64>(1, n_push)}, {&mut, 3 * std::max<u64>(1, n_mutex)}});
    mk::BalanceTable t;
    t.keys = table.p; t.sums = table.p + 2 * slots;
    t.count = (unsigned long long*)(table.p + 4 * slots); t.first = (unsigned long long*)(table.p + 5 * slots); t.mask = slots - 1;
    CUDA_OK(cudaMemsetAsync(t.keys, 0xFF, 2 * slots * sizeof(u64), stream));
    CUDA_OK(cudaMemsetAsync(t.sums, 0, 3 * slots * sizeof(u64), stream));
    CUDA_OK(cudaMemsetAsync(t.first, 0xFF, slots * sizeof(u64), stream));
    CUDA_OK(cudaMemsetAsync(ctr.p, 0, 5 * sizeof(u64), stream));
    // the twin's table of the same size; without the room for it this call runs the interpreter, the kernels unchecked
    if (twin && !alloc_if_free({{&tw_table, 6 * slots}, {&tw_mut, 3 * std::max<u64>(1, n_mutex)}})) drop_jit();
    if (twin) {
        tw_t.keys = tw_table.p; tw_t.sums = tw_table.p + 2 * slots;
        tw_t.count = (unsigned long long*)(tw_table.p + 4 * slots); tw_t.first = (unsigned long long*)(tw_table.p + 5 * slots); tw_t.mask = slots - 1;
        CUDA_OK(cudaMemsetAsync(tw_t.keys, 0xFF, 2 * slots * sizeof(u64), stream));
        CUDA_OK(cudaMemsetAsync(tw_t.sums, 0, 3 * slots * sizeof(u64), stream));
        CUDA_OK(cudaMemsetAsync(tw_t.first, 0xFF, slots * sizeof(u64), stream));
        CUDA_OK(cudaMemsetAsync(tw_ctr.p, 0, 5 * sizeof(u64), stream));
    }

    // 2. insert, boundary, finish
    for (auto& b : ba) { b.t = t; b.mutex_out = mut.p; }
    run_rows(1);
    if (twin) {
        // the same keys with the same sums, counts and least keys (placement follows the order of the atomics), and
        // the same mutex violations
        DevBuf cw; cw.alloc(3, stream);
        CUDA_OK(cudaMemsetAsync(cw.p, 0, 3 * sizeof(u64), stream));
        mk::launch_balance_compare(t, tw_t, (unsigned long long*)cw.p, stream);
        u64 w[3], c1[5], c2[5];
        CUDA_OK(cudaMemcpyAsync(w, cw.p, sizeof w, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaMemcpyAsync(c1, ctr.p, sizeof c1, cudaMemcpyDeviceToHost, stream));
        twin_counters(c2);
        CUDA_OK(cudaGetLastError());
        if (settle(w[0] != w[1] || w[2] || c1[1] != c2[1] || sorted_triples(mut.p, c1[1]) != sorted_triples(tw_mut.p, c2[1]), false)) {
            std::swap(table, tw_table); std::swap(mut, tw_mut); std::swap(t, tw_t);
            for (auto& b : ba) { b.t = t; b.mutex_out = mut.p; }
            CUDA_OK(cudaMemcpyAsync(ctr.p, tw_ctr.p, 5 * sizeof(u64), cudaMemcpyDeviceToDevice, stream));
        }
    }
    DevBuf bnd;
    if (n_boundary) {
        bnd.alloc(3 * n_boundary, stream);
        CUDA_OK(cudaMemcpyAsync(bnd.p, boundary, 3 * n_boundary * sizeof(u64), cudaMemcpyHostToDevice, stream));
        mk::launch_balance_boundary(t, bnd.p, (u32)n_boundary, stream);
    }
    mk::launch_balance_finish(t, counters, unm.p, stream);
    CUDA_OK(cudaMemcpyAsync(cnt, ctr.p, sizeof cnt, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    const u64 n_unm = cnt[4], n_distinct = cnt[3];
    std::vector<u64> uh(6 * n_unm), mh(3 * n_mutex);
    if (n_unm) CUDA_OK(cudaMemcpyAsync(uh.data(), unm.p, uh.size() * sizeof(u64), cudaMemcpyDeviceToHost, stream));
    if (n_mutex) CUDA_OK(cudaMemcpyAsync(mh.data(), mut.p, mh.size() * sizeof(u64), cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaGetLastError());

    // unmatched, ascending (c0, c1)
    std::vector<u64> ord(n_unm);
    for (u64 u = 0; u < n_unm; u++) ord[u] = u;
    std::sort(ord.begin(), ord.end(), [&](u64 a, u64 b) { return std::make_pair(uh[6 * a], uh[6 * a + 1]) < std::make_pair(uh[6 * b], uh[6 * b + 1]); });
    bal_unmatched.assign(n_unm, mdn_unmatched{});
    std::map<u64, u64> rank_of_slot;
    std::map<std::pair<u64, u64>, u64> rank_of_denom;
    u64 n_contrib = 0;
    for (u64 j = 0; j < n_unm; j++) {
        const u64* e = &uh[6 * ord[j]];
        mdn_unmatched& m = bal_unmatched[j];
        m.denom[0] = e[0]; m.denom[1] = e[1]; m.net_multiplicity = e[2]; m.n_pushes = e[3];
        u32 inst = (u32)(e[4] >> 48), q = (u32)(e[4] & 0xFFFFFFu);
        m.first_instance = inst == mk::BALANCE_BOUNDARY ? 0xFFFFFFFFu : inst;
        m.first_row = inst == mk::BALANCE_BOUNDARY ? ~0ull : (e[4] >> 24) & 0xFFFFFFu;
        m.first_interaction = q;
        rank_of_slot[e[5]] = j; rank_of_denom[{e[0], e[1]}] = j;
        n_contrib += e[3];
    }
    // 3. the pushes of the unmatched denominators, when the report can hold them
    bal_contrib.clear();
    const bool complete = n_contrib <= max_contrib;
    if (complete && n_contrib) {
        DevBuf con; con.alloc(3 * n_contrib, stream);
        CUDA_OK(cudaMemsetAsync(ctr.p, 0, 5 * sizeof(u64), stream));
        for (auto& b : ba) b.contrib_out = con.p;
        if (twin) {   // the twin collects from the finished table too
            tw_t = t;
            tw_con.alloc(3 * n_contrib, stream);
            CUDA_OK(cudaMemsetAsync(tw_ctr.p, 0, 5 * sizeof(u64), stream));
        }
        run_rows(2);
        CUDA_OK(cudaMemcpyAsync(cnt, ctr.p, sizeof cnt, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        if (twin) {
            u64 c2[5];
            twin_counters(c2);
            // a miscounting kernel may have written past the list: the interpreter's count bounds what is read
            if (settle(c2[2] != cnt[2] || sorted_triples(con.p, std::min(cnt[2], n_contrib)) != sorted_triples(tw_con.p, c2[2]), false)) {
                std::swap(con, tw_con); cnt[2] = c2[2];
            }
        }
        std::vector<u64> ch(3 * cnt[2]);
        if (cnt[2]) CUDA_OK(cudaMemcpyAsync(ch.data(), con.p, ch.size() * sizeof(u64), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        struct Rec { u64 rank, key, m; };
        std::vector<Rec> recs;
        for (u64 p = 0; p < cnt[2]; p++) recs.push_back({rank_of_slot.at(ch[3 * p]), ch[3 * p + 1], ch[3 * p + 2]});
        for (size_t q = 0; q < n_boundary; q++) {
            auto it = rank_of_denom.find({boundary[3 * q], boundary[3 * q + 1]});
            if (it != rank_of_denom.end()) recs.push_back({it->second, mk::balance_key(mk::BALANCE_BOUNDARY, 0, (u32)q), boundary[3 * q + 2]});
        }
        if (recs.size() != n_contrib) fail(MDN_ERR_CUDA, "balance check: %zu pushes collected, %llu counted", recs.size(), (unsigned long long)n_contrib);
        std::sort(recs.begin(), recs.end(), [](const Rec& a, const Rec& b) { return std::make_pair(a.rank, a.key) < std::make_pair(b.rank, b.key); });
        for (const Rec& r : recs) {
            mdn_balance_push p{};
            u32 inst = (u32)(r.key >> 48), q = (u32)(r.key & 0xFFFFFFu);
            p.multiplicity = r.m; p.interaction = q;
            if (inst == mk::BALANCE_BOUNDARY) { p.instance = 0xFFFFFFFFu; p.row = ~0ull; p.column = 0xFFFFFFFFu; }
            else { p.instance = inst; p.row = (r.key >> 24) & 0xFFFFFFu; p.column = LookupItems(airs[inst].lookup_v1).column(q); }
            bal_contrib.push_back(p);
        }
    }
    // every pass agreed: the kernels on their first use are checked (a call that lists no contributions checks the
    // count and insert passes)
    if (twin) settle(false, true);
    // mutex violations, (instance, row, column, group)
    std::vector<u64> mo(n_mutex);
    for (u64 v = 0; v < n_mutex; v++) mo[v] = v;
    std::sort(mo.begin(), mo.end(), [&](u64 a, u64 b) { return std::make_pair(mh[3 * a], mh[3 * a + 1]) < std::make_pair(mh[3 * b], mh[3 * b + 1]); });
    bal_mutex.clear();
    for (u64 v = 0; v < n_mutex && v < max_contrib; v++) {
        const u64* e = &mh[3 * mo[v]];
        mdn_mutex_violation mv{};
        mv.instance = (u32)(e[0] >> 32); mv.row = e[0] & 0xFFFFFFFFu; mv.column = (u32)(e[1] >> 32); mv.group = (u32)e[1]; mv.active_flags = (u32)e[2];
        bal_mutex.push_back(mv);
    }

    memset(out, 0, sizeof *out);
    out->n_pushes = n_push; out->n_denominators = n_distinct; out->n_unmatched = n_unm; out->n_mutex_violations = n_mutex;
    out->n_contributions = n_contrib; out->contributions_complete = complete; out->n_skipped_airs = skipped;
    out->unmatched = bal_unmatched.data(); out->contributions = complete ? bal_contrib.data() : nullptr;
    out->mutex_violations = bal_mutex.data(); out->n_mutex_listed = bal_mutex.size();
    out->holds = n_unm == 0 && n_mutex == 0;
}

// ---------------------------------------------------------------------------------------------
// check_lookup_folds: the constraint-path fold of every LogUp column on every row against an aux trace, without a
// proof  (debug/trace/mod.rs:191-207, builder.rs; the comparison of processor/src/trace/tests/lookup.rs:185-265)
// ---------------------------------------------------------------------------------------------
// start_check, then the main traces of the lookup AIRs staged; the challenges are an argument.  The aux traces come
// with the call (host row-major through the transpose, column-major device read in place) or from build_logup_aux on
// the same traces.  k_fold_rows runs once per AIR with a lowered lookup program; a second launch on the one failing row
// fetches its fold, expected and actual values.
// prepare_folds is everything before the row pass, shared with lookup_fold_census (which passes no folds_out).
void mdn_session::prepare_folds(const mdn_statement* st, const mdn_matrix* traces, const u64* rnd, const uint32_t* const* fold_marks,
                                const mdn_matrix* aux, const u64* const* aux_finals, u64* const* folds_out, u32 flags, const void* out,
                                FoldSetup& fs) {
    const auto [cm, on_device, k] = start_check(st, traces, &no_challenger, flags, out);
    fs.cm = cm; fs.on_device = on_device; fs.k = k;
    bind_order(st, false);

    // arguments: challenges, aux traces and their closing values, fold marks, fold buffers
    const u32 max_rand = check_randomness(rnd);
    if (!aux && aux_finals) fail(MDN_ERR_INVALID_ARG, "aux_finals given without aux: the device LogUp build supplies its own closing values");
    u32& skipped = fs.skipped;
    size_t& staging_words = fs.staging_words;
    for (u32 i = 0; i < k; i++) {
        const uint32_t* marks = fold_marks ? fold_marks[i] : nullptr;
        if (!lookup_air(i, marks ? "fold marks" : folds_out && folds_out[i] ? "a fold buffer" : nullptr, skipped)) continue;
        const u32 C = airs[i].lookup_cols;   // the folds cover the LogUp columns; an aux trace has every aux column
        if (aux) {
            const u32 aw = airs[i].desc.aux_width;
            if (aux[i].width != 2 * aw || aux[i].log_height != log_heights[i]) fail(MDN_ERR_INVALID_ARG, "AIR %u: the aux trace must be 2^%u rows of %u base columns", i, log_heights[i], 2 * aw);
            if (!aux[i].values) fail(MDN_ERR_INVALID_ARG, "aux trace %u is NULL", i);
            if (cm) check_column_major(aux[i], "aux trace", i);
            if (!aux_finals || !aux_finals[i]) fail(MDN_ERR_INVALID_ARG, "AIR %u: aux_finals is NULL", i);
            if (aux_finals[i][0] >= gl::P || aux_finals[i][1] >= gl::P) fail(MDN_ERR_INVALID_ARG, "AIR %u: aux_finals is not a canonical field element (>= p)", i);
        }
        if (folds_out && folds_out[i]) {
            if (on_device && ((uintptr_t)folds_out[i] & 15)) fail(MDN_ERR_INVALID_ARG, "AIR %u: a device fold buffer must be 16-byte aligned", i);
            if (!on_device) staging_words = std::max(staging_words, ((size_t)4 * C) << log_heights[i]);
        }
        if (!marks) continue;
        const LookupItems items(airs[i].lookup_v1);
        for (u32 q = 0; q < items.n; q++) {
            const u32 m = marks[q];
            if (m != 0 && m != 1 && m != 3) fail(MDN_ERR_INVALID_ARG, "AIR %u: fold mark %u of interaction %u (0, 1 or 3)", i, m, q);
            if (m != 3 && (q == 0 || items.column(q) != items.column(q - 1)))
                fail(MDN_ERR_INVALID_ARG, "AIR %u: interaction %u starts a column and must open a group (fold mark 3)", i, q);
            if (m == 0 && items.flag(q) != items.flag(q - 1))
                fail(MDN_ERR_INVALID_ARG, "AIR %u: interactions %u and %u are marked as one batch but do not share a flag node", i, q - 1, q);
        }
    }

    // raw main traces and aux slots of the lookup AIRs, column-major (column-major device aux traces are read where the
    // caller keeps them)
    for (u32 i = 0; i < k; i++) check_bundle_prep(i);
    std::vector<u32> lookups;
    for (u32 i = 0; i < k; i++) if (airs[i].has_lookup) lookups.push_back(i);
    fs.main_cm = stage_main(traces, lookups, cm, on_device);
    for (u32 i : lookups) if (airs[i].lookup_prep) bundle_prep_rows(i);
    fs.aux_cm.assign(k, nullptr);
    std::vector<u64*>& aux_cm = fs.aux_cm;
    size_t aux_total = 0;
    if (!(aux && cm)) for (u32 i : lookups) aux_total += ((size_t)1 << log_heights[i]) * 2 * airs[i].desc.aux_width;
    aux_c.coef_buf.alloc(aux_total, stream);
    size_t ao = 0;
    for (u32 i : lookups) {
        if (aux && cm) aux_cm[i] = const_cast<u64*>(aux[i].values);
        else { aux_cm[i] = aux_c.coef_buf.p + ao; ao += ((size_t)1 << log_heights[i]) * 2 * airs[i].desc.aux_width; }
    }
    if (aux) {
        for (u32 i : lookups) upload_matrix(aux[i], on_device, aux_cm[i], cm);
        check_input_flag("an aux trace");
    }
    upload_leaves(rnd, 2 * (size_t)max_rand);
    std::vector<DevBuf>& d_marks = fs.marks;
    d_marks.resize(k);
    for (u32 i = 0; i < k; i++) {
        if (!airs[i].has_lookup || !fold_marks || !fold_marks[i]) continue;
        const u32 nc = LookupItems(airs[i].lookup_v1).n;
        if (!nc) continue;
        d_marks[i].alloc(((size_t)nc + 1) / 2, stream);
        CUDA_OK(cudaMemcpyAsync(d_marks[i].p, fold_marks[i], nc * sizeof(u32), cudaMemcpyHostToDevice, stream));
    }
    // the prover path to check when no aux trace is given: k_logup_rows + the scan, as mdn_prove builds it
    fs.finals.assign(k, gl::e2(0, 0));
    std::vector<E2>& finals = fs.finals;
    std::vector<u32> pos(k);
    for (u32 j = 0; j < k; j++) pos[order[j]] = j;
    for (u32 i = 0; i < k; i++) {
        if (!airs[i].has_lookup) continue;
        if (aux) { finals[i] = gl::e2(aux_finals[i][0], aux_finals[i][1]); continue; }
        u64 fin[2] = {0, 0};
        build_logup_aux(pos[i], fs.main_cm[i], airs[i].raw_prep.p, aux_cm[i], fin, false);
        finals[i] = gl::e2(fin[0], fin[1]);
    }
    load_lookup_check_jit();
}

void mdn_session::check_lookup_folds(const mdn_statement* st, const mdn_matrix* traces, const u64* rnd, const uint32_t* const* fold_marks,
                                     const mdn_matrix* aux, const u64* const* aux_finals, u64* const* folds_out, u32 flags, mdn_fold_report* out) {
    FoldSetup fs;
    prepare_folds(st, traces, rnd, fold_marks, aux, aux_finals, folds_out, flags, out, fs);
    const u32 k = fs.k;
    const bool on_device = fs.on_device, cm = fs.cm;
    // host fold buffers are filled through one device staging buffer, sized for the largest of them
    DevBuf staging;
    if (fs.staging_words) alloc_checked("the folds of the largest AIR need", {{&staging, fs.staging_words}});

    // per AIR: {first (row << 32 | column), failing rows, zero U}; then the probe's 9 words and its scratch counters
    DevBuf res; res.alloc(3 * (size_t)k + 12, stream);
    std::vector<u64> host_res(3 * (size_t)k + 12, 0);
    for (u32 i = 0; i < k; i++) host_res[3 * i] = ~0ull;
    host_res[3 * (size_t)k + 9] = ~0ull;
    CUDA_OK(cudaMemcpyAsync(res.p, host_res.data(), host_res.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
    std::vector<mk::LookupFoldArgs> fa(k);
    for (u32 i = 0; i < k; i++) {
        if (!airs[i].has_lookup) continue;
        mk::LookupFoldArgs& f = fa[i];
        f = fold_args<mk::LookupFoldArgs>(i, fs);
        u64* user = folds_out ? folds_out[i] : nullptr;
        f.folds_out = user && !on_device ? staging.p : user; f.folds_cm = cm;
        f.row0 = 0; f.n_rows = (size_t)1 << log_heights[i];
        f.first = (unsigned long long*)(res.p + 3 * i); f.failing_rows = f.first + 1; f.zero_u = f.first + 2;
        if (jit::Kernel* kn = row_kernel(airs[i], JIT_FOLD)) {
            jit::LookupCheckJitArgs ja = fold_jit_args(f);
            ja.folds_out = f.folds_out; ja.folds_cm = f.folds_cm; ja.row0 = f.row0; ja.n_rows = f.n_rows;
            ja.first = f.first; ja.zero_u = f.zero_u;
            launch_jit(*kn, ja, f.n_rows);
            jit_lookup_check_used[i] = 1;
            if (unchecked(*kn)) {
                // the interpreter runs the same rows into its own three words and folds: both are compared
                const size_t fw = f.folds_out ? ((size_t)4 * f.n_cols) << f.log_n : 0;
                DevBuf tw; tw.alloc(4 + fw, stream);
                const u64 init[3] = {~0ull, 0, 0};   // first, failing rows, zero U
                CUDA_OK(cudaMemcpyAsync(tw.p, init, sizeof init, cudaMemcpyHostToDevice, stream));
                mk::LookupFoldArgs t = f;
                t.first = (unsigned long long*)tw.p; t.failing_rows = t.first + 1; t.zero_u = t.first + 2;
                t.folds_out = fw ? tw.p + 4 : nullptr;   // 16-byte aligned: the kernels store folds in pairs of words
                if (mk::launch_fold_rows(t, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: lookup program too large for the interpreter", i);
                compare_jit(*kn, JIT_FOLD, &jit_lookup_check_used[i], {{res.p + 3 * i, tw.p, 3}, {f.folds_out, t.folds_out, fw}});
            }
        } else if (mk::launch_fold_rows(f, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: lookup program too large for the interpreter", i);
        if (user && !on_device) {
            CUDA_OK(cudaMemcpyAsync(user, staging.p, (((size_t)4 * f.n_cols) << f.log_n) * sizeof(u64), cudaMemcpyDeviceToHost, stream));
            CUDA_OK(cudaStreamSynchronize(stream));   // the staging buffer serves the next AIR
            f.folds_out = nullptr;
        }
    }
    CUDA_OK(cudaMemcpyAsync(host_res.data(), res.p, 3 * (size_t)k * sizeof(u64), cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaGetLastError());

    memset(out, 0, sizeof *out);
    out->n_skipped_airs = fs.skipped;
    for (u32 i = 0; i < k; i++) { out->failing_rows += host_res[3 * i + 1]; out->zero_u += host_res[3 * i + 2]; }
    for (u32 i = 0; i < k; i++) {
        u64 first = host_res[3 * i];
        if (!airs[i].has_lookup || first == ~0ull) continue;
        out->instance = i; out->row = first >> 32; out->column = (u32)first;
        // the values: the same kernel on that one row, recording that column (its own atomics go to scratch words)
        mk::LookupFoldArgs f = fa[i];
        u64* probe = res.p + 3 * (size_t)k;
        f.folds_out = nullptr; f.row0 = out->row; f.n_rows = 1; f.probe_col = out->column; f.probe = probe;
        f.first = (unsigned long long*)(probe + 9); f.failing_rows = f.first + 1; f.zero_u = f.first + 2;
        if (mk::launch_fold_rows(f, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: lookup program too large for the interpreter", i);
        u64 pv[9];
        CUDA_OK(cudaMemcpyAsync(pv, probe, sizeof pv, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        out->kind = (u32)pv[0];
        memcpy(out->fold, pv + 1, 4 * sizeof(u64)); memcpy(out->expected, pv + 5, 2 * sizeof(u64)); memcpy(out->actual, pv + 7, 2 * sizeof(u64));
        break;
    }
    out->holds = out->failing_rows == 0;
}

// ---------------------------------------------------------------------------------------------
// lookup_fold_census: every disagreement of check_lookup_folds, per column and in row order, without a proof
// ---------------------------------------------------------------------------------------------
// prepare_folds as check_lookup_folds; then per lookup AIR (instance order) k_fold_census_rows fills that AIR's slice of
// one per-row count array, concatenated in instance order, and its per-column tally; one exclusive scan of the counts
// gives every disagreeing row its first record slot and the total.  k_fold_census_list then writes the first
// max_failures records in (instance, row, column) order, and in probe mode the records at the reported tallies' first
// rows (plus the least disagreement's, when truncation drops it).  Counts, minima, maxima and the scan do not depend on
// the order the atomics ran in, so neither does anything reported.
static_assert(sizeof(mdn_fold_failure) == mk::FOLD_RECORD_WORDS * sizeof(u64), "mdn_fold_failure is the kernel's record");
static_assert(sizeof(mdn_fold_tally) == 10 * sizeof(u64), "mdn_fold_tally: 80 bytes");
void mdn_session::lookup_fold_census(const mdn_statement* st, const mdn_matrix* traces, const u64* rnd, const uint32_t* const* fold_marks,
                                     const mdn_matrix* aux, const u64* const* aux_finals, u32 flags, mdn_fold_failure* failures, u64 max_failures,
                                     mdn_fold_tally* tallies, u64 max_tallies, mdn_fold_census_report* out) {
    FoldSetup fs;
    prepare_folds(st, traces, rnd, fold_marks, aux, aux_finals, nullptr, flags, out, fs);
    const u32 k = fs.k;

    // per-row counts of the lookup AIRs (u32, instance order), their offsets, one 4-word tally per column, two counters
    std::vector<size_t> row_base(k + 1, 0), tally_base(k + 1, 0);
    for (u32 i = 0; i < k; i++) {
        const bool lk = airs[i].has_lookup;
        row_base[i + 1] = row_base[i] + (lk ? (size_t)1 << log_heights[i] : 0);
        tally_base[i + 1] = tally_base[i] + (lk ? 4 * (size_t)airs[i].lookup_cols : 0);
    }
    const size_t rows = row_base[k];
    DevBuf counts, offsets, tally, words, scratch;
    counts.alloc(std::max<size_t>(1, (rows + 1) / 2), stream);
    offsets.alloc(std::max<size_t>(1, rows), stream);
    tally.alloc(std::max<size_t>(1, tally_base[k]), stream);
    words.alloc(2, stream);                                             // rows with a disagreement, disagreements
    scratch.alloc(std::max<size_t>(1, (rows + 2047) / 2048), stream);  // block sums of the scan
    std::vector<u64> host_tally(std::max<size_t>(1, tally_base[k]), 0);
    for (size_t q = 0; q < tally_base[k]; q += 4) host_tally[q + 2] = ~0ull;
    CUDA_OK(cudaMemcpyAsync(tally.p, host_tally.data(), host_tally.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
    CUDA_OK(cudaMemsetAsync(words.p, 0, 2 * sizeof(u64), stream));
    u32* d_counts = reinterpret_cast<u32*>(counts.p);
    u64 checked_rows = 0;   // rows with a disagreement of AIRs whose row pass was compared on first use (not in words[0])
    std::vector<mk::FoldCensusArgs> fa(k);
    for (u32 i = 0; i < k; i++) {
        if (!airs[i].has_lookup) continue;
        mk::FoldCensusArgs& f = fa[i];
        f = fold_args<mk::FoldCensusArgs>(i, fs);
        f.instance = i;
        f.row_count = d_counts + row_base[i];
        f.tally = (unsigned long long*)(tally.p + tally_base[i]);
        f.failing_rows = (unsigned long long*)words.p;
        f.offsets = offsets.p + row_base[i];
        jit::Kernel* kn = row_kernel(airs[i], JIT_FOLD_CENSUS);
        if (!kn) {
            if (mk::launch_fold_census_rows(f, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: lookup program too large for the interpreter", i);
            continue;
        }
        const size_t N = (size_t)1 << f.log_n, nt = 4 * (size_t)f.n_cols;
        jit::LookupCheckJitArgs ja = fold_jit_args(f);
        ja.row_count = f.row_count; ja.tally = f.tally;
        // first use of this kernel in the session: the kernel's failing rows go to a word of their own, and the
        // interpreter runs the same rows into its own counts, tally and word; all three must agree word for word
        const bool first_use = unchecked(*kn);
        DevBuf twin;
        if (first_use) {
            twin.alloc((N + 1) / 2 + nt + 2, stream);
            CUDA_OK(cudaMemcpyAsync(twin.p + (N + 1) / 2, host_tally.data() + tally_base[i], nt * sizeof(u64), cudaMemcpyHostToDevice, stream));
            CUDA_OK(cudaMemsetAsync(twin.p + (N + 1) / 2 + nt, 0, 2 * sizeof(u64), stream));
            ja.failing_rows = (unsigned long long*)(twin.p + (N + 1) / 2 + nt);
        }
        launch_jit(*kn, ja, N);
        jit_lookup_check_used[i] = 1;
        if (!first_use) continue;
        mk::FoldCensusArgs t = f;
        t.row_count = reinterpret_cast<u32*>(twin.p); t.tally = (unsigned long long*)(twin.p + (N + 1) / 2);
        t.failing_rows = (unsigned long long*)(twin.p + (N + 1) / 2 + nt + 1);
        if (mk::launch_fold_census_rows(t, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: lookup program too large for the interpreter", i);
        std::vector<u32> cnt_j(N), cnt_i(N);
        std::vector<u64> tw(nt + 2), tj(nt);
        CUDA_OK(cudaMemcpyAsync(cnt_j.data(), f.row_count, N * sizeof(u32), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaMemcpyAsync(cnt_i.data(), twin.p, N * sizeof(u32), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaMemcpyAsync(tj.data(), f.tally, nt * sizeof(u64), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaMemcpyAsync(tw.data(), twin.p + (N + 1) / 2, (nt + 2) * sizeof(u64), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        CUDA_OK(cudaGetLastError());
        const bool differs = cnt_j != cnt_i || !std::equal(tj.begin(), tj.end(), tw.begin()) || tw[nt] != tw[nt + 1];
        if (settle_jit(*kn, JIT_FOLD_CENSUS, differs, &jit_lookup_check_used[i])) {   // the interpreter's counts and tally stand
            CUDA_OK(cudaMemcpyAsync(f.row_count, twin.p, N * sizeof(u32), cudaMemcpyDeviceToDevice, stream));
            CUDA_OK(cudaMemcpyAsync(f.tally, twin.p + (N + 1) / 2, nt * sizeof(u64), cudaMemcpyDeviceToDevice, stream));
        }
        checked_rows += tw[nt + 1];
    }
    if (rows) mk::launch_count_exclusive_scan(d_counts, rows, offsets.p, words.p + 1, scratch.p, stream);
    u64 host_words[2];
    CUDA_OK(cudaMemcpyAsync(host_tally.data(), tally.p, host_tally.size() * sizeof(u64), cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaMemcpyAsync(host_words, words.p, sizeof host_words, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaGetLastError());
    host_words[0] += checked_rows;

    // the disagreeing (instance, column) pairs in order, and the least disagreement: the first failing instance's least
    // (first_row, column)
    std::vector<mdn_fold_tally> all;
    size_t least = SIZE_MAX;
    u64 zero_u = 0;
    for (u32 i = 0; i < k; i++) {
        if (!airs[i].has_lookup) continue;
        for (u32 c = 0; c < airs[i].lookup_cols; c++) {
            const u64* t = host_tally.data() + tally_base[i] + 4 * (size_t)c;
            if (!t[0]) continue;
            mdn_fold_tally ft{};
            ft.instance = i; ft.column = c; ft.failing_rows = t[0]; ft.zero_u_rows = t[1]; ft.first_row = t[2]; ft.last_row = t[3];
            all.push_back(ft);
            zero_u += t[1];
            if (least == SIZE_MAX || (all[least].instance == i && t[2] < all[least].first_row)) least = all.size() - 1;
        }
    }
    memset(out, 0, sizeof *out);
    out->disagreements = host_words[1];
    out->n_failures = std::min<u64>(out->disagreements, max_failures);
    out->failing_columns = all.size();
    out->n_tallies = std::min<u64>(all.size(), max_tallies);

    // records at the first rows of the reported tallies and of the least disagreement: probe mode, one launch per instance
    const size_t W = mk::FOLD_RECORD_WORDS;
    std::vector<size_t> probed;
    for (size_t q = 0; q < out->n_tallies; q++) probed.push_back(q);
    if (least != SIZE_MAX && least >= out->n_tallies) probed.push_back(least);   // `all` is in instance order: still sorted
    DevBuf d_probes, d_records, d_failures;
    if (!probed.empty()) {
        std::vector<u64> pr;
        for (size_t q : probed) { pr.push_back(all[q].first_row); pr.push_back(all[q].column); }
        d_probes.alloc(pr.size(), stream);
        d_records.alloc(W * probed.size(), stream);
        CUDA_OK(cudaMemcpyAsync(d_probes.p, pr.data(), pr.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
        for (size_t b = 0; b < probed.size();) {
            u32 i = all[probed[b]].instance;
            size_t e = b;
            while (e < probed.size() && all[probed[e]].instance == i) e++;
            mk::FoldCensusArgs f = fa[i];
            f.probes = d_probes.p + 2 * b; f.n_probes = e - b; f.failures = d_records.p + W * b;
            if (mk::launch_fold_census_list(f, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: lookup program too large for the interpreter", i);
            b = e;
        }
    }
    // the first n_failures records, every AIR with a disagreeing column writing its own slots
    if (out->n_failures) {
        alloc_checked("the list of " + std::to_string(out->n_failures) + " disagreements needs", {{&d_failures, W * out->n_failures}});
        for (u32 i = 0; i < k; i++) {
            if (!airs[i].has_lookup) continue;
            bool any = false;
            for (u32 c = 0; c < airs[i].lookup_cols && !any; c++) any = host_tally[tally_base[i] + 4 * (size_t)c] != 0;
            if (!any) continue;
            mk::FoldCensusArgs f = fa[i];
            f.max_failures = out->n_failures; f.failures = d_failures.p;
            if (mk::launch_fold_census_list(f, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "AIR %u: lookup program too large for the interpreter", i);
        }
    }
    std::vector<mdn_fold_failure> records(probed.size());
    if (!probed.empty()) CUDA_OK(cudaMemcpyAsync(records.data(), d_records.p, records.size() * sizeof(mdn_fold_failure), cudaMemcpyDeviceToHost, stream));
    if (out->n_failures) CUDA_OK(cudaMemcpyAsync(failures, d_failures.p, out->n_failures * sizeof(mdn_fold_failure), cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaGetLastError());
    for (size_t q = 0; q < probed.size(); q++) {
        mdn_fold_tally& t = all[probed[q]];
        t.first_kind = records[q].kind;
        memcpy(t.first_expected, records[q].expected, sizeof t.first_expected); memcpy(t.first_actual, records[q].actual, sizeof t.first_actual);
    }
    for (size_t q = 0; q < out->n_tallies; q++) tallies[q] = all[q];

    // `first`: what check_lookup_folds reports for the same call
    mdn_fold_report& f = out->first;
    f.n_skipped_airs = fs.skipped;
    f.failing_rows = host_words[0];
    f.zero_u = zero_u;
    if (least != SIZE_MAX) {
        const size_t q = std::find(probed.begin(), probed.end(), least) - probed.begin();
        const mdn_fold_failure& r = records[q];
        f.kind = r.kind; f.instance = r.instance; f.column = r.column; f.row = r.row;
        memcpy(f.fold, r.fold, sizeof f.fold); memcpy(f.expected, r.expected, sizeof f.expected); memcpy(f.actual, r.actual, sizeof f.actual);
    }
    f.holds = f.failing_rows == 0;
}

// mdn_aux_builder_device for instance `inst`: the aux columns go straight into `aux_slot` (column-major, on the session's
// stream), the aux values into `values`
void mdn_session::call_device_aux_builder(u32 inst, const mdn_matrix& main, u64* aux_slot, std::vector<u64>& values) {
    const mdn_air& a = airs[inst].desc;
    values.assign(2 * (size_t)a.num_aux_values + 1, 0);
    std::vector<u64> r;
    for (u32 q = 0; q < a.num_randomness; q++) { r.push_back(randomness[q].a); r.push_back(randomness[q].b); }
    r.push_back(0);
    if (dev_aux(dev_aux_ctx, inst, &main, r.data(), a.aux_width ? aux_slot : nullptr, values.data(), (void*)stream) != 0)
        fail(MDN_ERR_AUX_BUILDER, "device aux builder failed for instance %u", inst);
}

// aux traces (instance order, EF flattened to base), aux values; commit + observe (mod.rs:397-422).  In a column-major
// proof `aux` holds device matrices; `builder_main` (the proof's main traces) calls the device aux builder instead,
// which writes every slot in place, so the ingest only checks them.
void mdn_session::commit_aux(const mdn_matrix* aux, const u64* const* aux_values, bool zero_aux, const mdn_matrix* builder_main) {
    if (!in_proof) fail(MDN_ERR_INVALID_ARG, "commit_aux called outside a proof");
    u32 k = (u32)airs.size(), lb = params.log_blowup;
    CUDA_OK(cudaEventRecord(ev[3], stream));
    size_t coef_total = 0, lde_total = 0;
    for (u32 j = 0; j < k; j++) {
        u32 inst = order[j];
        size_t N = (size_t)1 << log_heights[inst];
        u32 w = 2 * airs[inst].desc.aux_width;
        coef_total += N * w; lde_total += (N << lb) * w;
    }
    aux_c.coef_buf.alloc(coef_total, stream);
    aux_c.lde_buf.alloc(lde_total, stream);
    upload_leaves((const u64*)randomness.data(), 2 * randomness.size());
    size_t co = 0, lo = 0;
    std::vector<u32> pos(k);
    for (u32 j = 0; j < k; j++) {
        u32 inst = order[j];
        size_t N = (size_t)1 << log_heights[inst];
        u32 w = 2 * airs[inst].desc.aux_width;
        aux_c.mats.push_back(CommittedMat{aux_c.lde_buf.p + lo, aux_c.coef_buf.p + co, log_heights[inst], w});
        pos[inst] = j;
        co += N * w; lo += (N << lb) * w;
    }
    // the device aux builder, instance order, for the AIRs without a lowered LookupAir
    std::vector<mdn_matrix> built;
    std::vector<std::vector<u64>> built_values;
    std::vector<const u64*> built_ptrs;
    if (builder_main) {
        built.resize(k); built_values.resize(k); built_ptrs.assign(k, nullptr);
        for (u32 i = 0; i < k; i++) {
            if (airs[i].has_lookup) continue;
            CommittedMat& m = aux_c.mats[pos[i]];
            call_device_aux_builder(i, builder_main[i], m.coef, built_values[i]);
            built[i] = mdn_matrix{m.coef, m.log_n, m.width};
            built_ptrs[i] = built_values[i].data();
        }
        aux = built.data(); aux_values = built_ptrs.data(); zero_aux = false;
    }
    std::vector<u64> flat_values;
    aux_values_p.assign(k, {}); aux_values_off.assign(k, 0);
    for (u32 j = 0; j < k; j++) {
        u32 inst = order[j];
        u32 w = 2 * airs[inst].desc.aux_width;
        CommittedMat& m = aux_c.mats[j];
        u64 logup_final[2] = {0, 0};
        const bool dev_aux = airs[inst].has_lookup;
        if (dev_aux) build_logup_aux(j, airs[inst].raw_main_cm, airs[inst].lookup_prep || airs[inst].reg_prep ? bundle_prep_rows(inst) : nullptr, m.coef, logup_final);
        else if (w) {
            if (zero_aux) CUDA_OK(cudaMemsetAsync(m.coef, 0, ((size_t)1 << m.log_n) * w * sizeof(u64), stream));
            else {
                if (!aux[inst].values) fail(MDN_ERR_INVALID_ARG, "aux trace %u is NULL", inst);
                if (aux[inst].width != w || aux[inst].log_height != log_heights[inst]) fail(MDN_ERR_INVALID_ARG, "aux trace %u has the wrong shape", inst);
                if (col_major && !builder_main) check_column_major(aux[inst], "aux trace", inst);
                upload_matrix(aux[inst], col_major, m.coef, col_major);   // a builder's slot: check only
            }
        }
        u32 nav = airs[inst].desc.num_aux_values;
        aux_values_off[j] = flat_values.size();
        if (nav && !dev_aux && !zero_aux && (!aux_values || !aux_values[inst])) fail(MDN_ERR_INVALID_ARG, "aux values of instance %u are NULL", inst);
        for (u32 v = 0; v < 2 * nav; v++) {
            u64 x = dev_aux ? logup_final[v] : (zero_aux ? 0 : aux_values[inst][v]);
            if (x >= gl::P) fail(MDN_ERR_INVALID_ARG, "non-canonical aux value");
            aux_values_p[j].push_back(x); flat_values.push_back(x);
        }
    }
    if (!zero_aux) check_input_flag("an aux trace");
    // Statement::eval_external on the aux values in instance order -- including the finals of aux traces built on the
    // device -- before anything is committed (prover/mod.rs:383-395, ProverError::ExternalAssertionFailed)
    {
        u32 failed = 0;
        int rc = eval_external(&failed);
        if (rc > 0) fail(MDN_ERR_EXTERNAL_ASSERTION, "external assertion %u failed", failed);
        if (rc < 0) fail(MDN_ERR_EXTERNAL_ASSERTION, "eval_external reported a reduction error");
    }
    if (constraint_guard) guard_constraints(flat_values);
    for (AirHost& h : airs) { h.raw_main.release(); h.raw_prep.release(); }
    lde_and_commit(aux_c, nullptr, nullptr);
    tr.send_commitment(aux_c.root);
    memcpy(dbg_roots[1], aux_c.root, 32);
    for (auto& vs : aux_values_p) for (u64 v : vs) tr.send_field(v);
    d_aux_values.alloc(std::max<size_t>(1, flat_values.size()), stream);
    if (!flat_values.empty()) CUDA_OK(cudaMemcpyAsync(d_aux_values.p, flat_values.data(), flat_values.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaEventRecord(ev[4], stream));
}

// ---------------------------------------------------------------------------------------------
// finish: constraints, quotient commit, OOD point, PCS opening  (mod.rs:424-577)
// ---------------------------------------------------------------------------------------------
void mdn_session::finish() {
    if (!in_proof) fail(MDN_ERR_INVALID_ARG, "finish called outside a proof");
    u32 k = (u32)airs.size(), lb = params.log_blowup, B = 1u << lb;
    u32 log_lde = log_max_n + lb;
    size_t Nmax = (size_t)1 << log_max_n, L = Nmax << lb;
    // 3. alpha, beta (mod.rs:425-426)
    E2 alpha = tr.ch.sample_ext(), beta = tr.ch.sample_ext();
    // 4. constraint evaluation + beta accumulation, ascending height (mod.rs:445-537)
    DevBuf acc_pp[2];
    std::vector<DevBuf> jit_apow;   // alive until the constraint kernels have run
    jit_used.clear();
    int acc_cur = -1;
    u32 acc_prev_log = 0;
    for (u32 j = 0; j < k; j++) {
        u32 inst = order[j];
        AirHost& air = airs[inst];
        u32 ln = log_heights[inst];
        int nxt = acc_cur < 0 ? 0 : 1 - acc_cur;
        acc_pp[nxt].alloc((size_t)2 << (ln + lb), stream);
        mk::ConstraintArgs ca;
        ca.main_lde = main_c.mats[j].lde; ca.main_width = main_c.mats[j].width;
        ca.aux_lde = aux_c.mats[j].lde; ca.aux_width_base = aux_c.mats[j].width;
        ca.prep_lde = nullptr;   // same height and coset as the main trace (mod.rs:463-476)
        if (has_prep) for (size_t q = 0; q < prep_air.size(); q++) if (prep_air[q] == inst) ca.prep_lde = prep_c.mats[q].lde;
        ca.log_n = ln; ca.log_blowup = lb; ca.air = air.dev;
        ca.publics = d_publics.p; ca.challenges = d_randomness.p; ca.aux_values = d_aux_values.p + aux_values_off[j];
        ca.alpha = alpha; ca.beta = beta;
        ca.acc_in = acc_cur < 0 ? nullptr : acc_pp[acc_cur].p; ca.acc_in_log_n = acc_prev_log; ca.acc_out = acc_pp[nxt].p;
        ca.T = &ntt(ln).T;
        ca.t0 = t0(); ca.nt = nt();            // this rank's cosets (all of them on one GPU)
        ProfScope ps(prof, PC_CONSTRAINTS);
        jit::Kernel* kn = row_kernel(air, JIT_PROOF);
        jit_used.push_back(kn ? 1 : 0);
        if (kn) {
            // alpha^(K-1-k) for the K constraints in emission order
            u32 K = air.n_constraints;
            std::vector<E2> apow(std::max(1u, K));
            { E2 x = gl::e2(1, 0); for (u32 q = K; q-- > 0;) { apow[q] = x; x = gl::e2_mul(x, alpha); } }
            jit_apow.emplace_back(); jit_apow.back().alloc(2 * (size_t)std::max(1u, K), stream);
            CUDA_OK(cudaMemcpyAsync(jit_apow.back().p, apow.data(), apow.size() * sizeof(E2), cudaMemcpyHostToDevice, stream));
            CUDA_OK(cudaStreamSynchronize(stream));   // apow is a stack vector
            jit::JitArgs ja{};
            ja.main_lde = ca.main_lde; ja.aux_lde = ca.aux_lde; ja.prep_lde = ca.prep_lde;
            ja.publics = ca.publics; ja.challenges = ca.challenges; ja.aux_values = ca.aux_values;
            ja.periodic = air.dev.periodic; ja.apow = jit_apow.back().p;
            ja.acc_in = ca.acc_in; ja.acc_out = ca.acc_out; ja.w_hi = ca.T->w_hi; ja.w_lo = ca.T->w_lo;
            ja.shift = gl::lde_shift(ln + lb); ja.w_l = gl::two_adic_generator(ln + lb); ja.w_h_inv = gl::inv(gl::two_adic_generator(ln));
            { u64 s_pow_n = gl::exp_pow2(ja.shift, ln), w_b = gl::two_adic_generator(lb), x = 1;   // Z_H on coset t (domain.rs:742-749)
              for (u32 t = 0; t < B; t++) { ja.zh[t] = gl::sub(gl::mul(s_pow_n, x), 1); ja.inv_zh[t] = gl::inv(ja.zh[t]); x = gl::mul(x, w_b); } }
            ja.beta_a = beta.a; ja.beta_b = beta.b;
            ja.log_n = ln; ja.log_b = lb; ja.acc_in_log_n = ca.acc_in_log_n; ja.lo_bits = ca.T->lo_bits; ja.log_max_period = air.dev.log_max_period;
            size_t Lj = (size_t)1 << (ln + lb), own = (size_t)ca.nt << ln;
            ja.pad = ca.t0 | (ca.nt << 8);
            launch_jit(*kn, ja, own);
            if (unchecked(*kn)) {
                // the interpreter evaluates the same points: those of this rank's cosets are compared, on every rank
                // alike (the ranks' allocation sequences have to stay identical).  The other cosets of both
                // accumulators are never read: the next AIR and the quotient read this rank's cosets only.
                DevBuf chk; chk.alloc(2 * Lj, stream);
                mk::ConstraintArgs cb = ca; cb.acc_out = chk.p;
                if (mk::launch_constraints(cb, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "constraint program too large for the interpreter");
                const size_t o = (size_t)ca.t0 << ln;
                compare_jit(*kn, JIT_PROOF, &jit_used.back(), {{ca.acc_out + o, chk.p + o, own}, {ca.acc_out + Lj + o, chk.p + Lj + o, own}}, true);
            }
        } else if (mk::launch_constraints(ca, stream) != 0) fail(MDN_ERR_UNSUPPORTED, "constraint program too large for the interpreter");
        acc_cur = nxt; acc_prev_log = ln;
    }
    DevBuf acc = std::move(acc_pp[acc_cur]);
    acc_pp[1 - acc_cur].release();
    CUDA_OK(cudaEventRecord(ev[5], stream));
    const u32 tb = t0(), tn = nt();
    if (keep_debug) {
        if (sharded()) {   // debug export only: collect every rank's cosets of the accumulator
            shard_barrier();
            for (u32 coord = 0; coord < 2; coord++) { u64* own = acc.p + (size_t)coord * L + (size_t)tb * Nmax; mk::launch_push(own, peers_of(own), shard_rank, shard_world, (size_t)tn * Nmax, stream); }
            shard_barrier();
        }
        // natural order on gJ: index r*B + t  <- planes [coord][t*N + r]
        std::vector<u64> planes(2 * L);
        CUDA_OK(cudaMemcpyAsync(planes.data(), acc.p, 2 * L * sizeof(u64), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        // natural order on gJ_max (N*D points): index r*D + t  <- coset t*(B/D) of the planes
        u32 Dq = 1u << log_qd, cs = B >> log_qd;
        dbg_quot_acc.assign(2 * Nmax * Dq, 0);
        for (size_t t = 0; t < Dq; t++)
            for (size_t r = 0; r < Nmax; r++) {
                dbg_quot_acc[2 * (r * Dq + t)] = planes[t * cs * Nmax + r];
                dbg_quot_acc[2 * (r * Dq + t) + 1] = planes[L + t * cs * Nmax + r];
            }
    }
    // 5. quotient commit (quotient.rs:143-217).  The accumulator was evaluated on all B cosets of gK
    //    (for a satisfied AIR that equals the reference's evaluate-on-gJ-then-upsample, quotient.rs:45-56,
    //    because C/Z_H is then a polynomial of degree < N*D); chunk t < D is the LDE coset t*(B/D).
    //    The committed matrix has column 2t + coord.
    //    Split over ranks: chunk t lives on the rank that owns coset t*(B/D); that rank interpolates it and stores
    //    the coefficients into every rank (the all-gather of chunk coefficients of SURVEY 8(e), as peer stores),
    //    then every rank evaluates all chunks on its own cosets.
    const u32 D = 1u << log_qd, cstep = B >> log_qd;
    {
        NttPlan& plan = ntt(log_max_n);
        PremulPlan& pm = premul_quotient(log_max_n, log_qd);
        size_t rq = prof.begin(PC_NTT);
        ntt_bytes += (double)(Nmax + L) * 2 * D * 8.0 / (sharded() ? shard_world : 1);
        // own chunks: c with c*cstep in [tb, tb + tn)
        u32 c_lo = (tb + cstep - 1) / cstep, c_hi = std::min(D, (tb + tn + cstep - 1) / cstep);
        if (c_hi > c_lo)
            for (u32 coord = 0; coord < 2; coord++)
                mk::launch_intt(acc.p + (size_t)coord * L + (size_t)c_lo * cstep * Nmax, (size_t)cstep * Nmax, c_hi - c_lo, plan.T, stream);
        if (sharded()) {
            shard_barrier();   // every rank is done writing / reading its accumulator planes
            for (u32 c = c_lo; c < c_hi; c++)
                for (u32 coord = 0; coord < 2; coord++) {
                    u64* chunk = acc.p + (size_t)coord * L + (size_t)c * cstep * Nmax;
                    mk::launch_push(chunk, peers_of(chunk), shard_rank, shard_world, Nmax, stream);
                }
            shard_barrier();
        }
        quot_c.lde_buf.alloc(L * 2 * D, stream);
        quot_c.coef_buf = std::move(acc);
        quot_c.mats.push_back(CommittedMat{quot_c.lde_buf.p, quot_c.coef_buf.p, log_max_n, 2 * D});
        std::vector<mk::FwdItem> items;
        for (u32 t = 0; t < D; t++)
            for (u32 coord = 0; coord < 2; coord++)
                for (u32 t2 = tb; t2 < tb + tn; t2++)
                    items.push_back(mk::FwdItem{quot_c.coef_buf.p + (size_t)coord * L + (size_t)t * cstep * Nmax,
                                                quot_c.lde_buf.p + (size_t)(2 * t + coord) * L + (size_t)t2 * Nmax, t * B + t2, 0});
        DevBuf d_items; d_items.alloc(items.size() * sizeof(mk::FwdItem) / sizeof(u64), stream);
        CUDA_OK(cudaMemcpyAsync(d_items.p, items.data(), items.size() * sizeof(mk::FwdItem), cudaMemcpyHostToDevice, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        // groups of whole chunks keep the working set near L2 size
        u32 per = 2 * tn;   // items per chunk t
        u32 chunks_per_launch = std::max(1u, B / tn);
        for (u32 t = 0; t < D; t += chunks_per_launch) {
            u32 cn = std::min(chunks_per_launch, D - t);
            mk::launch_fwd_ntt((const mk::FwdItem*)d_items.p + (size_t)t * per, cn * per, plan.T, pm.P, stream);
        }
        prof.end(rq);
        build_tree(quot_c);
        tr.send_commitment(quot_c.root);
        memcpy(dbg_roots[2], quot_c.root, 32);
    }
    CUDA_OK(cudaEventRecord(ev[6], stream));
    // 6. OOD point: resample while z = 0, z in H, or z in gK  (domain.rs:539-552)
    u64 shift = gl::lde_shift(log_lde), shift_inv = gl::inv(shift);
    E2 z;
    for (;;) {
        z = tr.ch.sample_ext();
        if (z.a == 0 && z.b == 0) continue;
        if (gl::e2_eq(gl::e2_exp_pow2(z, log_max_n), gl::e2(1, 0))) continue;
        if (gl::e2_eq(gl::e2_exp_pow2(gl::e2_mulf(z, shift_inv), log_lde), gl::e2(1, 0))) continue;
        break;
    }
    ood_z = z;
    u64 omega_h = gl::two_adic_generator(log_max_n);
    E2 z_next = gl::e2_mulf(z, omega_h);

    // 7. PCS opening (pcs/prover.rs:34-102)
    // 7a. OOD evaluations of every committed column at z^(r_m), (z*w_H)^(r_m)
    //     (deep/interpolate.rs:127-203; computed here from the coefficient columns)
    // group order [preprocessed?, main, aux, quotient] (mod.rs:551-559)
    std::vector<Committed*> groups;
    if (has_prep) groups.push_back(&prep_c);
    groups.push_back(&main_c); groups.push_back(&aux_c); groups.push_back(&quot_c);
    const int ng = (int)groups.size(), gq = ng - 1;
    struct MatEval { std::vector<u64> v; };   // width x 4
    std::vector<std::vector<MatEval>> evals(ng);
    {
        // Split over ranks: a column's dot product with the weight vector is a sum over coefficient slots, so rank g
        // takes slots [g*N/G, (g+1)*N/G) of every (tall enough) column -- it builds only that slice of each weight
        // vector -- and the G partial sums per column meet in every rank's buffer (peer stores) and are added on the host.
        size_t ood_region = prof.begin(PC_OOD);
        // all dot products are queued first and fetched with ONE device->host copy
        size_t total_cols = 0;
        for (int g = 0; g < ng; g++) for (auto& cm : groups[g]->mats) total_cols += cm.width;
        const size_t T = std::max<size_t>(1, total_cols * 4);
        const u32 G = sharded() ? shard_world : 1, me = sharded() ? shard_rank : 0, lg = sharded() ? shard_log_g : 0;
        DevBuf d_all; d_all.alloc(T * G, stream);
        u64* d_out = d_all.p + (size_t)me * T;
        auto sliced = [&](u32 ln) { return G > 1 && ln >= lg + shard_min_log; };
        std::vector<DevBuf> keep;                              // weight vectors / partial sums stay alive until the copy
        std::map<u32, std::pair<u64*, u64*>> weights;          // per log height: (w0, w1), this rank's slice
        auto make_w = [&](u32 ln, E2 y0, E2 y1) {
            size_t S = sliced(ln) ? ((size_t)1 << (ln - lg)) : ((size_t)1 << ln), p0 = sliced(ln) ? S * me : 0;
            keep.emplace_back(); keep.back().alloc(2 * S, stream); u64* a = keep.back().p;
            keep.emplace_back(); keep.back().alloc(2 * S, stream); u64* b = keep.back().p;
            size_t tw = 2 * (((size_t)1 << (ln - ln / 2)) + ((size_t)1 << (ln / 2)));
            keep.emplace_back(); keep.back().alloc(2 * tw, stream); u64* sc = keep.back().p;
            mk::launch_pow_bitrev(y0, ln, a, sc, p0, S, stream);
            mk::launch_pow_bitrev(y1, ln, b, sc + tw, p0, S, stream);
            return std::make_pair(a, b);
        };
        size_t col_off = 0;
        struct Scale { size_t off; u64 n_inv; bool sliced; };
        std::vector<Scale> scale;                              // (first u64 index, 1/N, summed over ranks?) per matrix
        for (int g = 0; g < ng; g++) {
            evals[g].resize(groups[g]->mats.size());
            for (size_t m = 0; m < groups[g]->mats.size(); m++) {
                CommittedMat& cm = groups[g]->mats[m];
                evals[g][m].v.assign((size_t)cm.width * 4, 0);
                if (!cm.width) continue;
                u32 ln = cm.log_n, lr = log_max_n - ln;
                size_t Nm = (size_t)1 << ln;
                const bool sl = sliced(ln);
                const u32 ls = sl ? ln - lg : ln;                      // log of the slice this rank sums over
                const size_t S = (size_t)1 << ls, s0 = sl ? S * me : 0;
                u32 n_chunks = (u32)std::max<size_t>(1, std::min<size_t>(S / 4096, 256));   // k_ood_reduce walks the chunks serially
                if (g != gq) {
                    auto it = weights.find(ln);
                    if (it == weights.end()) it = weights.emplace(ln, make_w(ln, gl::e2_exp_pow2(z, lr), gl::e2_exp_pow2(z_next, lr))).first;
                    keep.emplace_back(); keep.back().alloc((size_t)cm.width * n_chunks * 4, stream);
                    mk::launch_ood_dot(cm.coef + s0, Nm, cm.width, ls, it->second.first, it->second.second, keep.back().p, n_chunks, stream);
                    mk::launch_ood_reduce(keep.back().p, cm.width, n_chunks, d_out + col_off * 4, stream);
                } else {
                    // quotient chunk t: stored coefficients are a_k * (g*w_J^t)^k (planes coord, column t*(B/D)),
                    // so q_t(y) is their evaluation at y / (g * w_J^t); outputs land at columns 2t, 2t+1.
                    u64 wj_inv = gl::inv(gl::two_adic_generator(log_max_n + log_qd));
                    for (u32 t = 0; t < D; t++) {
                        u64 f = gl::mul(shift_inv, gl::pow(wj_inv, t));
                        auto wv = make_w(ln, gl::e2_mulf(z, f), gl::e2_mulf(z_next, f));
                        keep.emplace_back(); keep.back().alloc((size_t)2 * n_chunks * 4, stream);
                        mk::launch_ood_dot(cm.coef + (size_t)t * cstep * Nm + s0, (size_t)B * Nm, 2, ls, wv.first, wv.second, keep.back().p, n_chunks, stream);
                        mk::launch_ood_reduce(keep.back().p, 2, n_chunks, d_out + (col_off + 2 * t) * 4, stream);
                    }
                }
                scale.push_back(Scale{col_off * 4, gl::inv((u64)Nm), sl});   // launch_intt leaves coefficients scaled by N
                col_off += cm.width;
            }
        }
        prof.end(ood_region);
        if (G > 1) {
            shard_barrier();                                   // d_all is a fresh allocation on every rank
            mk::launch_push(d_out, peers_of(d_out), shard_rank, shard_world, T, stream);
            shard_barrier();
        }
        std::vector<u64> host(T * G);
        CUDA_OK(cudaMemcpyAsync(host.data(), d_all.p, host.size() * sizeof(u64), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        size_t si = 0;
        for (int g = 0; g < ng; g++)
            for (size_t m = 0; m < groups[g]->mats.size(); m++) {
                CommittedMat& cm = groups[g]->mats[m];
                if (!cm.width) continue;
                const Scale& sc = scale[si++];
                for (size_t q = 0; q < (size_t)cm.width * 4; q++) {
                    u64 v = host[(size_t)me * T + sc.off + q];
                    if (sc.sliced) { v = 0; for (u32 r = 0; r < G; r++) v = gl::add(v, host[(size_t)r * T + sc.off + q]); }
                    evals[g][m].v[q] = gl::mul(v, sc.n_inv);
                }
            }
    }
    // aligned flat evaluation lists per point (deep/prover.rs:150-154)
    std::vector<E2> flat[2];
    std::vector<u32> aligned_off;   // per (group, matrix): offset in the aligned index space
    u32 W = 0;
    for (int g = 0; g < ng; g++)
        for (size_t m = 0; m < groups[g]->mats.size(); m++) {
            u32 w = groups[g]->mats[m].width, aw = (w + align() - 1) / align() * align();   // Lmcs alignment: 8 for the sponge, 1 for the chaining hasher
            aligned_off.push_back(W);
            for (int p = 0; p < 2; p++) {
                for (u32 c = 0; c < w; c++) {
                    flat[p].push_back(gl::e2(evals[g][m].v[4 * c + 2 * p], evals[g][m].v[4 * c + 2 * p + 1]));
                }
                for (u32 c = w; c < aw; c++) flat[p].push_back(gl::e2(0, 0));
            }
            W += aw;
        }
    for (int p = 0; p < 2; p++) for (const E2& e : flat[p]) tr.send_ext(e);
    // 7b. DEEP grind + challenges (deep/prover.rs:157-162)
    grind(params.deep_pow_bits);
    E2 dalpha = tr.ch.sample_ext(), dbeta = tr.ch.sample_ext();
    E2 fz[2];
    for (int p = 0; p < 2; p++) { E2 a = gl::e2(0, 0); for (const E2& e : flat[p]) a = gl::e2_add(gl::e2_mul(a, dalpha), e); fz[p] = a; }
    std::vector<E2> apow(W);
    { E2 a = gl::e2(1, 0); for (u32 i = W; i-- > 0;) { apow[i] = a; a = gl::e2_mul(a, dalpha); } }
    // 7c. DEEP quotient over the LDE domain (deep/prover.rs:214-312)
    DevBuf d_apow; d_apow.alloc(2 * (size_t)W, stream);
    CUDA_OK(cudaMemcpyAsync(d_apow.p, apow.data(), W * sizeof(E2), cudaMemcpyHostToDevice, stream));
    // FRI shape (fri/mod.rs:80-94) and which layers stay split by coset: layer r (domain 2^(log_lde - la*r)) is
    // produced rank-locally while fri_layer_sharded() holds; the first small layer is stored into every rank and
    // everything after it is replicated.  The debug export of the DEEP evaluations needs layer 0 everywhere.
    const u32 la = params.log_folding_arity;
    u32 rounds; size_t final_deg;
    {
        u32 target = params.log_final_degree + lb;
        u32 steps = log_lde > target ? log_lde - target : 0;
        rounds = (steps + la - 1) / la;
        u32 lf = log_lde > la * rounds ? log_lde - la * rounds : 0;
        final_deg = (size_t)1 << (lf > lb ? lf - lb : 0);
    }
    std::vector<char> layer_sh(rounds + 1, 0);
    for (u32 r = 0; r <= rounds && log_lde >= la * r; r++) {
        bool shd = fri_layer_sharded(log_lde - la * r) && r < rounds && !(r == 0 && keep_debug);
        layer_sh[r] = shd && (r == 0 || layer_sh[r - 1]);
        if (!layer_sh[r]) break;
    }
    std::vector<DevBuf> fri_layers;   // EF interleaved, natural domain order
    fri_layers.emplace_back(); fri_layers[0].alloc(2 * L, stream);
    {
        mk::DeepArgs da; da.n_mats = 0;
        std::vector<mk::DeepMat> all_mats;
        size_t mi = 0;
        for (int g = 0; g < ng; g++)
            for (size_t m = 0; m < groups[g]->mats.size(); m++, mi++) {
                CommittedMat& cm = groups[g]->mats[m];
                if (!cm.width) continue;
                all_mats.push_back(mk::DeepMat{cm.lde, cm.width, cm.log_n, aligned_off[mi], 0});
            }
        // descriptors travel through device memory, so the number of committed matrices is not limited
        DevBuf d_mats; d_mats.alloc(std::max<size_t>(1, all_mats.size() * sizeof(mk::DeepMat) / sizeof(u64)), stream);
        CUDA_OK(cudaMemcpyAsync(d_mats.p, all_mats.data(), all_mats.size() * sizeof(mk::DeepMat), cudaMemcpyHostToDevice, stream));
        CUDA_OK(cudaStreamSynchronize(stream));   // all_mats is a stack vector
        da.m = (const mk::DeepMat*)d_mats.p; da.n_mats = (int)all_mats.size();
        // NB: the quotient matrix's device columns are already in committed order (2t + coord).
        da.log_n_max = log_max_n; da.log_blowup = lb; da.apow = d_apow.p; da.total_w = W;
        da.z0 = z; da.z1 = z_next; da.fz0 = fz[0]; da.fz1 = fz[1]; da.beta = dbeta;
        da.out = push_dst(fri_layers[0].p, sharded() && !layer_sh[0] ? mk::PUSH_ALL : mk::PUSH_LOCAL);
        da.T = &ntt(log_max_n).T; da.t0 = tb; da.nt = tn;
        if (sharded() && !layer_sh[0]) shard_barrier();   // fresh target buffer on every rank
        { ProfScope ps(prof, PC_DEEP); mk::launch_deep(da, stream); }
        if (sharded() && !layer_sh[0]) shard_barrier();
    }
    CUDA_OK(cudaStreamSynchronize(stream));
    if (keep_debug) {
        // export in the reference's bit-reversed order
        std::vector<u64> nat(2 * L);
        CUDA_OK(cudaMemcpy(nat.data(), fri_layers[0].p, 2 * L * sizeof(u64), cudaMemcpyDeviceToHost));
        dbg_deep.assign(2 * L, 0);
        for (size_t i = 0; i < L; i++) {
            size_t br = gl::bitrev32((u32)i, log_lde);
            dbg_deep[2 * br] = nat[2 * i]; dbg_deep[2 * br + 1] = nat[2 * i + 1];
        }
    }
    // 7d. FRI commit phase (fri/prover.rs:93-242)
    std::vector<Tree> fri_trees(rounds);
    std::vector<char> fri_split(rounds, 0);
    dbg_fri_roots.clear();
    u32 log_dom = log_lde;
    for (u32 r = 0; r < rounds; r++) {
        if (log_dom < la) fail(MDN_ERR_INVALID_ARG, "FRI domain too small for the folding arity");
        size_t q = (size_t)1 << (log_dom - la);
        Tree& t = fri_trees[r];
        t.depth = log_dom - la;
        t.nodes.alloc((2 * q - 1) * 4, stream);
        const bool in_sh = layer_sh[r] != 0;                       // this rank holds its cosets' entries of layer r only
        const bool split = in_sh && tree_sharded(t.depth);         // sub-tree per rank, else a replicated tree
        fri_split[r] = split;
        const u32 ft0 = in_sh ? tb : 0, fnt = in_sh ? tn : B;
        mk::PushDst dig = push_dst(t.layer(t.depth), in_sh ? (split ? mk::PUSH_OWNER : mk::PUSH_ALL) : mk::PUSH_LOCAL, t.depth - (split ? shard_log_g : 0));
        if (in_sh) shard_barrier();
        {
            ProfScope ps(prof, PC_FRI);
            perms += (q * (la == 3 ? 2 : 1) + q - 1) / (in_sh ? shard_world : 1);
            if (hash_kind == MDN_HASH_BLAKE3) mk::launch_fri_leaf_hash_b3(fri_layers[r].p, q, la, dig, lb, ft0, fnt, stream);
            else if (hash_kind == MDN_HASH_KECCAK) mk::launch_fri_leaf_hash_kk(fri_layers[r].p, q, la, dig, lb, ft0, fnt, stream);
            else mk::launch_fri_leaf_hash(fri_layers[r].p, q, la, dig, lb, ft0, fnt, stream, perm());
        }
        if (in_sh) shard_barrier();
        if (!split) {
            ProfScope ps(prof, PC_FRI);
            compress_subtree(t, t.depth, 0, 0);
        } else {
            const u32 lg = shard_log_g;
            {
                ProfScope ps(prof, PC_FRI);
                compress_subtree(t, t.depth, lg, shard_rank);
            }
            u64* mine = t.layer(lg) + (size_t)shard_rank * 4;
            mk::launch_push(mine, peers_of(mine), shard_rank, shard_world, 4, stream);
            shard_barrier();
            ProfScope ps(prof, PC_FRI);
            compress_subtree(t, lg, 0, 0);
        }
        u64 root[4];
        CUDA_OK(cudaMemcpyAsync(root, t.layer(0), sizeof root, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        tr.send_commitment(root);
        dbg_fri_roots.insert(dbg_fri_roots.end(), root, root + 4);
        grind(params.folding_pow_bits);
        E2 fb = tr.ch.sample_ext();
        fri_layers.emplace_back(); fri_layers[r + 1].alloc(2 * q, stream);
        {
            const bool bcast = in_sh && !layer_sh[r + 1];          // the first replicated layer: stored into every rank
            mk::PushDst nxt = push_dst(fri_layers[r + 1].p, bcast ? mk::PUSH_ALL : mk::PUSH_LOCAL);
            if (bcast) shard_barrier();
            { ProfScope ps(prof, PC_FRI); mk::launch_fri_fold(fri_layers[r].p, log_dom, la, fb, nxt, lb, ft0, fnt, stream); }
            if (bcast) shard_barrier();
        }
        log_dom -= la;
    }
    shard_check_enqueue();        // evaluated after the synchronisation of the final-layer copy below
    // final polynomial (fri/prover.rs:228-239): values on the size-final_deg subgroup are the
    // final-layer entries at natural indices i*B; iDFT on the host, sent in descending order.
    {
        size_t dom = (size_t)1 << log_dom;
        std::vector<u64> lay(2 * dom);
        CUDA_OK(cudaMemcpyAsync(lay.data(), fri_layers[rounds].p, 2 * dom * sizeof(u64), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        shard_check_finish("FRI commit phase");
        size_t stride = dom / final_deg;
        u32 lf = 0; while (((size_t)1 << lf) < final_deg) lf++;
        u64 wi = gl::inv(gl::two_adic_generator(lf)), ninv = gl::inv((u64)final_deg);
        std::vector<E2> coeff(final_deg);
        for (size_t kk = 0; kk < final_deg; kk++) {
            u64 wk = gl::pow(wi, kk), x = 1;
            E2 a = gl::e2(0, 0);
            for (size_t i = 0; i < final_deg; i++) {
                E2 e = gl::e2(lay[2 * i * stride], lay[2 * i * stride + 1]);
                a = gl::e2_add(a, gl::e2_mulf(e, x));
                x = gl::mul(x, wk);
            }
            coeff[kk] = gl::e2_mulf(a, ninv);
        }
        for (size_t i = final_deg; i-- > 0;) tr.send_ext(coeff[i]);
    }
    // 7e. query grind + indices (pcs/prover.rs:73-84)
    grind(params.query_pow_bits);
    std::vector<size_t> qs;
    for (u32 i = 0; i < params.num_queries; i++) qs.push_back((size_t)tr.ch.sample_bits(log_lde));
    dbg_queries.assign(qs.begin(), qs.end());
    Indices ti = Indices::make(qs, log_lde);
    // 7f. openings: one pointer list, one gather (pcs/prover.rs:89-101; lifted_tree.rs:155-180).  Split over ranks,
    //     every opened word has an owner -- the rank holding that LDE coset / FRI coset / Merkle sub-tree -- which
    //     stores it into every rank's value buffer (-1: replicated data, read locally).
    std::vector<const u64*> ptrs;
    std::vector<int> owner;
    struct Emit { int kind; size_t count; size_t pad; };   // kind 0: `count` fields then `pad` zero fields; 1: commitment (4)
    std::vector<Emit> plan;
    for (int g = 0; g < ng; g++) {
        Committed& c = *groups[g];
        const bool replicated = (&c == &prep_c);   // the preprocessed bundle is committed once, whole, on every rank
        Indices leafs = ti.folded(c.tree.depth);
        for (size_t idx : leafs.idx)
            for (auto& cm : c.mats) {
                u32 ldm = cm.log_n + lb;
                size_t im = idx & (((size_t)1 << ldm) - 1);
                size_t t = im & (B - 1), rr = im >> lb;
                size_t pos = (t << cm.log_n) + rr, Lm = (size_t)1 << ldm;
                for (u32 col = 0; col < cm.width; col++) { ptrs.push_back(cm.lde + (size_t)col * Lm + pos); owner.push_back(replicated ? -1 : coset_owner((u32)t)); }
                plan.push_back(Emit{0, cm.width, (size_t)((cm.width + align() - 1) / align() * align() - cm.width)});
            }
        for (auto& ds : hostfs::missing_siblings(leafs)) {
            // split tree: a node below the sub-root level exists only on the rank owning its leaf range
            int own = -1;
            if (!replicated && tree_sharded(c.tree.depth) && ds.first > shard_log_g) own = (int)(ds.second >> (ds.first - shard_log_g));
            for (int q = 0; q < 4; q++) { ptrs.push_back(c.tree.layer(ds.first) + ds.second * 4 + q); owner.push_back(own); }
            plan.push_back(Emit{1, 4, 0});
        }
    }
    {
        Indices fi = ti;
        u32 ld = log_lde;
        for (u32 r = 0; r < rounds; r++) {
            fi = fi.folded(fi.depth > la ? fi.depth - la : 0);
            size_t q = (size_t)1 << (ld - la);
            const u64* lay = fri_layers[r].p;
            u32 a = 1u << la;
            for (size_t idx : fi.idx) {
                int own = layer_sh[r] ? coset_owner((u32)(idx & (B - 1))) : -1;    // the row's 2^la entries share idx's coset
                for (u32 e = 0; e < a; e++) {
                    size_t src = idx + (size_t)gl::bitrev32(e, la) * q;
                    ptrs.push_back(lay + 2 * src); ptrs.push_back(lay + 2 * src + 1);
                    owner.push_back(own); owner.push_back(own);
                }
                plan.push_back(Emit{0, 2 * (size_t)a, 0});
            }
            for (auto& ds : hostfs::missing_siblings(fi)) {
                int own = -1;
                if (fri_split[r] && ds.first > shard_log_g) own = (int)(ds.second >> (ds.first - shard_log_g));
                for (int qq = 0; qq < 4; qq++) { ptrs.push_back(fri_trees[r].layer(ds.first) + ds.second * 4 + qq); owner.push_back(own); }
                plan.push_back(Emit{1, 4, 0});
            }
            ld -= la;
        }
    }
    {
        DevBuf d_ptrs, d_vals, d_owner; d_ptrs.alloc(ptrs.size(), stream); d_vals.alloc(ptrs.size(), stream);
        CUDA_OK(cudaMemcpyAsync(d_ptrs.p, ptrs.data(), ptrs.size() * sizeof(u64), cudaMemcpyHostToDevice, stream));
        if (!sharded()) {
            ProfScope ps(prof, PC_GATHER); mk::launch_gather((const u64* const*)d_ptrs.p, d_vals.p, ptrs.size(), stream);
        } else {
            d_owner.alloc((owner.size() + 1) / 2, stream);
            CUDA_OK(cudaMemcpyAsync(d_owner.p, owner.data(), owner.size() * sizeof(int), cudaMemcpyHostToDevice, stream));
            shard_barrier();
            { ProfScope ps(prof, PC_GATHER); mk::launch_gather_push((const u64* const*)d_ptrs.p, (const int*)d_owner.p, peers_of(d_vals.p), shard_rank, shard_world, ptrs.size(), stream); }
            shard_barrier();
        }
        std::vector<u64> vals(ptrs.size());
        CUDA_OK(cudaMemcpyAsync(vals.data(), d_vals.p, vals.size() * sizeof(u64), cudaMemcpyDeviceToHost, stream));
        shard_check_enqueue();
        CUDA_OK(cudaStreamSynchronize(stream));
        shard_check_finish("query openings");
        size_t o = 0;
        for (auto& e : plan) {
            if (e.kind == 0) { for (size_t i = 0; i < e.count; i++) tr.hint_field(vals[o++]); for (size_t i = 0; i < e.pad; i++) tr.hint_field(0); }
            else { tr.hint_commitment(&vals[o]); o += 4; }
        }
    }
    CUDA_OK(cudaEventRecord(ev[7], stream));
    CUDA_OK(cudaEventSynchronize(ev[7]));
    // 8. StarkProofData (mod.rs:572-577)
    out_heights.clear();
    for (u32 h : log_heights) out_heights.push_back((uint8_t)h);
    out_fields = std::move(tr.fields);
    out_commitments = std::move(tr.commitments);
    cudaEventElapsedTime(&timings.h2d_transpose, ev[0], ev[1]);
    cudaEventElapsedTime(&timings.commit_main, ev[1], ev[2]);
    cudaEventElapsedTime(&timings.commit_aux, ev[3], ev[4]);
    cudaEventElapsedTime(&timings.evaluate_constraints, ev[4], ev[5]);
    cudaEventElapsedTime(&timings.commit_quotient, ev[5], ev[6]);
    cudaEventElapsedTime(&timings.open, ev[6], ev[7]);
    cudaEventElapsedTime(&timings.total, ev[0], ev[7]);
    timings.kernel_launches = mk::launch_count();
    prof.resolve(timings.kernel_ms, timings.kernel_regions);
    timings.leaf_hash_bytes = leaf_bytes; timings.ntt_bytes = ntt_bytes; timings.permutations = perms;
    in_proof = false; shard_active = false;   // the API wrapper returns the proof's device memory to the arena once this frame is gone
}

// =============================================================================================
// C ABI
// =============================================================================================
#define API_TRY(s) try {
#define API_CATCH(s) } catch (const MdnError& e) { (s)->error = e.what(); (s)->reset_proof(); return e.code; } \
    catch (const std::exception& e) { (s)->error = e.what(); (s)->reset_proof(); return MDN_ERR_INVALID_ARG; } return MDN_OK;

namespace {
// the challenges the call sampled, two words each, when the caller asks for them
void copy_randomness(const mdn_session* s, uint64_t* out) {
    if (out) for (size_t i = 0; i < s->randomness.size(); i++) { out[2 * i] = s->randomness[i].a; out[2 * i + 1] = s->randomness[i].b; }
}

const char IN_PROOF[] = " called inside a proof (between mdn_prove_begin and mdn_prove_finish)";

// A trace check (mdn_check_constraints and the others) named `name`: refused before any device work inside a staged
// proof, so that the proof stays intact, then on a session split over ranks, then with `refused` (the caller's own
// argument error, or NULL).  `check` runs in the proof arena, which is released afterwards; the challenges it sampled
// go to `randomness_out` when given.
template <class F> int run_check(mdn_session* s, const char* name, const char* refused, uint64_t* randomness_out, F check) {
    if (!s) return MDN_ERR_INVALID_ARG;
    if (s->in_proof) { s->error = name + std::string(IN_PROOF); return MDN_ERR_INVALID_ARG; }
    if (s->shard_world > 1) { s->error = name + std::string(" does not run on a session split over ranks (mdn_session_set_shard world > 1)"); return MDN_ERR_UNSUPPORTED; }
    if (refused) { s->error = refused; return MDN_ERR_INVALID_ARG; }
    API_TRY(s)
    {
        ArenaScope proof_memory(s->use_arena ? &s->arena : nullptr);
        CUDA_OK(cudaSetDevice(s->device));
        check();
        copy_randomness(s, randomness_out);
    }
    s->reset_proof();
    API_CATCH(s)
}
}  // namespace

extern "C" {

int mdn_session_create(const mdn_pcs_params* params, int cuda_device, mdn_session** out) {
    if (!params || !out) { g_create_error = "null argument"; return MDN_ERR_INVALID_ARG; }
    // PcsParams::new (pcs/params.rs:53-99), before any device is touched
    if (params->log_folding_arity < 1 || params->log_folding_arity > 3) { g_create_error = "invalid folding arity: log_arity " + std::to_string(params->log_folding_arity) + " (must be 1, 2, or 3)"; return MDN_ERR_INVALID_ARG; }
    if (params->log_blowup == 0) { g_create_error = "log_blowup must be at least 1"; return MDN_ERR_INVALID_ARG; }
    if (params->num_queries == 0) { g_create_error = "num_queries must be at least 1"; return MDN_ERR_INVALID_ARG; }
    if (params->log_final_degree + params->log_blowup < params->log_folding_arity - 1) {
        g_create_error = "log_final_degree " + std::to_string(params->log_final_degree) + " + log_blowup " + std::to_string(params->log_blowup) + " is below the minimum target " +
                         std::to_string(params->log_folding_arity - 1) + " reachable by fixed-arity folding";
        return MDN_ERR_INVALID_ARG;
    }
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        g_create_error = std::string("no usable CUDA device: ") + cudaGetErrorString(e) + " (this backend has no CPU fallback)";
        return MDN_ERR_NO_DEVICE;
    }
    if (cuda_device < 0 || cuda_device >= count) { g_create_error = "CUDA device index out of range"; return MDN_ERR_NO_DEVICE; }
    if (params->num_queries == 0 || params->log_blowup == 0) { g_create_error = "invalid PCS parameters"; return MDN_ERR_INVALID_ARG; }
    auto* s = new mdn_session();
    s->params = *params; s->device = cuda_device;
    try {
        CUDA_OK(cudaSetDevice(cuda_device));
        CUDA_OK(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
        CUDA_OK(cudaStreamCreateWithFlags(&s->copy_stream, cudaStreamNonBlocking));
        for (auto& evn : s->copy_ev) CUDA_OK(cudaEventCreateWithFlags(&evn, cudaEventDisableTiming));
        for (auto& evn : s->ev) CUDA_OK(cudaEventCreate(&evn));
        // the input and error flag word of the ingest, transpose and compare kernels; outside any proof arena
        s->d_flag.alloc(1, s->stream);
        CUDA_OK(cudaMemsetAsync(s->d_flag.p, 0, 8, s->stream));
        cudaMemPool_t pool;
        CUDA_OK(cudaDeviceGetDefaultMemPool(&pool, cuda_device));
        uint64_t thr = ~0ull;
        CUDA_OK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
        mk::upload_constants();
        CUDA_OK(cudaDeviceSynchronize());
    } catch (const std::exception& ex) { g_create_error = ex.what(); delete s; return MDN_ERR_CUDA; }
    *out = s;
    return MDN_OK;
}

void mdn_session_destroy(mdn_session* s) {
    if (!s) return;
    cudaSetDevice(s->device);
    // every stream-ordered allocation must be returned before the stream goes away
    s->reset_proof();
    s->allgather = nullptr;     // the peers may be gone already: unmap without a rendezvous
    s->shard_teardown();
    s->prep_c = Committed();
    s->d_publics.release(); s->d_randomness.release(); s->d_aux_values.release(); s->d_flag.release();
    s->ntt_plans.clear(); s->premul_plans.clear();
    for (auto& a : s->airs) a.jit = {};
    s->jit_kernels.clear();
    cudaStreamSynchronize(s->stream);
    s->arena.destroy();
    for (auto& evn : s->ev) cudaEventDestroy(evn);
    for (auto& evn : s->copy_ev) cudaEventDestroy(evn);
    for (int b = 0; b < 2; b++) if (s->bounce[b]) { cudaFreeHost(s->bounce[b]); cudaEventDestroy(s->bounce_ev[b]); }
    cudaStreamDestroy(s->copy_stream);
    cudaStreamDestroy(s->stream);
    delete s;
}

const char* mdn_last_error(const mdn_session* s) { return s ? s->error.c_str() : g_create_error.c_str(); }

static void fill_proof(mdn_session* s, mdn_proof* out) {
    out->log_trace_heights = s->out_heights.data(); out->n_heights = s->out_heights.size();
    out->fields = s->out_fields.data(); out->n_fields = s->out_fields.size();
    out->commitments = s->out_commitments.data(); out->n_commitments = s->out_commitments.size() / 4;
}

int mdn_prove_begin(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces, const mdn_challenger* challenger,
                    uint32_t flags, uint64_t main_root[4], uint64_t* randomness_out) {
    if (!s) return MDN_ERR_INVALID_ARG;
    API_TRY(s)
    ArenaScope proof_memory(s->use_arena ? &s->arena : nullptr);
    CUDA_OK(cudaSetDevice(s->device));
    s->prove_begin(st, traces, challenger, flags);
    if (main_root) memcpy(main_root, s->main_c.root, 32);
    copy_randomness(s, randomness_out);
    API_CATCH(s)
}

int mdn_prove_commit_aux(mdn_session* s, const mdn_matrix* aux, const uint64_t* const* aux_values, uint64_t aux_root[4]) {
    if (!s) return MDN_ERR_INVALID_ARG;
    API_TRY(s)
    ArenaScope proof_memory(s->use_arena ? &s->arena : nullptr);
    CUDA_OK(cudaSetDevice(s->device));
    s->commit_aux(aux, aux_values, aux == nullptr);
    if (aux_root) memcpy(aux_root, s->aux_c.root, 32);
    API_CATCH(s)
}

int mdn_prove_finish(mdn_session* s, mdn_proof* out) {
    if (!s || !out) return MDN_ERR_INVALID_ARG;
    API_TRY(s)
    ArenaScope proof_memory(s->use_arena ? &s->arena : nullptr);
    CUDA_OK(cudaSetDevice(s->device));
    s->finish();
    fill_proof(s, out);
    s->release_proof_memory();
    API_CATCH(s)
}

int mdn_prove(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces, const mdn_challenger* challenger,
              mdn_aux_builder build_aux, void* aux_ctx, uint32_t flags, mdn_proof* out) {
    if (!s || !out) return MDN_ERR_INVALID_ARG;
    API_TRY(s)
    const bool cm = column_major(flags);
    if (cm && build_aux) fail(MDN_ERR_INVALID_ARG, "with MDN_FLAG_COLUMN_MAJOR the aux traces come from the device aux builder (mdn_session_set_device_aux_builder): build_aux must be NULL");
    ArenaScope proof_memory(s->use_arena ? &s->arena : nullptr);
    CUDA_OK(cudaSetDevice(s->device));
    s->prove_begin(st, traces, challenger, flags);
    if (cm && s->dev_aux) {
        s->commit_aux(nullptr, nullptr, false, traces);
    } else if (!build_aux) {
        s->commit_aux(nullptr, nullptr, true);
    } else {
        if (flags & MDN_FLAG_DEVICE_TRACES) fail(MDN_ERR_UNSUPPORTED, "an aux builder needs host-resident main traces");
        u32 k = st->n_airs;
        std::vector<std::vector<u64>> aux_bufs(k), val_bufs(k);
        std::vector<mdn_matrix> aux_mats(k);
        std::vector<const u64*> val_ptrs(k);
        for (u32 i = 0; i < k; i++) {
            const mdn_air& a = st->airs[i];
            if (a.lookup) { aux_mats[i] = mdn_matrix{nullptr, traces[i].log_height, 2 * a.aux_width}; val_ptrs[i] = nullptr; continue; }   // built on the device
            size_t N = (size_t)1 << traces[i].log_height;
            aux_bufs[i].assign(N * 2 * a.aux_width, 0);
            val_bufs[i].assign(2 * (size_t)a.num_aux_values + 1, 0);
            std::vector<u64> r;
            for (u32 q = 0; q < a.num_randomness; q++) { r.push_back(s->randomness[q].a); r.push_back(s->randomness[q].b); }
            r.push_back(0);
            if (build_aux(aux_ctx, i, &traces[i], r.data(), aux_bufs[i].data(), val_bufs[i].data()) != 0)
                fail(MDN_ERR_AUX_BUILDER, "aux builder failed for instance %u", i);
            aux_mats[i] = mdn_matrix{aux_bufs[i].data(), traces[i].log_height, 2 * a.aux_width};
            val_ptrs[i] = val_bufs[i].data();
        }
        s->commit_aux(aux_mats.data(), val_ptrs.data(), false);
    }
    s->finish();
    fill_proof(s, out);
    s->release_proof_memory();
    API_CATCH(s)
}

int mdn_check_constraints(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces, const mdn_matrix* preprocessed,
                          const mdn_challenger* challenger, mdn_aux_builder build_aux, void* aux_ctx, uint32_t flags,
                          uint64_t* randomness_out, mdn_constraint_report* out) {
    return run_check(s, "mdn_check_constraints", nullptr, randomness_out,
                     [&] { s->check_constraints(st, traces, preprocessed, challenger, build_aux, aux_ctx, flags, out); });
}

int mdn_constraint_census(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces, const mdn_matrix* preprocessed,
                          const mdn_challenger* challenger, mdn_aux_builder build_aux, void* aux_ctx, uint32_t flags,
                          uint64_t* randomness_out, mdn_constraint_failure* failures, uint64_t max_failures,
                          mdn_constraint_tally* tallies, uint64_t max_tallies, mdn_constraint_census_report* out) {
    const char* refused = !out ? "null argument"
                        : !failures && max_failures ? "failures is NULL but max_failures is not 0"
                        : !tallies && max_tallies ? "tallies is NULL but max_tallies is not 0" : nullptr;
    return run_check(s, "mdn_constraint_census", refused, randomness_out,
                     [&] { s->constraint_census(st, traces, preprocessed, challenger, build_aux, aux_ctx, flags, failures, max_failures, tallies, max_tallies, out); });
}

int mdn_check_trace_balance(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces, const uint64_t* randomness,
                            const uint64_t* boundary, size_t n_boundary, const uint32_t* const* mutex_sites,
                            uint64_t max_contributions, uint32_t flags, mdn_balance_report* out) {
    return run_check(s, "mdn_check_trace_balance", nullptr, nullptr,
                     [&] { s->check_trace_balance(st, traces, randomness, boundary, n_boundary, mutex_sites, max_contributions, flags, out); });
}

int mdn_check_lookup_folds(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces, const uint64_t* randomness,
                           const uint32_t* const* fold_marks, const mdn_matrix* aux, const uint64_t* const* aux_finals,
                           uint64_t* const* folds_out, uint32_t flags, mdn_fold_report* out) {
    return run_check(s, "mdn_check_lookup_folds", nullptr, nullptr,
                     [&] { s->check_lookup_folds(st, traces, randomness, fold_marks, aux, aux_finals, folds_out, flags, out); });
}

int mdn_lookup_fold_census(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces, const uint64_t* randomness,
                           const uint32_t* const* fold_marks, const mdn_matrix* aux, const uint64_t* const* aux_finals, uint32_t flags,
                           mdn_fold_failure* failures, uint64_t max_failures, mdn_fold_tally* tallies, uint64_t max_tallies,
                           mdn_fold_census_report* out) {
    const char* refused = !out ? "null argument"
                        : !failures && max_failures ? "failures is NULL but max_failures is not 0"
                        : !tallies && max_tallies ? "tallies is NULL but max_tallies is not 0" : nullptr;
    return run_check(s, "mdn_lookup_fold_census", refused, nullptr,
                     [&] { s->lookup_fold_census(st, traces, randomness, fold_marks, aux, aux_finals, flags, failures, max_failures, tallies, max_tallies, out); });
}

size_t mdn_proof_serialize(const mdn_proof* p, uint8_t* out, size_t cap) {
    size_t need = 8 + p->n_heights + 8 + 8 * p->n_fields + 8 + 32 * p->n_commitments;
    if (!out || cap < need) return need;
    auto put64 = [&](uint64_t v) { for (int i = 0; i < 8; i++) *out++ = (uint8_t)(v >> (8 * i)); };
    put64(p->n_heights); memcpy(out, p->log_trace_heights, p->n_heights); out += p->n_heights;
    put64(p->n_fields); for (size_t i = 0; i < p->n_fields; i++) put64(p->fields[i]);
    put64(p->n_commitments); for (size_t i = 0; i < 4 * p->n_commitments; i++) put64(p->commitments[i]);
    return need;
}

int mdn_coset_lde_batch(mdn_session* s, const mdn_matrix* mat, uint32_t added_bits, uint64_t shift, uint64_t* out) {
    if (!s || !mat || !out) return MDN_ERR_INVALID_ARG;
    API_TRY(s)
    CUDA_OK(cudaSetDevice(s->device));
    if (added_bits != s->params.log_blowup) fail(MDN_ERR_UNSUPPORTED, "added_bits must equal the session's log_blowup");
    if (mat->log_height > 22) fail(MDN_ERR_UNSUPPORTED, "trace height 2^%u exceeds the supported 2^22", mat->log_height);
    if (mat->log_height + added_bits > 32) fail(MDN_ERR_DOMAIN, "LDE log order %u exceeds two-adicity 32", mat->log_height + added_bits);
    if (s->in_proof) fail(MDN_ERR_INVALID_ARG, "mdn_coset_lde_batch called inside a proof");
    if (shift != gl::lde_shift(mat->log_height + added_bits)) fail(MDN_ERR_UNSUPPORTED, "only the canonical LDE shift 7^(2^(32-log_lde)) is supported");
    Committed c;
    size_t N = (size_t)1 << mat->log_height, L = N << added_bits;
    c.coef_buf.alloc(N * mat->width, s->stream); c.lde_buf.alloc(L * mat->width, s->stream);
    c.mats.push_back(CommittedMat{c.lde_buf.p, c.coef_buf.p, mat->log_height, mat->width});
    s->upload_matrix(*mat, false, c.coef_buf.p);
    s->check_input_flag("the matrix");
    s->lde_matrix(c.mats[0]);          // the LDE only: no tree
    DevBuf rm; rm.alloc(L * mat->width, s->stream);
    mk::launch_export_lde_bitrev_rm(c.lde_buf.p, mat->log_height, added_bits, mat->width, rm.p, s->stream);
    CUDA_OK(cudaMemcpyAsync(out, rm.p, L * mat->width * sizeof(u64), cudaMemcpyDeviceToHost, s->stream));
    CUDA_OK(cudaStreamSynchronize(s->stream));
    API_CATCH(s)
}

// The matrices are trace-domain evaluations (height N); the committed tree is the one
// `commit_traces` builds: LDE by the session blowup then build_aligned_tree.
int mdn_lmcs_commit(mdn_session* s, const mdn_matrix* mats, uint32_t n_mats, uint64_t root[4]) {
    if (!s || !mats || !root || !n_mats) return MDN_ERR_INVALID_ARG;
    API_TRY(s)
    CUDA_OK(cudaSetDevice(s->device));
    u32 lb = s->params.log_blowup;
    Committed c;
    size_t ct = 0, lt = 0;
    for (u32 i = 0; i < n_mats; i++) {
        if (i && mats[i].log_height < mats[i - 1].log_height) fail(MDN_ERR_INVALID_ARG, "matrices must be sorted by ascending height");
        size_t N = (size_t)1 << mats[i].log_height; ct += N * mats[i].width; lt += (N << lb) * mats[i].width;
    }
    c.coef_buf.alloc(ct, s->stream); c.lde_buf.alloc(lt, s->stream);
    size_t co = 0, lo = 0;
    for (u32 i = 0; i < n_mats; i++) {
        size_t N = (size_t)1 << mats[i].log_height;
        c.mats.push_back(CommittedMat{c.lde_buf.p + lo, c.coef_buf.p + co, mats[i].log_height, mats[i].width});
        s->upload_matrix(mats[i], false, c.coef_buf.p + co);
        co += N * mats[i].width; lo += (N << lb) * mats[i].width;
    }
    s->check_input_flag("a matrix");
    s->lde_and_commit(c, nullptr, nullptr);
    memcpy(root, c.root, 32);
    API_CATCH(s)
}

int mdn_poseidon2_permute(mdn_session* s, uint64_t* states, size_t n) {
    if (!s || !states) return MDN_ERR_INVALID_ARG;
    API_TRY(s)
    CUDA_OK(cudaSetDevice(s->device));
    DevBuf d; d.alloc(12 * n, s->stream);
    CUDA_OK(cudaMemcpyAsync(d.p, states, 12 * n * sizeof(u64), cudaMemcpyHostToDevice, s->stream));
    mk::launch_poseidon2_batch(d.p, n, s->stream);
    CUDA_OK(cudaMemcpyAsync(states, d.p, 12 * n * sizeof(u64), cudaMemcpyDeviceToHost, s->stream));
    CUDA_OK(cudaStreamSynchronize(s->stream));
    API_CATCH(s)
}

void mdn_challenger_observe(mdn_challenger* c, const uint64_t* felts, size_t n) {
    Duplex d;
    memcpy(d.st, c->sponge_state, sizeof d.st);
    memcpy(d.in, c->input_buffer, sizeof d.in);
    d.in_len = c->input_len; d.out_len = c->output_len;
    for (size_t i = 0; i < n; i++) d.observe(felts[i]);
    memcpy(c->sponge_state, d.st, sizeof d.st);
    for (u32 i = 0; i < 8; i++) c->input_buffer[i] = i < d.in_len ? d.in[i] : 0;
    c->input_len = d.in_len; c->output_len = d.out_len;
}
uint64_t mdn_challenger_sample(mdn_challenger* c) {
    Duplex d;
    memcpy(d.st, c->sponge_state, sizeof d.st);
    memcpy(d.in, c->input_buffer, sizeof d.in);
    d.in_len = c->input_len; d.out_len = c->output_len;
    u64 v = d.sample();
    memcpy(c->sponge_state, d.st, sizeof d.st);
    for (u32 i = 0; i < 8; i++) c->input_buffer[i] = i < d.in_len ? d.in[i] : 0;
    c->input_len = d.in_len; c->output_len = d.out_len;
    return v;
}

long long mdn_get_info(mdn_session* s, mdn_info what, uint64_t* out, size_t cap) {
    if (!s && what != MDN_INFO_JIT_CACHE) return -1;
    std::vector<u64> v;
    switch (what) {
        case MDN_INFO_JIT_CACHE: {
            const jit::CacheStats& c = jit::cache_stats();
            v = {c.disk_hits.load(), c.disk_misses.load(), c.rejected.load(), c.write_failures.load(), c.compiles.load(),
                 c.compile_ns.load() / 1000000};
            break;
        }
        case MDN_INFO_MAIN_ROOT: v.assign(s->dbg_roots[0], s->dbg_roots[0] + 4); break;
        case MDN_INFO_AUX_ROOT: v.assign(s->dbg_roots[1], s->dbg_roots[1] + 4); break;
        case MDN_INFO_QUOTIENT_ROOT: v.assign(s->dbg_roots[2], s->dbg_roots[2] + 4); break;
        case MDN_INFO_OOD_POINT: v = {s->ood_z.a, s->ood_z.b}; break;
        case MDN_INFO_QUOTIENT_ACC: v = s->dbg_quot_acc; break;
        case MDN_INFO_DEEP_EVALS: v = s->dbg_deep; break;
        case MDN_INFO_FRI_ROOTS: v = s->dbg_fri_roots; break;
        case MDN_INFO_QUERY_INDICES: v = s->dbg_queries; break;
        case MDN_INFO_JIT: v = s->jit_used; break;
        case MDN_INFO_JIT_CHECK: v = s->jit_check_used; break;
        case MDN_INFO_JIT_LOOKUP_CHECK: v = s->jit_lookup_check_used; break;
        case MDN_INFO_POOL: {
            cudaMemPool_t pool; uint64_t a[4] = {0, 0, 0, 0};
            if (cudaDeviceGetDefaultMemPool(&pool, s->device) == cudaSuccess) {
                cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReservedMemCurrent, &a[0]);
                cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReservedMemHigh, &a[1]);
                cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &a[2]);
                cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemHigh, &a[3]);
            }
            v.assign(a, a + 4);
            { size_t cap = 0; for (auto& sl : s->arena.slabs) cap += sl.size; v.push_back(cap); v.push_back(s->arena.slabs.size()); v.push_back(s->arena.grow_events); v.push_back(s->arena.live); }
            break;
        }
        case MDN_INFO_BUILD: v = {2, 2}; break;
        default: return -1;
    }
    if (out) for (size_t i = 0; i < v.size() && i < cap; i++) out[i] = v[i];
    return (long long)v.size();
}

int mdn_session_set_shard(mdn_session* s, uint32_t rank, uint32_t world, mdn_allgather_fn fn, void* ctx) {
    if (!s) return MDN_ERR_INVALID_ARG;
    if (world == 0 || (world & (world - 1)) || world > mk::MAX_RANKS || rank >= world || (world > 1 && !fn)) {
        s->error = "invalid shard configuration (world must be a power of two <= 8, callback required)"; return MDN_ERR_INVALID_ARG;
    }
    if (s->in_proof) { s->error = "mdn_session_set_shard called inside a proof"; return MDN_ERR_INVALID_ARG; }
    try {
        CUDA_OK(cudaSetDevice(s->device));
        s->shard_teardown();
        if (world == 1) return MDN_OK;
        s->shard_rank = rank; s->shard_world = world; s->allgather = fn; s->allgather_ctx = ctx;
        s->shard_log_g = 0; while ((1u << s->shard_log_g) < world) s->shard_log_g++;
        if (const char* e = getenv("MDN_SHARD_MIN_LOG")) s->shard_min_log = (u32)atoi(e);
        // the proof arena starts over as a shared arena: every slab is mapped into every rank when it is created
        s->arena.destroy();
        s->arena.on_new_slab = [s](char* base, size_t size) { s->shard_map_slab(base, size); };
        s->arena.before_drop_slabs = [s]() { s->shard_unmap_slabs(); };
        // barrier flags: one slot per source rank, zeroed before any peer can see the buffer
        CUDA_OK(cudaMalloc((void**)&s->sync_local, 4096));
        CUDA_OK(cudaMemsetAsync(s->sync_local, 0, 4096, s->stream));
        CUDA_OK(cudaStreamSynchronize(s->stream));
        cudaIpcMemHandle_t h;
        CUDA_OK(cudaIpcGetMemHandle(&h, s->sync_local));
        std::vector<u64> mine(8), all(8 * (size_t)world);
        memcpy(mine.data(), &h, 64);
        if (fn(ctx, mine.data(), all.data(), 8) != 0) fail(MDN_ERR_INVALID_ARG, "all-gather callback failed");
        for (u32 g = 0; g < world; g++) {
            if (g == rank) { s->sync_flags.p[g] = s->sync_local; continue; }
            cudaIpcMemHandle_t hg; memcpy(&hg, &all[8 * (size_t)g], 64);
            void* m = nullptr;
            CUDA_OK(cudaIpcOpenMemHandle(&m, hg, cudaIpcMemLazyEnablePeerAccess));
            s->sync_flags.p[g] = (u64*)m;
        }
        s->sync_epoch = 0;
        // rendezvous: no rank may go on (and possibly fail and free its buffer) before every rank has mapped it
        { std::vector<u64> one(1, 0), got(world); if (fn(ctx, one.data(), got.data(), 1) != 0) fail(MDN_ERR_INVALID_ARG, "all-gather callback failed"); }
    } catch (const MdnError& e) { s->error = e.what(); return e.code; }
    catch (const std::exception& e) { s->error = e.what(); return MDN_ERR_INVALID_ARG; }
    return MDN_OK;
}

int mdn_session_set_hash(mdn_session* s, mdn_hash_kind kind) {
    if (!s) return MDN_ERR_INVALID_ARG;
    if (kind < MDN_HASH_POSEIDON2 || kind > MDN_HASH_RPX) { s->error = "unknown hash configuration"; return MDN_ERR_UNSUPPORTED; }
    if (s->in_proof) { s->error = "mdn_session_set_hash called inside a proof"; return MDN_ERR_INVALID_ARG; }
    if (s->has_prep && kind != s->hash_kind) { s->error = "the preprocessed bundle was committed under the other hash: remove it first"; return MDN_ERR_INVALID_ARG; }
    s->hash_kind = kind;
    return MDN_OK;
}
int mdn_session_set_hash_challenger(mdn_session* s, const mdn_hash_challenger* c) {
    if (!s || !c || (c->input_len && !c->input_buffer) || (c->output_len && !c->output_buffer)) return MDN_ERR_INVALID_ARG;
    if (c->input_len % 4 || c->output_len > 32) { s->error = "hash challenger: the input buffer must be whole 32-bit words and the output buffer at most 32 bytes"; return MDN_ERR_INVALID_ARG; }
    s->hash_ch_in.assign(c->input_buffer, c->input_buffer + c->input_len);
    s->hash_ch_out.assign(c->output_buffer, c->output_buffer + c->output_len);
    return MDN_OK;
}

int mdn_session_set_external_check(mdn_session* s, mdn_external_check fn, void* ctx) {
    if (!s) return MDN_ERR_INVALID_ARG;
    s->external_check = fn; s->external_ctx = ctx;
    return MDN_OK;
}

int mdn_session_set_constraint_guard(mdn_session* s, uint32_t enable) {
    if (!s) return MDN_ERR_INVALID_ARG;
    if (enable > 1) { s->error = "mdn_session_set_constraint_guard: enable must be 0 or 1"; return MDN_ERR_INVALID_ARG; }
    if (s->in_proof) { s->error = std::string("mdn_session_set_constraint_guard") + IN_PROOF; return MDN_ERR_INVALID_ARG; }
    s->constraint_guard = enable == 1;
    return MDN_OK;
}

int mdn_last_constraint_report(const mdn_session* s, mdn_constraint_report* out) {
    if (!s || !out) return MDN_ERR_INVALID_ARG;
    *out = s->guard_report;
    return MDN_OK;
}

int mdn_session_set_device_aux_builder(mdn_session* s, mdn_aux_builder_device fn, void* ctx) {
    if (!s) return MDN_ERR_INVALID_ARG;
    s->dev_aux = fn; s->dev_aux_ctx = fn ? ctx : nullptr;
    return MDN_OK;
}

int mdn_session_set_preprocessed(mdn_session* s, const mdn_statement* st, const mdn_matrix* preprocessed, uint64_t commitment_out[4]) {
    if (!s) return MDN_ERR_INVALID_ARG;
    try {
        CUDA_OK(cudaSetDevice(s->device));
        s->set_preprocessed(st, preprocessed);
        if (commitment_out) { if (s->has_prep) memcpy(commitment_out, s->prep_c.root, 32); else memset(commitment_out, 0, 32); }
    } catch (const MdnError& e) { s->error = e.what(); s->prep_c = Committed(); s->has_prep = false; return e.code; }
    catch (const std::exception& e) { s->error = e.what(); s->prep_c = Committed(); s->has_prep = false; return MDN_ERR_INVALID_ARG; }
    return MDN_OK;
}

const char* mdn_jit_status(mdn_session* s) {
    static thread_local std::string msg;
    jit::Nvrtc& n = jit::nvrtc();
    msg = n.ok() ? "nvrtc " + std::to_string(n.version / 100) + "." + std::to_string(n.version % 100) : "nvrtc unavailable (" + n.why + ")";
    if (s && !s->jit_note.empty()) msg += "; " + s->jit_note;
    return msg.c_str();
}

int mdn_session_set_jit(mdn_session* s, uint32_t min_nodes) {
    if (!s) return MDN_ERR_INVALID_ARG;
    s->jit_min_nodes = min_nodes;
    return MDN_OK;
}

int mdn_jit_set_cache_dir(const char* dir) {
    std::string err;
    if (!jit::set_cache_dir(dir, &err)) { g_create_error = err; return MDN_ERR_INVALID_ARG; }
    return MDN_OK;
}

// Codegen + NVRTC only (no device needed): returns the cubin size, or a negative status with the compiler log
// in *err (static buffer).  Lets CPU-only CI check that an AIR lowers and compiles.
long long mdn_jit_compile_check(const uint32_t* program, uint32_t program_words, const char** err) {
    static thread_local std::string msg;
    try {
        std::vector<u32> v1;
        if (program && program_words >= 6 && program[0] == 0x504B4C4Du && program[1] == 2) {
            // a version-2 lookup program: its interaction part, split with every range the program itself can satisfy
            const u32 nn = program[2], nc = program[3], nr = program[5];
            u32 n_cols = 1;
            for (u32 q = 0; q < nc && (size_t)6 + 3 * (size_t)nn + 4 * (size_t)q < program_words; q++) n_cols = std::max(n_cols, program[6 + 3 * (size_t)nn + 4 * (size_t)q] + 1);
            mdn_air a{};
            a.width = a.num_randomness = a.num_periodic_columns = a.preprocessed_width = ~0u;
            a.aux_width = n_cols + nr; a.num_aux_values = 1;
            try { v1 = split_lookup_v2(0, a, ~0u, mdn_lookup{n_cols, program_words, program}).v1; }
            catch (const MdnError& e) { msg = e.what(); if (err) *err = msg.c_str(); return MDN_ERR_INVALID_ARG; }
            program = v1.data(); program_words = (u32)v1.size();
        }
        const bool lookup = program && program_words >= 5 && program[0] == 0x504B4C4Du;
        if (!program || program_words < 5 || (program[0] != 0x5249414Du && !lookup) || program[1] != 1 ||
            (size_t)program_words != 5 + 3 * (size_t)program[2] + (lookup ? 4 : 1) * (size_t)program[3] + 2 * (size_t)program[4]) { msg = "bad program"; if (err) *err = msg.c_str(); return MDN_ERR_INVALID_ARG; }
        for (u32 j = 0; j < program[2]; j++) {
            u32 op = program[5 + 3 * j], x = program[6 + 3 * j], y = program[7 + 3 * j];
            if (op > 15 || (op >= 10 && op <= 12 && (x >= j || y >= j)) || (op == 13 && x >= j) || ((op == 8) && x >= program[4]) || (op == 9 && x + 1 >= program[4])) { msg = "malformed node"; if (err) *err = msg.c_str(); return MDN_ERR_INVALID_ARG; }
        }
        if (lookup) {
            u32 n_cols = 0;
            for (u32 q = 0; q < program[3]; q++) {
                const u32* it = program + 5 + 3 * (size_t)program[2] + 4 * (size_t)q;
                if ((it[1] != 0xFFFFFFFFu && it[1] >= program[2]) || it[2] >= program[2] || it[3] >= program[2] || it[0] >= 16) { msg = "bad interaction"; if (err) *err = msg.c_str(); return MDN_ERR_INVALID_ARG; }
                n_cols = std::max(n_cols, it[0] + 1);
            }
            return (long long)jit::cubin_for(program, program_words, nullptr, jit::MODE_LOOKUP, n_cols).size();
        }
        for (u32 q = 0; q < program[3]; q++) if (program[5 + 3 * (size_t)program[2] + q] >= program[2]) { msg = "bad constraint id"; if (err) *err = msg.c_str(); return MDN_ERR_INVALID_ARG; }
        return (long long)jit::cubin_for(program, program_words, nullptr).size();
    } catch (const std::exception& e) { msg = e.what(); if (err) *err = msg.c_str(); return MDN_ERR_UNSUPPORTED; }
}

// sizeof / offsetof of every struct of the boundary, so a binding (ctypes, Rust #[repr(C)]) can assert its layout
size_t mdn_abi_layout(uint32_t* out, size_t cap) {
    const uint32_t v[] = {
        (uint32_t)sizeof(mdn_pcs_params), (uint32_t)sizeof(mdn_challenger), (uint32_t)sizeof(mdn_lookup), (uint32_t)sizeof(mdn_air),
        (uint32_t)offsetof(mdn_air, program), (uint32_t)offsetof(mdn_air, periodic_values), (uint32_t)offsetof(mdn_air, preprocessed_width),
        (uint32_t)offsetof(mdn_air, lookup), (uint32_t)sizeof(mdn_matrix), (uint32_t)sizeof(mdn_statement), (uint32_t)sizeof(mdn_proof),
        (uint32_t)sizeof(mdn_timings), (uint32_t)offsetof(mdn_timings, kernel_ms), (uint32_t)offsetof(mdn_timings, permutations)};
    size_t n = sizeof v / sizeof v[0];
    if (out) for (size_t i = 0; i < n && i < cap; i++) out[i] = v[i];
    return n;
}

int mdn_set_debug(mdn_session* s, int enable) {
    if (!s) return MDN_ERR_INVALID_ARG;
    s->keep_debug = enable != 0;
    return MDN_OK;
}

int mdn_get_timings(mdn_session* s, mdn_timings* out) {
    if (!s || !out) return MDN_ERR_INVALID_ARG;
    *out = s->timings;
    return MDN_OK;
}

}  // extern "C"
