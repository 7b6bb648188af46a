// Host-side mirror of the reference's proving interface, in C++ over the C ABI (include/miden_b200.h).
//
// The reference host is Rust; this image has no Rust toolchain, so the layer a Rust maintainer would write above
// the FFI (INTEGRATION.md) is restated here in C++ with the reference's names and argument meaning:
//
//   reference (crates/lifted-stark, prover/src/lib.rs)            here
//   ------------------------------------------------------------  -----------------------------------------------
//   PcsParams::new(..)                      pcs/params.rs:35-99   miden::PcsParams
//   StarkConfig (pcs + lmcs + dft + challenger)  config.rs:26-45  miden::StarkConfig   (device instead of dft/lmcs)
//   LiftedAir: width / aux_width / num_randomness / eval ..       miden::Air           (eval lowered to an op-list)
//   Statement::new(airs, air_inputs, aux_inputs)                  miden::Statement
//   ProverStatement::new(statement, traces)                       miden::ProverStatement   (shape errors -> InstanceError)
//   Preprocessed::build(&statement, &config) / .commitment()      miden::Preprocessed::build / commitment()
//   ProverInstance::new(&config, &prover_statement, preprocessed) miden::ProverInstance
//   ProverInstance::prove(challenger) -> StarkOutput              ProverInstance::prove(challenger) -> StarkOutput
//   StarkProofData { log_trace_heights, transcript }              miden::StarkProofData
//   debug::check_constraints(&prover_statement, challenger)       miden::check_constraints(config, statement, challenger)
//     (debug.rs:70-214; panics -> ConstraintViolation)             (every constraint on every row, on the device, no proof)
//   lookup::debug::check_trace_balance(air, main, .., challenges)  miden::check_trace_balance(config, statement, challenges, ..)
//   lookup::debug::collect_column_oracle_folds(air, main, ..)      miden::check_lookup_folds(config, statement, challenges, ..)
//     (air/src/lookup/debug/trace/mod.rs:169-309) -> BalanceReport  -> miden::BalanceReport (to_string() = its Display)
//   ProverError::{Instance, Domain, ..}  prover/mod.rs:582-596    miden::ProverError { kind, what() }
//   HashFunction::{Blake3_256, Keccak, Rpo256, Poseidon2, Rpx256} -> the config constructor (prover/src/lib.rs:245-301)
//                                                                 miden::HashFunction + StarkConfig::with_hash
//
// Header-only; link with -lmiden_b200.  There is no CPU fallback: constructing a StarkConfig without a usable
// CUDA device throws ProverError{NoDevice}.
#pragma once
#include "../../include/miden_b200.h"
#include <algorithm>
#include <array>
#include <cstdint>
#include <functional>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

namespace miden {

using Felt = uint64_t;                       // canonical Goldilocks element (crates/field/src/native/mod.rs:58)
using QuadFelt = std::array<Felt, 2>;        // (c0, c1) of F[u]/(u^2 - 7)
using Commitment = std::array<Felt, 4>;      // Hash<Felt, Felt, 4>

struct ProverError : std::runtime_error {
    enum Kind { Instance, Domain, Cuda, Unsupported, AuxBuilder, NoDevice, ExternalAssertion } kind;
    ProverError(Kind k, const std::string& m) : std::runtime_error(m), kind(k) {}
    static Kind from_status(int rc) {
        switch (rc) {
            case MDN_ERR_DOMAIN: return Domain;
            case MDN_ERR_CUDA: return Cuda;
            case MDN_ERR_UNSUPPORTED: return Unsupported;
            case MDN_ERR_AUX_BUILDER: return AuxBuilder;
            case MDN_ERR_NO_DEVICE: return NoDevice;
            case MDN_ERR_EXTERNAL_ASSERTION: return ExternalAssertion;
            default: return Instance;
        }
    }
};

struct PcsParams {
    uint32_t log_blowup = 3, log_folding_arity = 2, log_final_degree = 7;
    uint32_t folding_pow_bits = 4, deep_pow_bits = 12, num_queries = 27, query_pow_bits = 16;   // air/src/config.rs:55-67
    mdn_pcs_params raw() const { return {log_blowup, log_folding_arity, log_final_degree, folding_pow_bits, deep_pow_bits, num_queries, query_pow_bits}; }
};

// `HashFunction` of miden_prover::prove_stark's match (prover/src/lib.rs:245-301) = which miden_air::config constructor applies
enum class HashFunction { Poseidon2 = MDN_HASH_POSEIDON2, Blake3_256 = MDN_HASH_BLAKE3, Keccak = MDN_HASH_KECCAK, Rpo256 = MDN_HASH_RPO, Rpx256 = MDN_HASH_RPX };

// p3 DuplexChallenger<Felt, Poseidon2, 12, 8> state (air/src/config.rs:223,264-271)
struct Challenger {
    mdn_challenger raw{};
    void observe(Felt x) { mdn_challenger_observe(&raw, &x, 1); }
    void observe_slice(const std::vector<Felt>& xs) { if (!xs.empty()) mdn_challenger_observe(&raw, xs.data(), xs.size()); }
    Felt sample() { return mdn_challenger_sample(&raw); }
};

// RowMajorMatrix<Felt> view: height = 2^log_height
struct RowMajorMatrix {
    std::vector<Felt> values;
    uint32_t log_height = 0, width = 0;
    RowMajorMatrix() {}
    RowMajorMatrix(std::vector<Felt> v, uint32_t w) : values(std::move(v)), width(w) {
        size_t h = w ? values.size() / w : 0;
        if (!w || h * w != values.size() || (h & (h - 1)) || !h) throw ProverError(ProverError::Instance, "matrix height must be a power of two");
        while ((size_t(1) << log_height) < h) log_height++;
    }
    size_t height() const { return size_t(1) << log_height; }
    mdn_matrix raw() const { return {values.data(), log_height, width}; }
};

// Recording builder for `LiftedAir::eval` (the symbolic capture a Rust shim performs once per AIR)
class AirBuilder {
public:
    struct Expr { uint32_t id; };
    Expr main(uint32_t offset, uint32_t col) { return node(0, offset, col); }
    Expr aux(uint32_t offset, uint32_t col) { return node(1, offset, col); }
    Expr public_value(uint32_t i) { return node(2, i, 0); }
    Expr challenge(uint32_t i) { return node(3, i, 0); }
    Expr aux_value(uint32_t i) { return node(4, i, 0); }
    Expr is_first_row() { return node(5, 0, 0); }
    Expr is_last_row() { return node(6, 0, 0); }
    Expr is_transition() { return node(7, 0, 0); }
    Expr constant(Felt v) { consts_.push_back(v); return node(8, (uint32_t)consts_.size() - 1, 0); }
    Expr periodic(uint32_t col) { return node(14, col, 0); }
    Expr preprocessed(uint32_t offset, uint32_t col) { return node(15, offset, col); }
    Expr add(Expr a, Expr b) { return node(10, a.id, b.id); }
    Expr sub(Expr a, Expr b) { return node(11, a.id, b.id); }
    Expr mul(Expr a, Expr b) { return node(12, a.id, b.id); }
    Expr neg(Expr a) { return node(13, a.id, 0); }
    void assert_zero(Expr e) { constraints_.push_back(e.id); }
    void assert_zero_ext(Expr e) { constraints_.push_back(e.id); }
    std::vector<uint32_t> finish() const {
        std::vector<uint32_t> w = {0x5249414Du, 1u, (uint32_t)(nodes_.size() / 3), (uint32_t)constraints_.size(), (uint32_t)consts_.size()};
        w.insert(w.end(), nodes_.begin(), nodes_.end());
        w.insert(w.end(), constraints_.begin(), constraints_.end());
        for (Felt c : consts_) { w.push_back((uint32_t)c); w.push_back((uint32_t)(c >> 32)); }
        return w;
    }
private:
    Expr node(uint32_t op, uint32_t a, uint32_t b) { nodes_.insert(nodes_.end(), {op, a, b}); return Expr{(uint32_t)(nodes_.size() / 3 - 1)}; }
    std::vector<uint32_t> nodes_, constraints_;
    std::vector<Felt> consts_;
};

// One AIR of the MultiAir: the shape queries of LiftedAir plus the lowered eval
struct Air {
    uint32_t width = 0, aux_width = 0, num_aux_values = 0, num_randomness = 0, log_quotient_degree = 0, preprocessed_width = 0;
    std::vector<uint32_t> program;                 // AirBuilder::finish()
    std::vector<Felt> periodic_values;             // row-major (1 << log_max_period) x num_periodic_columns
    uint32_t num_periodic_columns = 0, log_max_period = 0;
    std::vector<uint32_t> lookup_program;          // lowered LookupAir (empty: aux trace from the host builder)
    uint32_t lookup_columns = 0;
    RowMajorMatrix preprocessed_trace;             // BaseAir::preprocessed_trace(); width 0 = None
};

struct Statement {
    std::vector<Air> airs;
    std::vector<Felt> air_inputs;                  // public values
    std::vector<Felt> observe_felts;               // what Statement::observe absorbs (AIR specific)
    // default MultiAir::observe: len(air_inputs), air_inputs, max_aux_inputs (0), len(aux_inputs) (0)
    static Statement with_default_observe(std::vector<Air> airs, std::vector<Felt> air_inputs) {
        Statement s; s.airs = std::move(airs); s.air_inputs = std::move(air_inputs);
        s.observe_felts.push_back(s.air_inputs.size());
        s.observe_felts.insert(s.observe_felts.end(), s.air_inputs.begin(), s.air_inputs.end());
        s.observe_felts.push_back(0); s.observe_felts.push_back(0);
        return s;
    }
};

struct ProverStatement {
    Statement statement;
    std::vector<RowMajorMatrix> traces;            // instance order
    ProverStatement(Statement s, std::vector<RowMajorMatrix> t) : statement(std::move(s)), traces(std::move(t)) {
        if (traces.size() != statement.airs.size()) throw ProverError(ProverError::Instance, "trace count does not match the AIR count");
        for (size_t i = 0; i < traces.size(); i++)
            if (traces[i].width != statement.airs[i].width) throw ProverError(ProverError::Instance, "trace width does not match its AIR");
    }
};

// A trace that already lives on the GPU, column-major: entry (row r, column c) at values[(c << log_height) | r] on the
// config's device, 16-byte aligned.  Not owned: it must stay valid and unchanged while a prove / check runs.
struct ColumnMajorDeviceMatrix {
    const Felt* values = nullptr;
    uint32_t log_height = 0, width = 0;
    size_t height() const { return size_t(1) << log_height; }
    mdn_matrix raw() const { return {values, log_height, width}; }
};

// ProverStatement over device-resident column-major traces (MDN_FLAG_DEVICE_TRACES | MDN_FLAG_COLUMN_MAJOR)
struct DeviceProverStatement {
    Statement statement;
    std::vector<ColumnMajorDeviceMatrix> traces;   // instance order
    DeviceProverStatement(Statement s, std::vector<ColumnMajorDeviceMatrix> t) : statement(std::move(s)), traces(std::move(t)) {
        if (traces.size() != statement.airs.size()) throw ProverError(ProverError::Instance, "trace count does not match the AIR count");
        for (size_t i = 0; i < traces.size(); i++)
            if (traces[i].width != statement.airs[i].width) throw ProverError(ProverError::Instance, "trace width does not match its AIR");
    }
};

// LiftedAir::build_aux_trace on the GPU, for the AIRs that do not ship a lowered LookupAir: write the 2*aux_width base
// columns of `aux_out` (device, column-major, height rows; nullptr when aux_width is 0) with work enqueued on `stream`
// (the session's cudaStream_t) or finished before returning, and fill `aux_values`.
using DeviceAuxBuilder = std::function<void(uint32_t instance, const ColumnMajorDeviceMatrix& main, const std::vector<QuadFelt>& challenges,
                                            Felt* aux_out, std::vector<QuadFelt>& aux_values, void* stream)>;

// GenericStarkConfig: PCS parameters + the pre-bound challenger prototype; owns the device session
class StarkConfig {
public:
    StarkConfig(PcsParams params, Challenger challenger_prototype, int cuda_device = 0) : params_(params), proto_(challenger_prototype) {
        mdn_pcs_params p = params.raw();
        mdn_session* s = nullptr;
        int rc = mdn_session_create(&p, cuda_device, &s);
        if (rc != MDN_OK) throw ProverError(ProverError::from_status(rc), mdn_last_error(nullptr));
        session_.reset(s, mdn_session_destroy);
    }
    // blake3_256_config / keccak_config / rpo_config / rpx_config instead of poseidon2_config.  For the two byte-oriented
    // configurations `hash_challenger_input` is the HashChallenger's input buffer after config.challenger() +
    // observe_protocol_params (relation digest + 8 parameter felts, little-endian u64) and the Challenger prototype is unused;
    // for RPO / RPX the prototype must be the duplex state built over that permutation.
    StarkConfig& with_hash(HashFunction h, const std::vector<uint8_t>& hash_challenger_input = {}) {
        int rc = mdn_session_set_hash(session_.get(), (mdn_hash_kind)h);
        if (rc != MDN_OK) throw ProverError(ProverError::from_status(rc), mdn_last_error(session_.get()));
        if (h == HashFunction::Blake3_256 || h == HashFunction::Keccak) {
            mdn_hash_challenger hc{hash_challenger_input.data(), hash_challenger_input.size(), nullptr, 0};
            rc = mdn_session_set_hash_challenger(session_.get(), &hc);
            if (rc != MDN_OK) throw ProverError(ProverError::from_status(rc), mdn_last_error(session_.get()));
        }
        hash_ = h;
        return *this;
    }
    HashFunction hash() const { return hash_; }
    bool hash_challenger() const { return hash_ == HashFunction::Blake3_256 || hash_ == HashFunction::Keccak; }
    const PcsParams& pcs() const { return params_; }
    Challenger challenger() const { return proto_; }
    mdn_session* session() const { return session_.get(); }
    const std::shared_ptr<mdn_session>& shared_session() const { return session_; }
private:
    PcsParams params_; Challenger proto_;
    HashFunction hash_ = HashFunction::Poseidon2;
    std::shared_ptr<mdn_session> session_;
};

struct TranscriptData { std::vector<Felt> fields; std::vector<Commitment> commitments; };
struct StarkProofData { std::vector<uint8_t> log_trace_heights; TranscriptData transcript; };
struct StarkOutput { StarkProofData proof; };

// LiftedAir::build_aux_trace for the AIRs that do not ship a lowered LookupAir
using AuxBuilder = std::function<void(uint32_t instance, const RowMajorMatrix& main, const std::vector<QuadFelt>& challenges,
                                      std::vector<Felt>& aux_flat /* height x 2*aux_width */, std::vector<QuadFelt>& aux_values)>;

namespace detail {
struct Lowered {                                   // C structs pointing into a Statement
    std::vector<mdn_lookup> lookups; std::vector<mdn_air> airs; mdn_statement st{};
    explicit Lowered(const Statement& s) {
        lookups.resize(s.airs.size()); airs.resize(s.airs.size());
        for (size_t i = 0; i < s.airs.size(); i++) {
            const Air& a = s.airs[i];
            mdn_air& r = airs[i];
            r = mdn_air{};
            r.width = a.width; r.aux_width = a.aux_width; r.num_aux_values = a.num_aux_values; r.num_randomness = a.num_randomness;
            r.log_quotient_degree = a.log_quotient_degree; r.program_words = (uint32_t)a.program.size(); r.program = a.program.data();
            r.periodic_values = a.periodic_values.empty() ? nullptr : a.periodic_values.data();
            r.num_periodic_columns = a.num_periodic_columns; r.log_max_period = a.log_max_period; r.preprocessed_width = a.preprocessed_width;
            if (!a.lookup_program.empty()) {
                lookups[i] = mdn_lookup{a.lookup_columns, (uint32_t)a.lookup_program.size(), a.lookup_program.data()};
                r.lookup = &lookups[i];
            }
        }
        st.airs = airs.data(); st.n_airs = (uint32_t)airs.size();
        st.public_values = s.air_inputs.data(); st.n_public_values = (uint32_t)s.air_inputs.size();
        st.observe_felts = s.observe_felts.data(); st.n_observe_felts = (uint32_t)s.observe_felts.size();
    }
};
inline void check(const StarkConfig& c, int rc) {
    if (rc != MDN_OK) throw ProverError(ProverError::from_status(rc), mdn_last_error(c.session()));
}
// the mdn_aux_builder seam over an AuxBuilder
struct AuxCall {
    const ProverStatement* ps; const AuxBuilder* aux;
    static int call(void* ctx, uint32_t instance, const mdn_matrix* main, const uint64_t* randomness, uint64_t* aux_out, uint64_t* aux_values) {
        const AuxCall* self = (const AuxCall*)ctx;
        try {
            const Air& a = self->ps->statement.airs[instance];
            std::vector<QuadFelt> ch(a.num_randomness);
            for (uint32_t i = 0; i < a.num_randomness; i++) ch[i] = {randomness[2 * i], randomness[2 * i + 1]};
            std::vector<Felt> flat((size_t(1) << main->log_height) * 2 * a.aux_width, 0);
            std::vector<QuadFelt> vals(a.num_aux_values, QuadFelt{0, 0});
            (*self->aux)(instance, self->ps->traces[instance], ch, flat, vals);
            for (size_t i = 0; i < flat.size(); i++) aux_out[i] = flat[i];
            for (size_t i = 0; i < vals.size(); i++) { aux_values[2 * i] = vals[i][0]; aux_values[2 * i + 1] = vals[i][1]; }
            return 0;
        } catch (...) { return -1; }
    }
};
// the mdn_aux_builder_device seam over a DeviceAuxBuilder, installed on the session for one call
struct DeviceAuxCall {
    const DeviceProverStatement* ps; const DeviceAuxBuilder* aux;
    static int call(void* ctx, uint32_t instance, const mdn_matrix*, const uint64_t* randomness, uint64_t* aux_out, uint64_t* aux_values, void* stream) {
        const DeviceAuxCall* self = (const DeviceAuxCall*)ctx;
        try {
            const Air& a = self->ps->statement.airs[instance];
            std::vector<QuadFelt> ch(a.num_randomness);
            for (uint32_t i = 0; i < a.num_randomness; i++) ch[i] = {randomness[2 * i], randomness[2 * i + 1]};
            std::vector<QuadFelt> vals(a.num_aux_values, QuadFelt{0, 0});
            (*self->aux)(instance, self->ps->traces[instance], ch, aux_out, vals, stream);
            for (size_t i = 0; i < vals.size(); i++) { aux_values[2 * i] = vals[i][0]; aux_values[2 * i + 1] = vals[i][1]; }
            return 0;
        } catch (...) { return -1; }
    }
    struct Installed {       // the builder is a session setting: removed again when the call returns or throws
        mdn_session* s;
        Installed(mdn_session* s_, DeviceAuxCall* c) : s(s_) { if (*c->aux) mdn_session_set_device_aux_builder(s, &DeviceAuxCall::call, c); }
        ~Installed() { mdn_session_set_device_aux_builder(s, nullptr, nullptr); }
    };
};
inline StarkOutput to_output(const mdn_proof& proof) {
    StarkOutput out;
    out.proof.log_trace_heights.assign(proof.log_trace_heights, proof.log_trace_heights + proof.n_heights);
    out.proof.transcript.fields.assign(proof.fields, proof.fields + proof.n_fields);
    out.proof.transcript.commitments.resize(proof.n_commitments);
    for (size_t i = 0; i < proof.n_commitments; i++) for (int k = 0; k < 4; k++) out.proof.transcript.commitments[i][k] = proof.commitments[4 * i + k];
    return out;
}
}  // namespace detail

// The panic of debug::check_constraints as an exception, with the report of mdn_check_constraints
struct ConstraintViolation : std::runtime_error {
    mdn_constraint_report report;
    explicit ConstraintViolation(const mdn_constraint_report& r) : std::runtime_error(message(r)), report(r) {}
    static std::string message(const mdn_constraint_report& r) {
        if (r.kind == 2) return "external assertion " + std::to_string(r.constraint) + " is non-zero";              // debug.rs:117
        return "constraint not satisfied at instance " + std::to_string(r.instance) + ", row " + std::to_string(r.row);   // debug.rs:273-281
    }
};

// debug::check_constraints(&prover_statement, challenger) (crates/lifted-stark/src/debug.rs:70-214): every constraint of every
// AIR on every trace row, on the device, without proving.  Throws ConstraintViolation for the first failure the reference
// panics on; ExecutionTrace::check_constraints passes config.challenger() without observe_protocol_params, so the caller
// chooses the seed.  The preprocessed traces are the AIRs' own (Air::preprocessed_trace).
inline void check_constraints(const StarkConfig& config, const ProverStatement& ps, Challenger challenger, AuxBuilder aux = nullptr) {
    detail::Lowered low(ps.statement);
    std::vector<mdn_matrix> mats, prep;
    bool any_prep = false;
    for (const RowMajorMatrix& t : ps.traces) mats.push_back(t.raw());
    for (const Air& a : ps.statement.airs) {
        prep.push_back(a.preprocessed_width ? a.preprocessed_trace.raw() : mdn_matrix{nullptr, 0, 0});
        any_prep |= a.preprocessed_width > 0;
    }
    detail::AuxCall ctx{&ps, &aux};
    mdn_constraint_report rep{};
    detail::check(config, mdn_check_constraints(config.session(), &low.st, mats.data(), any_prep ? prep.data() : nullptr,
                                                config.hash_challenger() ? nullptr : &challenger.raw, aux ? &detail::AuxCall::call : nullptr,
                                                &ctx, 0, nullptr, &rep));
    if (!rep.holds) throw ConstraintViolation(rep);
}
// The same check on device-resident column-major traces, read in place (nothing is uploaded or copied); the aux traces
// come from `aux` on the device (none: zero aux traces).
inline void check_constraints(const StarkConfig& config, const DeviceProverStatement& ps, Challenger challenger, DeviceAuxBuilder aux = nullptr) {
    detail::Lowered low(ps.statement);
    std::vector<mdn_matrix> mats, prep;
    bool any_prep = false;
    for (const ColumnMajorDeviceMatrix& t : ps.traces) mats.push_back(t.raw());
    for (const Air& a : ps.statement.airs) {
        prep.push_back(a.preprocessed_width ? a.preprocessed_trace.raw() : mdn_matrix{nullptr, 0, 0});
        any_prep |= a.preprocessed_width > 0;
    }
    detail::DeviceAuxCall ctx{&ps, &aux};
    detail::DeviceAuxCall::Installed installed(config.session(), &ctx);
    mdn_constraint_report rep{};
    detail::check(config, mdn_check_constraints(config.session(), &low.st, mats.data(), any_prep ? prep.data() : nullptr,
                                                config.hash_challenger() ? nullptr : &challenger.raw, nullptr, nullptr,
                                                MDN_FLAG_DEVICE_TRACES | MDN_FLAG_COLUMN_MAJOR, nullptr, &rep));
    if (!rep.holds) throw ConstraintViolation(rep);
}

// Every violated constraint of a statement (mdn_constraint_census), copied out of the call: `first` is what
// check_constraints reports, `tallies` one entry per failing (instance, constraint) and `failures` the violations in
// (instance, row, constraint) order, each list truncated to the capacity the call was given.
struct ConstraintCensus {
    mdn_constraint_census_report counts{};
    std::vector<mdn_constraint_failure> failures;
    std::vector<mdn_constraint_tally> tallies;
    const mdn_constraint_report& first() const { return counts.first; }
    bool holds() const { return counts.first.holds != 0; }
    // one line per failing constraint, then one per listed failure, in the wording of check_constraints' panics
    std::string to_string() const {
        std::string s;
        if (counts.first.kind == 2) s += ConstraintViolation::message(counts.first) + "\n";
        for (const mdn_constraint_tally& t : tallies)
            s += "constraint " + std::to_string(t.constraint) + " of instance " + std::to_string(t.instance) + " not satisfied on " +
                 std::to_string(t.failing_rows) + " rows (rows " + std::to_string(t.first_row) + " .. " + std::to_string(t.last_row) + ")\n";
        if (tallies.size() < counts.failing_constraints) s += "... " + std::to_string(counts.failing_constraints - tallies.size()) + " more failing constraints\n";
        for (const mdn_constraint_failure& f : failures)
            s += "constraint not satisfied at instance " + std::to_string(f.instance) + ", row " + std::to_string(f.row) +
                 " (constraint " + std::to_string(f.constraint) + ")\n";
        if (failures.size() < counts.violations) s += "... " + std::to_string(counts.violations - failures.size()) + " more violations\n";
        return s;
    }
};
// check_constraints without stopping at the first failure: returns the census instead of throwing (errors of the call
// itself still throw ProverError).  At most max_failures violations and max_tallies tallies are listed.
inline ConstraintCensus constraint_census(const StarkConfig& config, const ProverStatement& ps, Challenger challenger, AuxBuilder aux = nullptr,
                                          uint64_t max_failures = 1024, uint64_t max_tallies = 1024) {
    detail::Lowered low(ps.statement);
    std::vector<mdn_matrix> mats, prep;
    bool any_prep = false;
    for (const RowMajorMatrix& t : ps.traces) mats.push_back(t.raw());
    for (const Air& a : ps.statement.airs) {
        prep.push_back(a.preprocessed_width ? a.preprocessed_trace.raw() : mdn_matrix{nullptr, 0, 0});
        any_prep |= a.preprocessed_width > 0;
    }
    detail::AuxCall ctx{&ps, &aux};
    ConstraintCensus out;
    out.failures.resize(max_failures);
    out.tallies.resize(max_tallies);
    detail::check(config, mdn_constraint_census(config.session(), &low.st, mats.data(), any_prep ? prep.data() : nullptr,
                                                config.hash_challenger() ? nullptr : &challenger.raw, aux ? &detail::AuxCall::call : nullptr,
                                                &ctx, 0, nullptr, max_failures ? out.failures.data() : nullptr, max_failures,
                                                max_tallies ? out.tallies.data() : nullptr, max_tallies, &out.counts));
    out.failures.resize(out.counts.n_failures);
    out.tallies.resize(out.counts.n_tallies);
    return out;
}

// check_trace_balance's BalanceReport (air/src/lookup/debug/trace/mod.rs:44-95), copied out of the session.  A push names its
// interaction (the index in the AIR's lookup program) where the reference names its group and message; the caller maps
// the index back to its insert site.  Boundary emissions have instance / column 0xFFFFFFFF and row UINT64_MAX.
struct BalanceReport {
    struct Push { uint32_t instance, column, interaction; uint64_t row; Felt multiplicity; };
    struct Unmatched { QuadFelt denom; Felt net_multiplicity; uint64_t n_pushes; Push first; std::vector<Push> contributions; };
    struct MutexViolation { uint32_t instance; uint64_t row; uint32_t column, group, active_flags; };
    std::vector<Unmatched> unmatched;
    std::vector<MutexViolation> mutex_violations;
    uint64_t n_pushes = 0, n_denominators = 0, n_mutex_violations = 0;
    uint32_t n_skipped_airs = 0;
    bool contributions_complete = true;
    bool is_ok() const { return unmatched.empty() && n_mutex_violations == 0; }
    // the reference's Display (mod.rs:97-138): at most four pushes per unmatched denominator
    std::string to_string() const {
        if (is_ok()) return "BalanceReport: OK\n";
        std::string s = "BalanceReport: " + std::to_string(unmatched.size()) + " unmatched, " + std::to_string(n_mutex_violations) + " mutex violations\n";
        auto ef = [](const QuadFelt& q) { return "(" + std::to_string(q[0]) + ", " + std::to_string(q[1]) + ")"; };
        for (const Unmatched& u : unmatched) {
            s += "  denom " + ef(u.denom) + " net multiplicity " + std::to_string(u.net_multiplicity) + "\n";
            const std::vector<Push>& shown = u.contributions.empty() ? std::vector<Push>{u.first} : u.contributions;
            for (size_t i = 0; i < shown.size() && i < 4; i++)
                s += "    row=" + std::to_string(shown[i].row) + " col=" + std::to_string(shown[i].column) + " interaction=" + std::to_string(shown[i].interaction) +
                     " mult=" + std::to_string(shown[i].multiplicity) + (shown[i].instance == 0xFFFFFFFFu ? " [boundary]" : " instance=" + std::to_string(shown[i].instance)) + "\n";
            if (u.n_pushes > std::min<uint64_t>(shown.size(), 4)) s += "    \xE2\x80\xA6 " + std::to_string(u.n_pushes - std::min<uint64_t>(shown.size(), 4)) + " more contributions\n";
        }
        for (const MutexViolation& m : mutex_violations)
            s += "  mutex violation at row " + std::to_string(m.row) + " col " + std::to_string(m.column) + " group " + std::to_string(m.group) + ": " +
                 std::to_string(m.active_flags) + " active flags\n";
        return s;
    }
};

// check_trace_balance(air, main_trace, .., challenges) (air/src/lookup/debug/trace/mod.rs:169-189), jointly over every AIR of the
// statement with a lowered lookup program, on the device.  `challenges` = the randomness (alpha, beta, ...) the caller chose
// (e.g. what mdn_prove_begin sampled); `boundary` = the (denominator, multiplicity) pairs eval_boundary emits; `mutex_sites` =
// per AIR, empty or one word per interaction (include/miden_b200.h).  Throws ProverError on malformed input only.
inline BalanceReport check_trace_balance(const StarkConfig& config, const ProverStatement& ps, const std::vector<QuadFelt>& challenges,
                                         const std::vector<std::pair<QuadFelt, Felt>>& boundary = {},
                                         const std::vector<std::vector<uint32_t>>& mutex_sites = {}, uint64_t max_contributions = 1u << 16) {
    detail::Lowered low(ps.statement);
    std::vector<mdn_matrix> mats;
    for (const RowMajorMatrix& t : ps.traces) mats.push_back(t.raw());
    std::vector<Felt> rnd, bnd;
    for (const QuadFelt& c : challenges) { rnd.push_back(c[0]); rnd.push_back(c[1]); }
    for (const auto& b : boundary) { bnd.push_back(b.first[0]); bnd.push_back(b.first[1]); bnd.push_back(b.second); }
    std::vector<const uint32_t*> sites(ps.statement.airs.size(), nullptr);
    for (size_t i = 0; i < mutex_sites.size() && i < sites.size(); i++) if (!mutex_sites[i].empty()) sites[i] = mutex_sites[i].data();
    mdn_balance_report r{};
    detail::check(config, mdn_check_trace_balance(config.session(), &low.st, mats.data(), rnd.empty() ? nullptr : rnd.data(),
                                                   bnd.empty() ? nullptr : bnd.data(), boundary.size(), mutex_sites.empty() ? nullptr : sites.data(),
                                                   max_contributions, 0, &r));
    BalanceReport out;
    out.n_pushes = r.n_pushes; out.n_denominators = r.n_denominators; out.n_mutex_violations = r.n_mutex_violations;
    out.n_skipped_airs = r.n_skipped_airs; out.contributions_complete = r.contributions_complete != 0;
    size_t c = 0;
    for (uint64_t j = 0; j < r.n_unmatched; j++) {
        const mdn_unmatched& u = r.unmatched[j];
        BalanceReport::Unmatched e{{u.denom[0], u.denom[1]}, u.net_multiplicity, u.n_pushes,
                                   {u.first_instance, 0xFFFFFFFFu, u.first_interaction, u.first_row, 0}, {}};
        if (r.contributions_complete)
            for (uint64_t q = 0; q < u.n_pushes; q++, c++) {
                const mdn_balance_push& p = r.contributions[c];
                e.contributions.push_back({p.instance, p.column, p.interaction, p.row, p.multiplicity});
            }
        if (!e.contributions.empty()) e.first = e.contributions.front();
        out.unmatched.push_back(std::move(e));
    }
    for (uint64_t j = 0; j < r.n_mutex_listed; j++) {
        const mdn_mutex_violation& m = r.mutex_violations[j];
        out.mutex_violations.push_back({m.instance, m.row, m.column, m.group, m.active_flags});
    }
    return out;
}

// collect_column_oracle_folds(air, main_trace, .., challenges) (air/src/lookup/debug/trace/mod.rs:196-207) on the device,
// compared with an aux trace as assert_prover_matches_oracle compares them (processor/src/trace/tests/lookup.rs:185-265).
// `fold_marks` = per AIR, empty or one word per interaction (include/miden_b200.h); `aux` = empty to check the device
// LogUp build of the same traces, else per AIR the aux trace (host row-major, base-flattened) with its closing value in
// `aux_finals`; `folds` = NULL, or filled per AIR with rows x num_columns (V, U) pairs.  Throws ProverError on malformed input only.
struct FoldReport {
    bool holds = true;
    uint32_t kind = 0, instance = 0, column = 0;      // kind: 1 fraction column, 2 accumulator, 3 zero U
    uint64_t row = 0;
    QuadFelt v{}, u{}, expected{}, actual{};
    uint64_t failing_rows = 0, zero_u = 0;
    uint32_t n_skipped_airs = 0;
};
inline FoldReport check_lookup_folds(const StarkConfig& config, const ProverStatement& ps, const std::vector<QuadFelt>& challenges,
                                     const std::vector<std::vector<uint32_t>>& fold_marks = {}, const std::vector<RowMajorMatrix>& aux = {},
                                     const std::vector<QuadFelt>& aux_finals = {},
                                     std::vector<std::vector<std::pair<QuadFelt, QuadFelt>>>* folds = nullptr) {
    detail::Lowered low(ps.statement);
    const size_t k = ps.statement.airs.size();
    std::vector<mdn_matrix> mats, aux_mats;
    for (const RowMajorMatrix& t : ps.traces) mats.push_back(t.raw());
    for (const RowMajorMatrix& t : aux) aux_mats.push_back(t.raw());
    std::vector<Felt> rnd;
    for (const QuadFelt& c : challenges) { rnd.push_back(c[0]); rnd.push_back(c[1]); }
    std::vector<const uint32_t*> marks(k, nullptr);
    for (size_t i = 0; i < fold_marks.size() && i < k; i++) if (!fold_marks[i].empty()) marks[i] = fold_marks[i].data();
    std::vector<std::array<uint64_t, 2>> fin(k);
    std::vector<const uint64_t*> fin_p(k, nullptr);
    for (size_t i = 0; i < aux_finals.size() && i < k; i++) { fin[i] = {aux_finals[i][0], aux_finals[i][1]}; fin_p[i] = fin[i].data(); }
    std::vector<std::vector<uint64_t>> bufs(k);
    std::vector<uint64_t*> buf_p(k, nullptr);
    if (folds) for (size_t i = 0; i < k; i++) if (low.st.airs[i].lookup) {
        bufs[i].assign((size_t(4) * low.st.airs[i].aux_width) << mats[i].log_height, 0);
        buf_p[i] = bufs[i].data();
    }
    mdn_fold_report r{};
    detail::check(config, mdn_check_lookup_folds(config.session(), &low.st, mats.data(), rnd.empty() ? nullptr : rnd.data(),
                                                  fold_marks.empty() ? nullptr : marks.data(), aux.empty() ? nullptr : aux_mats.data(),
                                                  aux.empty() ? nullptr : fin_p.data(), folds ? buf_p.data() : nullptr, 0, &r));
    if (folds) {
        folds->assign(k, {});
        for (size_t i = 0; i < k; i++)
            for (size_t e = 0; e + 3 < bufs[i].size(); e += 4)
                (*folds)[i].push_back({QuadFelt{bufs[i][e], bufs[i][e + 1]}, QuadFelt{bufs[i][e + 2], bufs[i][e + 3]}});
    }
    FoldReport out;
    out.holds = r.holds != 0; out.kind = r.kind; out.instance = r.instance; out.column = r.column; out.row = r.row;
    out.v = {r.fold[0], r.fold[1]}; out.u = {r.fold[2], r.fold[3]};
    out.expected = {r.expected[0], r.expected[1]}; out.actual = {r.actual[0], r.actual[1]};
    out.failing_rows = r.failing_rows; out.zero_u = r.zero_u; out.n_skipped_airs = r.n_skipped_airs;
    return out;
}

// Preprocessed::build(&statement, &config): the LDE tree lives on the device inside the config's session
class Preprocessed {
public:
    // None when no AIR declares preprocessed columns (preprocessed.rs:83-89)
    static std::unique_ptr<Preprocessed> build(const Statement& s, const StarkConfig& config) {
        bool any = false;
        for (const Air& a : s.airs) any |= a.preprocessed_width > 0;
        if (!any) return nullptr;
        detail::Lowered low(s);
        std::vector<mdn_matrix> mats;
        for (const Air& a : s.airs) mats.push_back(a.preprocessed_width ? a.preprocessed_trace.raw() : mdn_matrix{nullptr, 0, 0});
        auto p = std::unique_ptr<Preprocessed>(new Preprocessed());
        detail::check(config, mdn_session_set_preprocessed(config.session(), &low.st, mats.data(), p->commitment_.data()));
        p->session_ = config.shared_session();
        return p;
    }
    // the bundle lives in the session while this object does (the reference lends `&Preprocessed` to each ProverInstance)
    ~Preprocessed() { if (session_) mdn_session_set_preprocessed(session_.get(), nullptr, nullptr, nullptr); }
    Preprocessed(const Preprocessed&) = delete;
    Preprocessed& operator=(const Preprocessed&) = delete;
    const Commitment& commitment() const { return commitment_; }
private:
    Preprocessed() {}
    Commitment commitment_{};
    std::shared_ptr<mdn_session> session_;
};

class ProverInstance {
public:
    // `preprocessed` must be non-null exactly when some AIR declares preprocessed columns (PresenceMismatch otherwise)
    ProverInstance(const StarkConfig& config, const ProverStatement& ps, const Preprocessed* preprocessed, AuxBuilder aux = nullptr)
        : config_(config), ps_(&ps), aux_(std::move(aux)) {
        check_presence(ps.statement, preprocessed);
    }
    // device-resident column-major traces; the aux traces are built on the device by `aux` (none: zero aux traces)
    ProverInstance(const StarkConfig& config, const DeviceProverStatement& ps, const Preprocessed* preprocessed, DeviceAuxBuilder aux = nullptr)
        : config_(config), dps_(&ps), dev_aux_(std::move(aux)) {
        check_presence(ps.statement, preprocessed);
    }
    StarkOutput prove(const Challenger& challenger) const {
        mdn_proof proof{};
        const mdn_challenger* ch = config_.hash_challenger() ? nullptr : &challenger.raw;
        if (dps_) {
            detail::Lowered low(dps_->statement);
            std::vector<mdn_matrix> mats;
            for (const ColumnMajorDeviceMatrix& t : dps_->traces) mats.push_back(t.raw());
            detail::DeviceAuxCall ctx{dps_, &dev_aux_};
            detail::DeviceAuxCall::Installed installed(config_.session(), &ctx);
            detail::check(config_, mdn_prove(config_.session(), &low.st, mats.data(), ch, nullptr, nullptr,
                                             MDN_FLAG_DEVICE_TRACES | MDN_FLAG_COLUMN_MAJOR, &proof));
            return detail::to_output(proof);
        }
        detail::Lowered low(ps_->statement);
        std::vector<mdn_matrix> mats;
        for (const RowMajorMatrix& t : ps_->traces) mats.push_back(t.raw());
        detail::AuxCall ctx{ps_, &aux_};
        int rc = mdn_prove(config_.session(), &low.st, mats.data(), ch, aux_ ? &detail::AuxCall::call : nullptr, &ctx, 0, &proof);
        detail::check(config_, rc);
        return detail::to_output(proof);
    }
private:
    static void check_presence(const Statement& s, const Preprocessed* preprocessed) {
        bool expected = false;
        for (const Air& a : s.airs) expected |= a.preprocessed_width > 0;
        if (expected != (preprocessed != nullptr)) throw ProverError(ProverError::Instance, "preprocessed presence mismatch");
    }
    const StarkConfig& config_;
    const ProverStatement* ps_ = nullptr; AuxBuilder aux_;
    const DeviceProverStatement* dps_ = nullptr; DeviceAuxBuilder dev_aux_;
};

}  // namespace miden
