//! `extern "C"` view of `include/miden_b200.h` (the C ABI of the backend).  Layouts are asserted at start-up against
//! `mdn_abi_layout` (see [`check_layout`]), so a header change cannot silently desynchronise the binding.
//!
//! `Felt` is `#[repr(transparent)]` over p3 `Goldilocks`, itself a canonical `u64`
//! (reference crates/field/src/native/mod.rs:58), so `RowMajorMatrix<Felt>::values.as_ptr() as *const u64` is the
//! `MdnMatrix.values` pointer without a copy; `QuadFelt` flattens to two `u64` (c0, c1) exactly as `flatten_to_base`
//! does (crates/lifted-stark/src/prover/mod.rs:403-409).
#![allow(non_camel_case_types)]

use core::ffi::{c_char, c_int, c_longlong, c_void};

pub const MDN_OK: c_int = 0;
pub const MDN_ERR_INVALID_ARG: c_int = -1;
pub const MDN_ERR_DOMAIN: c_int = -2;
pub const MDN_ERR_CUDA: c_int = -3;
pub const MDN_ERR_UNSUPPORTED: c_int = -4;
pub const MDN_ERR_AUX_BUILDER: c_int = -5;
pub const MDN_ERR_NO_DEVICE: c_int = -6;
pub const MDN_ERR_EXTERNAL_ASSERTION: c_int = -7;
/// The constraint guard refused the proof (`mdn_session_set_constraint_guard`); `mdn_last_constraint_report` has the report.
pub const MDN_ERR_CONSTRAINT_VIOLATED: c_int = -8;
pub const MDN_FLAG_DEVICE_TRACES: u32 = 1;
/// With `MDN_FLAG_DEVICE_TRACES` only: the device matrices are column-major, entry (r, c) at `values[(c << log_height) | r]`.
pub const MDN_FLAG_COLUMN_MAJOR: u32 = 2;

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct MdnPcsParams {
    pub log_blowup: u32,
    pub log_folding_arity: u32,
    pub log_final_degree: u32,
    pub folding_pow_bits: u32,
    pub deep_pow_bits: u32,
    pub num_queries: u32,
    pub query_pow_bits: u32,
}

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct MdnChallenger {
    pub sponge_state: [u64; 12],
    pub input_buffer: [u64; 8],
    pub input_len: u32,
    pub output_len: u32,
}

/// A lowered `LookupAir` (include/miden_b200.h `mdn_lookup`).  Its nodes may read PREPROCESSED (op 15) when the AIR
/// declares preprocessed columns: from the installed bundle in a proof and in the three lookup checks, from the call's
/// `preprocessed` argument in `mdn_check_constraints` / `mdn_constraint_census`.
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct MdnLookup {
    pub num_columns: u32,
    pub program_words: u32,
    pub program: *const u32,
}

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct MdnAir {
    pub width: u32,
    pub aux_width: u32,
    pub num_aux_values: u32,
    pub num_randomness: u32,
    pub log_quotient_degree: u32,
    pub program_words: u32,
    pub program: *const u32,
    pub periodic_values: *const u64,
    pub num_periodic_columns: u32,
    pub log_max_period: u32,
    pub preprocessed_width: u32,
    pub lookup: *const MdnLookup,
}

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct MdnMatrix {
    pub values: *const u64,
    pub log_height: u32,
    pub width: u32,
}

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct MdnStatement {
    pub airs: *const MdnAir,
    pub n_airs: u32,
    pub public_values: *const u64,
    pub n_public_values: u32,
    pub observe_felts: *const u64,
    pub n_observe_felts: u32,
}

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct MdnProof {
    pub log_trace_heights: *const u8,
    pub n_heights: usize,
    pub fields: *const u64,
    pub n_fields: usize,
    pub commitments: *const u64,
    pub n_commitments: usize,
}

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct MdnTimings {
    pub h2d_transpose: f32,
    pub commit_main: f32,
    pub commit_aux: f32,
    pub evaluate_constraints: f32,
    pub commit_quotient: f32,
    pub open: f32,
    pub total: f32,
    pub lde_main: f32,
    pub hash_main: f32,
    pub kernel_ms: [f32; 10],
    pub kernel_regions: [u32; 10],
    pub kernel_launches: u64,
    pub permutations: u64,
    pub leaf_hash_bytes: f64,
    pub ntt_bytes: f64,
}

/// `LiftedAir::build_aux_trace` trampoline (`mdn_aux_builder`).
pub type MdnAuxBuilder = Option<
    unsafe extern "C" fn(
        ctx: *mut c_void,
        instance: u32,
        main: *const MdnMatrix,
        randomness: *const u64,
        aux_out: *mut u64,
        aux_values: *mut u64,
    ) -> c_int,
>;
/// `mdn_aux_builder_device`: the aux trace of a column-major device-trace call, written into `aux_out` (device,
/// column-major) with work enqueued on `stream` (the session's `cudaStream_t`).
pub type MdnAuxBuilderDevice = Option<
    unsafe extern "C" fn(
        ctx: *mut c_void,
        instance: u32,
        main: *const MdnMatrix,
        randomness: *const u64,
        aux_out: *mut u64,
        aux_values: *mut u64,
        stream: *mut c_void,
    ) -> c_int,
>;
/// Bootstrap transport of a proof split over several GPUs (`mdn_allgather_fn`).
pub type MdnAllgather =
    Option<unsafe extern "C" fn(ctx: *mut c_void, send: *const u64, recv: *mut u64, n_u64: usize) -> c_int>;
/// `Statement::eval_external` trampoline (`mdn_external_check`).
pub type MdnExternalCheck = Option<
    unsafe extern "C" fn(
        ctx: *mut c_void,
        challenges: *const u64,
        n_challenges: u32,
        aux_values: *const *const u64,
        n_aux_values: *const u32,
        log_trace_heights: *const u8,
        n_airs: u32,
        failed_assertion: *mut u32,
    ) -> c_int,
>;

/// `mdn_constraint_report`: the outcome of `mdn_check_constraints` (48 bytes).
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct MdnConstraintReport {
    /// 1: every constraint is zero on every row and every external assertion is zero
    pub holds: u32,
    /// 0 none, 1 AIR constraint, 2 external assertion
    pub kind: u32,
    /// kind 1: AIR index in instance order
    pub instance: u32,
    /// kind 1: emission index in the AIR's program; kind 2: assertion index
    pub constraint: u32,
    pub row: u64,
    /// kind 1: (c0, c1) of that constraint at that row
    pub value: [u64; 2],
    pub failing_rows: u64,
}

/// `mdn_unmatched` (include/miden_b200.h): a denominator whose multiplicities do not sum to zero, with its least push.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct MdnUnmatched {
    pub denom: [u64; 2],
    pub net_multiplicity: u64,
    pub n_pushes: u64,
    /// u64::MAX for a boundary emission
    pub first_row: u64,
    /// 0xFFFFFFFF for a boundary emission
    pub first_instance: u32,
    /// interaction index in the AIR's lookup program; boundary: index in the boundary list
    pub first_interaction: u32,
}

/// `mdn_balance_push`: one push of an unmatched denominator.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct MdnBalancePush {
    pub row: u64,
    pub multiplicity: u64,
    pub instance: u32,
    pub column: u32,
    pub interaction: u32,
    pub reserved: u32,
}

/// `mdn_mutex_violation`: more than one site of a cached-encoding group active on one row.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct MdnMutexViolation {
    pub row: u64,
    pub instance: u32,
    pub column: u32,
    pub group: u32,
    pub active_flags: u32,
}

/// `mdn_balance_report`: the outcome of `mdn_check_trace_balance`; the arrays belong to the session.
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct MdnBalanceReport {
    pub holds: u32,
    pub contributions_complete: u32,
    pub n_pushes: u64,
    pub n_denominators: u64,
    pub n_unmatched: u64,
    pub n_mutex_violations: u64,
    pub n_contributions: u64,
    pub n_skipped_airs: u32,
    pub reserved: u32,
    pub unmatched: *const MdnUnmatched,
    pub contributions: *const MdnBalancePush,
    pub mutex_violations: *const MdnMutexViolation,
    pub n_mutex_listed: u64,
}

/// `mdn_constraint_failure`: constraint `constraint` of instance `instance` is non-zero at `row`.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct MdnConstraintFailure {
    pub instance: u32,
    pub constraint: u32,
    pub row: u64,
    pub value: [u64; 2],
}

/// `mdn_constraint_tally`: one (instance, constraint) that is non-zero on at least one row.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct MdnConstraintTally {
    pub instance: u32,
    pub constraint: u32,
    pub failing_rows: u64,
    pub first_row: u64,
    pub last_row: u64,
    pub first_value: [u64; 2],
}

/// `mdn_constraint_census_report`: the counts of `mdn_constraint_census`; `first` is what `mdn_check_constraints` reports.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct MdnConstraintCensus {
    pub first: MdnConstraintReport,
    pub violations: u64,
    pub n_failures: u64,
    pub failing_constraints: u64,
    pub n_tallies: u64,
}

/// `mdn_fold_report`: the outcome of `mdn_check_lookup_folds` (kind 1 fraction column, 2 accumulator, 3 zero U).
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct MdnFoldReport {
    pub holds: u32,
    pub kind: u32,
    pub instance: u32,
    pub column: u32,
    pub row: u64,
    pub fold: [u64; 4],
    pub expected: [u64; 2],
    pub actual: [u64; 2],
    pub failing_rows: u64,
    pub zero_u: u64,
    pub n_skipped_airs: u32,
    pub reserved: u32,
}

/// `mdn_fold_failure`: one (instance, row, column) where the aux trace departs from the fold (kind as `MdnFoldReport`).
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct MdnFoldFailure {
    pub instance: u32,
    pub column: u32,
    pub kind: u32,
    pub reserved: u32,
    pub row: u64,
    pub fold: [u64; 4],
    pub expected: [u64; 2],
    pub actual: [u64; 2],
}

/// `mdn_fold_tally`: one (instance, column) that disagrees on at least one row.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct MdnFoldTally {
    pub instance: u32,
    pub column: u32,
    pub failing_rows: u64,
    pub zero_u_rows: u64,
    pub first_row: u64,
    pub last_row: u64,
    pub first_kind: u32,
    pub reserved: u32,
    pub first_expected: [u64; 2],
    pub first_actual: [u64; 2],
}

/// `mdn_fold_census_report`: the counts of `mdn_lookup_fold_census`; `first` is what `mdn_check_lookup_folds` reports.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct MdnFoldCensus {
    pub first: MdnFoldReport,
    pub disagreements: u64,
    pub n_failures: u64,
    pub failing_columns: u64,
    pub n_tallies: u64,
}

pub enum MdnSession {}

/// `mdn_hash_kind` (include/miden_b200.h): which `miden_air::config` constructor the session follows.
#[repr(C)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum HashKind {
    Poseidon2 = 0,
    Blake3 = 1,
    Keccak = 2,
    /// `rpo_config`: the duplex challenger passed to `prove` must be built over `RpoPermutation256`
    Rpo = 3,
    /// `rpx_config`
    Rpx = 4,
}

/// `mdn_hash_challenger`: p3 `HashChallenger<u8, H, 32>`'s two buffers.
#[repr(C)]
pub struct MdnHashChallenger {
    pub input_buffer: *const u8,
    pub input_len: usize,
    pub output_buffer: *const u8,
    pub output_len: usize,
}

unsafe extern "C" {
    pub fn mdn_session_create(params: *const MdnPcsParams, cuda_device: c_int, out: *mut *mut MdnSession) -> c_int;
    pub fn mdn_session_destroy(s: *mut MdnSession);
    pub fn mdn_last_error(s: *const MdnSession) -> *const c_char;
    pub fn mdn_prove(
        s: *mut MdnSession,
        st: *const MdnStatement,
        traces: *const MdnMatrix,
        challenger: *const MdnChallenger,
        build_aux: MdnAuxBuilder,
        aux_ctx: *mut c_void,
        flags: u32,
        out: *mut MdnProof,
    ) -> c_int;
    pub fn mdn_prove_begin(
        s: *mut MdnSession,
        st: *const MdnStatement,
        traces: *const MdnMatrix,
        challenger: *const MdnChallenger,
        flags: u32,
        main_root: *mut u64,
        randomness_out: *mut u64,
    ) -> c_int;
    pub fn mdn_prove_commit_aux(
        s: *mut MdnSession,
        aux: *const MdnMatrix,
        aux_values: *const *const u64,
        aux_root: *mut u64,
    ) -> c_int;
    pub fn mdn_prove_finish(s: *mut MdnSession, out: *mut MdnProof) -> c_int;
    pub fn mdn_check_constraints(
        s: *mut MdnSession,
        st: *const MdnStatement,
        traces: *const MdnMatrix,
        preprocessed: *const MdnMatrix,
        challenger: *const MdnChallenger,
        build_aux: MdnAuxBuilder,
        aux_ctx: *mut c_void,
        flags: u32,
        randomness_out: *mut u64,
        out: *mut MdnConstraintReport,
    ) -> c_int;
    /// Declared only; like the rest of the crate, not compiled yet.
    pub fn mdn_constraint_census(
        s: *mut MdnSession,
        st: *const MdnStatement,
        traces: *const MdnMatrix,
        preprocessed: *const MdnMatrix,
        challenger: *const MdnChallenger,
        build_aux: MdnAuxBuilder,
        aux_ctx: *mut c_void,
        flags: u32,
        randomness_out: *mut u64,
        failures: *mut MdnConstraintFailure,
        max_failures: u64,
        tallies: *mut MdnConstraintTally,
        max_tallies: u64,
        out: *mut MdnConstraintCensus,
    ) -> c_int;
    pub fn mdn_check_trace_balance(
        s: *mut MdnSession,
        st: *const MdnStatement,
        traces: *const MdnMatrix,
        randomness: *const u64,
        boundary: *const u64,
        n_boundary: usize,
        mutex_sites: *const *const u32,
        max_contributions: u64,
        flags: u32,
        out: *mut MdnBalanceReport,
    ) -> c_int;
    pub fn mdn_check_lookup_folds(
        s: *mut MdnSession,
        st: *const MdnStatement,
        traces: *const MdnMatrix,
        randomness: *const u64,
        fold_marks: *const *const u32,
        aux: *const MdnMatrix,
        aux_finals: *const *const u64,
        folds_out: *const *mut u64,
        flags: u32,
        out: *mut MdnFoldReport,
    ) -> c_int;
    /// Declared only; like the rest of the crate, not compiled yet.
    pub fn mdn_lookup_fold_census(
        s: *mut MdnSession,
        st: *const MdnStatement,
        traces: *const MdnMatrix,
        randomness: *const u64,
        fold_marks: *const *const u32,
        aux: *const MdnMatrix,
        aux_finals: *const *const u64,
        flags: u32,
        failures: *mut MdnFoldFailure,
        max_failures: u64,
        tallies: *mut MdnFoldTally,
        max_tallies: u64,
        out: *mut MdnFoldCensus,
    ) -> c_int;
    pub fn mdn_session_set_preprocessed(
        s: *mut MdnSession,
        st: *const MdnStatement,
        preprocessed: *const MdnMatrix,
        commitment_out: *mut u64,
    ) -> c_int;
    pub fn mdn_session_set_shard(s: *mut MdnSession, rank: u32, world: u32, f: MdnAllgather, ctx: *mut c_void) -> c_int;
    pub fn mdn_session_set_external_check(s: *mut MdnSession, f: MdnExternalCheck, ctx: *mut c_void) -> c_int;
    /// 1: every later proof checks every constraint on every row with the proof's own challenges and returns
    /// `MDN_ERR_CONSTRAINT_VIOLATED` instead of proving a statement that does not hold; 0 (default): off.
    pub fn mdn_session_set_constraint_guard(s: *mut MdnSession, enable: u32) -> c_int;
    /// The report of the last guard run (`holds = 1`, `kind = 0` before any refusal and after a guard run that passed).
    pub fn mdn_last_constraint_report(s: *const MdnSession, out: *mut MdnConstraintReport) -> c_int;
    pub fn mdn_session_set_device_aux_builder(s: *mut MdnSession, f: MdnAuxBuilderDevice, ctx: *mut c_void) -> c_int;
    pub fn mdn_session_set_hash(s: *mut MdnSession, kind: c_int) -> c_int;
    pub fn mdn_session_set_hash_challenger(s: *mut MdnSession, c: *const MdnHashChallenger) -> c_int;
    pub fn mdn_session_set_jit(s: *mut MdnSession, min_nodes: u32) -> c_int;
    pub fn mdn_jit_compile_check(program: *const u32, program_words: u32, err: *mut *const c_char) -> c_longlong;
    pub fn mdn_get_timings(s: *mut MdnSession, out: *mut MdnTimings) -> c_int;
    pub fn mdn_abi_layout(out: *mut u32, cap: usize) -> usize;
}

/// Compare this file's `#[repr(C)]` layouts with the library's own `sizeof` / `offsetof` table.
pub fn check_layout() -> Result<(), String> {
    use core::mem::{offset_of, size_of};
    let mine: [u32; 14] = [
        size_of::<MdnPcsParams>() as u32,
        size_of::<MdnChallenger>() as u32,
        size_of::<MdnLookup>() as u32,
        size_of::<MdnAir>() as u32,
        offset_of!(MdnAir, program) as u32,
        offset_of!(MdnAir, periodic_values) as u32,
        offset_of!(MdnAir, preprocessed_width) as u32,
        offset_of!(MdnAir, lookup) as u32,
        size_of::<MdnMatrix>() as u32,
        size_of::<MdnStatement>() as u32,
        size_of::<MdnProof>() as u32,
        size_of::<MdnTimings>() as u32,
        offset_of!(MdnTimings, kernel_ms) as u32,
        offset_of!(MdnTimings, permutations) as u32,
    ];
    let mut theirs = [0u32; 14];
    let n = unsafe { mdn_abi_layout(theirs.as_mut_ptr(), theirs.len()) };
    if n != mine.len() || mine != theirs {
        return Err(format!("libmiden_b200 ABI layout mismatch: binding {mine:?}, library {theirs:?}"));
    }
    Ok(())
}
