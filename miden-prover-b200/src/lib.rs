//! `miden-prover-b200`: the H100 (sm_90a) STARK proving backend behind `miden_prover::prove_stark`.
//!
//! Drop-in point (reference prover/src/lib.rs:317-355): everything `prove_stark` does before and after the call
//!
//! ```text
//! ProverInstance::new(config, &prover_statement, None)?.prove(challenger)?      // prover/src/lib.rs:341-345
//! ```
//!
//! stays on the Rust side -- challenger seeding (`config.challenger()`, `observe_protocol_params`), `Statement` /
//! `ProverStatement` construction and validation, wincode serialisation of the proof -- and the call itself
//! (crates/lifted-stark/src/prover/mod.rs:230-578) is replaced by [`GpuStarkProver::prove`], which hands the traces,
//! the lowered AIRs and the challenger state to `mdn_prove` (include/miden_b200.h) and rebuilds the proof streams.
//!
//! What this crate adds on the Rust side:
//!   * [`lower::lower_air`]      -- `air.eval()` captured once per AIR with the `SymbolicAirBuilder` and flattened to
//!                                  the device op-list (the same capture the ACE codegen uses);
//!   * [`lookup::lower_lookup`]  -- `LookupAir::eval` recorded so that the LogUp aux trace is built on the device;
//!   * [`RecordingObserver`]     -- what `Statement::observe` absorbs, as a plain `Vec<Felt>` for `mdn_statement`;
//!   * the aux-builder and `eval_external` trampolines for AIRs / statements that keep host callbacks;
//!   * [`GpuSession`]            -- owns `mdn_session`, one per CUDA device; `set_shard` splits ONE proof over the GPUs
//!                                  of a box.
//!
//! NOT COMPILED in this repository: the build image has no Rust toolchain and no network.  The code is written against
//! the reference sources as read (workspace v0.28.0 @ db4fd2f6; file:line citations inline); the C side it binds to is
//! tested through the identical ctypes and C++ bindings (tests/test_abi.py, tests/cpp/test_host_api.cpp).

pub mod ffi;
pub mod lookup;
pub mod lower;

use core::ffi::{c_int, c_void};
use std::{ffi::CStr, ptr};

use miden_air::config::MidenStarkConfig;
use miden_core::{Felt, field::{BasedVectorSpace, PrimeCharacteristicRing, PrimeField64, QuadFelt}};
use miden_crypto::stark::{
    air::{LiftedAir, MultiAir, ProverStatement},
    challenger::{CanObserve, DuplexChallenger},
    matrix::{Matrix, dense::RowMajorMatrix},
    transcript::TranscriptData,
};
use miden_processor::ExecutionError;
use serde::Serialize;

use crate::{ffi::*, lower::LoweredAir};

// SESSION
// ================================================================================================

/// `StarkConfig` on the device: PCS parameters + one CUDA device (include/miden_b200.h `mdn_session`).
/// Not `Sync`: a session serves one proof at a time; create one per GPU (sessions are independent).
pub struct GpuSession {
    raw: *mut MdnSession,
}
unsafe impl Send for GpuSession {}

impl GpuSession {
    /// `params` = `miden_air::config::pcs_params()` (air/src/config.rs:55-81) for Miden proofs.
    pub fn new(params: MdnPcsParams, cuda_device: i32) -> Result<Self, ExecutionError> {
        check_layout().map_err(ExecutionError::ProvingError)?;
        let mut raw = ptr::null_mut();
        let rc = unsafe { mdn_session_create(&params, cuda_device as c_int, &mut raw) };
        if rc != MDN_OK {
            return Err(ExecutionError::ProvingError(last_error(ptr::null())));
        }
        Ok(Self { raw })
    }

    /// The Miden production parameters (air/src/config.rs:55-67).
    pub fn miden(cuda_device: i32) -> Result<Self, ExecutionError> {
        use miden_air::config::{DEEP_POW_BITS, FOLDING_POW_BITS, LOG_BLOWUP, LOG_FINAL_DEGREE, LOG_FOLDING_ARITY, NUM_QUERIES, QUERY_POW_BITS};
        Self::new(
            MdnPcsParams {
                log_blowup: LOG_BLOWUP as u32,
                log_folding_arity: LOG_FOLDING_ARITY as u32,
                log_final_degree: LOG_FINAL_DEGREE as u32,
                folding_pow_bits: FOLDING_POW_BITS as u32,
                deep_pow_bits: DEEP_POW_BITS as u32,
                num_queries: NUM_QUERIES as u32,
                query_pow_bits: QUERY_POW_BITS as u32,
            },
            cuda_device,
        )
    }

    /// Switch the session to another of the reference's STARK hash configurations (`miden_air::config`): `input_buffer` is
    /// the `HashChallenger`'s input buffer after `config.challenger()` + `observe_protocol_params` (32 bytes of relation
    /// digest + 8 parameter felts as little-endian u64); ignored for the algebraic configurations ([`HashKind::Poseidon2`],
    /// [`HashKind::Rpo`], [`HashKind::Rpx`]), whose duplex challenger -- built over the matching permutation -- is
    /// the argument of [`GpuStarkProver::prove`].
    pub fn set_hash(&mut self, kind: HashKind, input_buffer: &[u8]) -> Result<(), ExecutionError> {
        let rc = unsafe { mdn_session_set_hash(self.raw, kind as c_int) };
        if rc != MDN_OK {
            return Err(ExecutionError::ProvingError(last_error(self.raw)));
        }
        if matches!(kind, HashKind::Blake3 | HashKind::Keccak) {
            let hc = MdnHashChallenger { input_buffer: input_buffer.as_ptr(), input_len: input_buffer.len(), output_buffer: ptr::null(), output_len: 0 };
            let rc = unsafe { mdn_session_set_hash_challenger(self.raw, &hc) };
            if rc != MDN_OK {
                return Err(ExecutionError::ProvingError(last_error(self.raw)));
            }
        }
        Ok(())
    }

    /// Split every proof of this session over `world` processes (one per GPU of an NVLink box): every rank calls
    /// [`GpuStarkProver::prove`] with the same statement and traces and gets the byte-identical proof.  `allgather`
    /// is only the bootstrap transport of the CUDA IPC handles (64 bytes per rank when a proof arena slab is created);
    /// the proof data itself moves as peer-memory stores inside the kernels.  Collective.
    ///
    /// # Safety
    /// `allgather` / `ctx` must stay valid for the lifetime of the session.
    pub unsafe fn set_shard(&mut self, rank: u32, world: u32, allgather: MdnAllgather, ctx: *mut c_void) -> Result<(), ExecutionError> {
        let rc = unsafe { mdn_session_set_shard(self.raw, rank, world, allgather, ctx) };
        if rc != MDN_OK { Err(ExecutionError::ProvingError(last_error(self.raw))) } else { Ok(()) }
    }

    /// Per-phase device timings of the last proof (names follow the reference's tracing spans, prover/mod.rs:339-561).
    pub fn timings(&self) -> MdnTimings {
        let mut t = MdnTimings::default();
        unsafe { mdn_get_timings(self.raw, &mut t) };
        t
    }
}

impl Drop for GpuSession {
    fn drop(&mut self) {
        unsafe { mdn_session_destroy(self.raw) }
    }
}

fn last_error(s: *const MdnSession) -> String {
    unsafe { CStr::from_ptr(mdn_last_error(s)) }.to_string_lossy().into_owned()
}

// STATEMENT BINDING
// ================================================================================================

/// `CanObserve<Felt>` that records: `Statement::observe(&mut rec, heights)` (crates/lifted-air/src/statement.rs:216,
/// for Miden air/src/lib.rs:817-847) leaves exactly the felts `mdn_statement.observe_felts` must carry; the backend
/// absorbs them, then the instance count and the heights, as the reference does (prover/mod.rs:290-291).
#[derive(Default)]
pub struct RecordingObserver {
    pub felts: Vec<Felt>,
}
impl CanObserve<Felt> for RecordingObserver {
    fn observe(&mut self, value: Felt) {
        self.felts.push(value);
    }
}

/// `DuplexChallenger`'s public fields (air/src/config.rs:264-271) -> `mdn_challenger`.  `output_len` counts the unread
/// rate elements: p3 pops from the back of `output_buffer`, the C side reads `sponge_state[output_len - 1]`.
pub fn challenger_state<P>(ch: &DuplexChallenger<Felt, P, 12, 8>) -> MdnChallenger {
    let mut out = MdnChallenger { sponge_state: [0; 12], input_buffer: [0; 8], input_len: 0, output_len: 0 };
    for (d, s) in out.sponge_state.iter_mut().zip(ch.sponge_state.iter()) {
        *d = s.as_canonical_u64();
    }
    for (d, s) in out.input_buffer.iter_mut().zip(ch.input_buffer.iter()) {
        *d = s.as_canonical_u64();
    }
    out.input_len = ch.input_buffer.len() as u32;
    out.output_len = ch.output_buffer.len() as u32;
    out
}

// THE PROVER
// ================================================================================================

/// AIRs lowered once (they depend on the AIR definitions only) + the session.
pub struct GpuStarkProver<'s> {
    session: &'s mut GpuSession,
    lowered: Vec<LoweredAir>,
    /// per AIR: the lowered LookupAir (`mdn_lookup`), when the aux trace is to be built on the device
    lookups: Vec<Option<(u32, Vec<u32>)>>,
}

/// Context of the two host callbacks for the duration of one `mdn_prove`.
struct CallbackCtx<'a, MA: MultiAir<Felt, QuadFelt>> {
    statement: &'a ProverStatement<Felt, QuadFelt, MA>,
}

impl<'s> GpuStarkProver<'s> {
    /// Lower every AIR of `multi_air` (instance order).  `lookups[i] = Some(..)` (from [`lookup::lower_lookup`]) moves
    /// AIR i's aux build to the device; `None` keeps `build_aux_trace` on the host (callback).
    pub fn new<MA>(session: &'s mut GpuSession, multi_air: &MA, lookups: Vec<Option<(u32, Vec<u32>)>>) -> Self
    where
        MA: MultiAir<Felt, QuadFelt>,
    {
        let lowered: Vec<LoweredAir> = multi_air.airs().iter().map(lower::lower_air).collect();
        assert_eq!(lookups.len(), lowered.len());
        Self { session, lowered, lookups }
    }

    /// `ProverInstance::new(config, statement, None)?.prove(challenger)` on the device; returns the wincode bytes
    /// `prove_stark` returns (prover/src/lib.rs:347-354).
    ///
    /// `challenger` is the caller's pre-bound challenger (`config.challenger()` + `observe_protocol_params`,
    /// prover/src/lib.rs:329-330).
    pub fn prove<MA, P>(
        &mut self,
        statement: &ProverStatement<Felt, QuadFelt, MA>,
        challenger: &DuplexChallenger<Felt, P, 12, 8>,
    ) -> Result<Vec<u8>, ExecutionError>
    where
        MA: MultiAir<Felt, QuadFelt>,
    {
        let ch = challenger_state(challenger);
        let raw = self.prove_raw(statement, Some(&ch))?;
        // StarkProofData { log_trace_heights, transcript: TranscriptData { fields, commitments } }
        // (crates/lifted-stark/src/proof.rs:57-63; crates/stark-transcript/src/data.rs:11-15).  Its fields are
        // crate-private, so the bytes are produced from a mirror with the identical serde shape and the same wincode
        // configuration prove_stark uses; a `StarkProofData::from_parts` in lifted-stark would make this a move.
        let commitments: Vec<[Felt; 4]> = raw.commitments.iter().map(|c| c.map(Felt::new_unchecked)).collect();
        let wire = ProofWire { log_trace_heights: raw.log_trace_heights, transcript: TranscriptData::new(raw.fields, commitments) };
        serialize_wire(&wire)
    }

    /// The Blake3_256 configuration (`HashFunction::Blake3_256`, air/src/config.rs:276-307) after
    /// `session.set_hash(HashKind::Blake3, &input_buffer)`: commitments are `[u8; 32]`, the four little-endian u64 of a digest.
    pub fn prove_blake3<MA: MultiAir<Felt, QuadFelt>>(&mut self, statement: &ProverStatement<Felt, QuadFelt, MA>) -> Result<Vec<u8>, ExecutionError> {
        let raw = self.prove_raw(statement, None)?;
        let commitments: Vec<[u8; 32]> = raw
            .commitments
            .iter()
            .map(|c| {
                let mut b = [0u8; 32];
                for (i, w) in c.iter().enumerate() {
                    b[8 * i..8 * i + 8].copy_from_slice(&w.to_le_bytes());
                }
                b
            })
            .collect();
        serialize_wire(&ProofWireBytes { log_trace_heights: raw.log_trace_heights, transcript: TranscriptData::new(raw.fields, commitments) })
    }

    /// The Keccak configuration (`HashFunction::Keccak`, air/src/config.rs:309-353) after
    /// `session.set_hash(HashKind::Keccak, &input_buffer)`: commitments are `[u64; 4]` lanes.
    pub fn prove_keccak<MA: MultiAir<Felt, QuadFelt>>(&mut self, statement: &ProverStatement<Felt, QuadFelt, MA>) -> Result<Vec<u8>, ExecutionError> {
        let raw = self.prove_raw(statement, None)?;
        serialize_wire(&ProofWireLanes { log_trace_heights: raw.log_trace_heights, transcript: TranscriptData::new(raw.fields, raw.commitments) })
    }

    /// One proof on the device, hash-configuration agnostic: `challenger` is the duplex state for Poseidon2 and `None` for
    /// the byte-oriented configurations, whose pre-bound `HashChallenger` was installed with [`GpuSession::set_hash`].
    fn prove_raw<MA>(
        &mut self,
        statement: &ProverStatement<Felt, QuadFelt, MA>,
        challenger: Option<&MdnChallenger>,
    ) -> Result<RawProof, ExecutionError>
    where
        MA: MultiAir<Felt, QuadFelt>,
    {
        let traces: &[RowMajorMatrix<Felt>] = statement.traces();
        let st = statement.statement();
        let k = traces.len();
        let log_heights: Vec<u8> = traces.iter().map(|t| t.height().trailing_zeros() as u8).collect();

        // (a) AIR descriptors: pointers into `self.lowered` / `self.lookups`, alive for the call
        let lookup_structs: Vec<Option<MdnLookup>> = self
            .lookups
            .iter()
            .map(|l| l.as_ref().map(|(n, prog)| MdnLookup { num_columns: *n, program_words: prog.len() as u32, program: prog.as_ptr() }))
            .collect();
        let airs: Vec<MdnAir> = self
            .lowered
            .iter()
            .zip(&lookup_structs)
            .map(|(a, lk)| MdnAir {
                width: a.width,
                aux_width: a.aux_width,
                num_aux_values: a.num_aux_values,
                num_randomness: a.num_randomness,
                log_quotient_degree: a.log_quotient_degree,
                program_words: a.program.len() as u32,
                program: a.program.as_ptr(),
                periodic_values: if a.periodic_values.is_empty() { ptr::null() } else { a.periodic_values.as_ptr() },
                num_periodic_columns: a.num_periodic_columns,
                log_max_period: a.log_max_period,
                preprocessed_width: a.preprocessed_width,
                lookup: lk.as_ref().map_or(ptr::null(), |l| l as *const MdnLookup),
            })
            .collect();

        // (b) the felts Statement::observe absorbs
        let mut rec = RecordingObserver::default();
        st.observe(&mut rec, &log_heights);
        let observe_felts: Vec<u64> = rec.felts.iter().map(Felt::as_canonical_u64).collect();
        let public_values: Vec<u64> = st.air_inputs().iter().map(Felt::as_canonical_u64).collect();

        // (c) traces: Felt is repr(transparent) over a canonical u64, so the matrices are passed in place.  They are
        //     pageable memory; with feature `host-register` they are pinned for the duration of the call so the H2D
        //     copy runs at DMA speed (the backend otherwise stages pageable buffers through pinned bounce buffers).
        let mats: Vec<MdnMatrix> = traces
            .iter()
            .map(|t| MdnMatrix { values: t.values.as_ptr() as *const u64, log_height: t.height().trailing_zeros(), width: t.width() as u32 })
            .collect();
        #[cfg(feature = "host-register")]
        let _pins: Vec<pin::Registration> = traces.iter().map(|t| pin::Registration::new(&t.values)).collect();

        let mdn_st = MdnStatement {
            airs: airs.as_ptr(),
            n_airs: k as u32,
            public_values: public_values.as_ptr(),
            n_public_values: public_values.len() as u32,
            observe_felts: observe_felts.as_ptr(),
            n_observe_felts: observe_felts.len() as u32,
        };
        let ch: *const MdnChallenger = challenger.map_or(ptr::null(), |c| c as *const MdnChallenger);

        // (d) host callbacks: build_aux_trace for AIRs without a lowered lookup; eval_external for the statement
        let mut ctx = CallbackCtx { statement };
        let ctx_ptr = &mut ctx as *mut CallbackCtx<'_, MA> as *mut c_void;
        // (a NULL builder would mean all-zero aux traces, testing/airs/miden.rs:84-94; the callback is simply never
        //  invoked for an AIR that ships a lookup program)
        let aux_cb: MdnAuxBuilder = Some(aux_trampoline::<MA>);
        unsafe { mdn_session_set_external_check(self.session.raw, Some(external_trampoline::<MA>), ctx_ptr) };

        let mut proof = core::mem::MaybeUninit::<MdnProof>::uninit();
        let rc = unsafe { mdn_prove(self.session.raw, &mdn_st, mats.as_ptr(), ch, aux_cb, ctx_ptr, 0, proof.as_mut_ptr()) };
        unsafe { mdn_session_set_external_check(self.session.raw, None, ptr::null_mut()) };
        if rc != MDN_OK {
            // ProverError -> ExecutionError::ProvingError(String) (prover/src/lib.rs:336-345)
            return Err(ExecutionError::ProvingError(last_error(self.session.raw)));
        }
        let proof = unsafe { proof.assume_init() };

        // (e) the proof streams, copied out of the session's buffers (valid until the next call on the session)
        let log_trace_heights = unsafe { core::slice::from_raw_parts(proof.log_trace_heights, proof.n_heights) }.to_vec();
        let fields: Vec<Felt> = unsafe { core::slice::from_raw_parts(proof.fields, proof.n_fields) }.iter().map(|&v| Felt::new_unchecked(v)).collect();
        let commitments: Vec<[u64; 4]> = unsafe { core::slice::from_raw_parts(proof.commitments, 4 * proof.n_commitments) }
            .chunks_exact(4)
            .map(|c| [c[0], c[1], c[2], c[3]])
            .collect();
        Ok(RawProof { log_trace_heights, fields, commitments })
    }

    /// `debug::check_constraints(&statement, challenger)` (crates/lifted-stark/src/debug.rs:70-214) on the device: every
    /// constraint of every AIR on every trace row, without proving.  Mirrors `ExecutionTrace::check_constraints`
    /// (processor/src/trace/mod.rs:251-278), which passes `config.challenger()` WITHOUT `observe_protocol_params`; pass
    /// the same here.  Panics with the reference's texts on the first failure.
    pub fn check_constraints<MA, P>(&mut self, statement: &ProverStatement<Felt, QuadFelt, MA>, challenger: &DuplexChallenger<Felt, P, 12, 8>)
    where
        MA: MultiAir<Felt, QuadFelt>,
    {
        let traces: &[RowMajorMatrix<Felt>] = statement.traces();
        let st = statement.statement();
        let log_heights: Vec<u8> = traces.iter().map(|t| t.height().trailing_zeros() as u8).collect();
        let lookup_structs: Vec<Option<MdnLookup>> = self
            .lookups
            .iter()
            .map(|l| l.as_ref().map(|(n, prog)| MdnLookup { num_columns: *n, program_words: prog.len() as u32, program: prog.as_ptr() }))
            .collect();
        let airs: Vec<MdnAir> = self
            .lowered
            .iter()
            .zip(&lookup_structs)
            .map(|(a, lk)| MdnAir {
                width: a.width,
                aux_width: a.aux_width,
                num_aux_values: a.num_aux_values,
                num_randomness: a.num_randomness,
                log_quotient_degree: a.log_quotient_degree,
                program_words: a.program.len() as u32,
                program: a.program.as_ptr(),
                periodic_values: if a.periodic_values.is_empty() { ptr::null() } else { a.periodic_values.as_ptr() },
                num_periodic_columns: a.num_periodic_columns,
                log_max_period: a.log_max_period,
                preprocessed_width: a.preprocessed_width,
                lookup: lk.as_ref().map_or(ptr::null(), |l| l as *const MdnLookup),
            })
            .collect();
        let mut rec = RecordingObserver::default();
        st.observe(&mut rec, &log_heights);
        let observe_felts: Vec<u64> = rec.felts.iter().map(Felt::as_canonical_u64).collect();
        let public_values: Vec<u64> = st.air_inputs().iter().map(Felt::as_canonical_u64).collect();
        let mats: Vec<MdnMatrix> = traces
            .iter()
            .map(|t| MdnMatrix { values: t.values.as_ptr() as *const u64, log_height: t.height().trailing_zeros(), width: t.width() as u32 })
            .collect();
        // BaseAir::preprocessed_trace per AIR, re-materialised as debug.rs does (width 0 where none)
        let preps: Vec<Option<RowMajorMatrix<Felt>>> = st.airs().iter().map(|a| a.preprocessed_trace()).collect();
        let prep_mats: Vec<MdnMatrix> = preps
            .iter()
            .map(|p| match p {
                Some(m) => MdnMatrix { values: m.values.as_ptr() as *const u64, log_height: m.height().trailing_zeros(), width: m.width() as u32 },
                None => MdnMatrix { values: ptr::null(), log_height: 0, width: 0 },
            })
            .collect();
        let prep_ptr = if preps.iter().any(Option::is_some) { prep_mats.as_ptr() } else { ptr::null() };
        let mdn_st = MdnStatement {
            airs: airs.as_ptr(),
            n_airs: traces.len() as u32,
            public_values: public_values.as_ptr(),
            n_public_values: public_values.len() as u32,
            observe_felts: observe_felts.as_ptr(),
            n_observe_felts: observe_felts.len() as u32,
        };
        let ch = challenger_state(challenger);
        let mut ctx = CallbackCtx { statement };
        let ctx_ptr = &mut ctx as *mut CallbackCtx<'_, MA> as *mut c_void;
        unsafe { mdn_session_set_external_check(self.session.raw, Some(external_trampoline::<MA>), ctx_ptr) };
        let mut rep = MdnConstraintReport::default();
        let rc = unsafe {
            mdn_check_constraints(self.session.raw, &mdn_st, mats.as_ptr(), prep_ptr, &ch, Some(aux_trampoline::<MA>), ctx_ptr, 0, ptr::null_mut(), &mut rep)
        };
        unsafe { mdn_session_set_external_check(self.session.raw, None, ptr::null_mut()) };
        assert_eq!(rc, MDN_OK, "check_constraints failed: {}", last_error(self.session.raw));
        match rep.kind {
            2 => panic!("external assertion {} is non-zero", rep.constraint),                            // debug.rs:117
            1 => panic!("constraint not satisfied at instance {}, row {}", rep.instance, rep.row),      // debug.rs:273-281
            _ => {}
        }
    }

    /// `check_trace_balance(air, main, periodic, publics, var_len_publics, challenges)` (air/src/lookup/debug/trace/mod.rs:169-189)
    /// on the device, jointly over every AIR with a device lookup (Miden's buses close across AIRs).  `boundary` is what the
    /// statement's `eval_boundary` emitted into a [`RecordingBoundary`]; `mutex_sites[i]` is AIR i's annotation (one word per
    /// interaction, include/miden_b200.h) and `site_names[i][k]` the `insert` name of its interaction k, which the report
    /// uses in place of the reference's `msg_repr`.  Like the rest of this crate, not compiled in this repository.
    pub fn check_trace_balance<MA>(
        &mut self,
        statement: &ProverStatement<Felt, QuadFelt, MA>,
        challenges: &[QuadFelt],
        boundary: &RecordingBoundary,
        mutex_sites: &[Option<Vec<u32>>],
        site_names: &[Vec<&'static str>],
        max_contributions: u64,
    ) -> GpuBalanceReport
    where
        MA: MultiAir<Felt, QuadFelt>,
    {
        let traces: &[RowMajorMatrix<Felt>] = statement.traces();
        let st = statement.statement();
        let lookup_structs: Vec<Option<MdnLookup>> = self
            .lookups
            .iter()
            .map(|l| l.as_ref().map(|(n, prog)| MdnLookup { num_columns: *n, program_words: prog.len() as u32, program: prog.as_ptr() }))
            .collect();
        let airs: Vec<MdnAir> = self
            .lowered
            .iter()
            .zip(&lookup_structs)
            .map(|(a, lk)| MdnAir {
                width: a.width,
                aux_width: a.aux_width,
                num_aux_values: a.num_aux_values,
                num_randomness: a.num_randomness,
                log_quotient_degree: a.log_quotient_degree,
                program_words: a.program.len() as u32,
                program: a.program.as_ptr(),
                periodic_values: if a.periodic_values.is_empty() { ptr::null() } else { a.periodic_values.as_ptr() },
                num_periodic_columns: a.num_periodic_columns,
                log_max_period: a.log_max_period,
                preprocessed_width: a.preprocessed_width,
                lookup: lk.as_ref().map_or(ptr::null(), |l| l as *const MdnLookup),
            })
            .collect();
        let public_values: Vec<u64> = st.air_inputs().iter().map(Felt::as_canonical_u64).collect();
        let mats: Vec<MdnMatrix> = traces
            .iter()
            .map(|t| MdnMatrix { values: t.values.as_ptr() as *const u64, log_height: t.height().trailing_zeros(), width: t.width() as u32 })
            .collect();
        let mdn_st = MdnStatement {
            airs: airs.as_ptr(),
            n_airs: traces.len() as u32,
            public_values: public_values.as_ptr(),
            n_public_values: public_values.len() as u32,
            observe_felts: ptr::null(),
            n_observe_felts: 0,
        };
        let ef = |q: &QuadFelt| -> [u64; 2] {
            let c = q.as_basis_coefficients_slice();
            [c[0].as_canonical_u64(), c[1].as_canonical_u64()]
        };
        let rnd: Vec<u64> = challenges.iter().flat_map(|c| ef(c)).collect();
        let bnd: Vec<u64> = boundary.emissions.iter().flat_map(|(_, d, m)| { let d = ef(d); [d[0], d[1], m.as_canonical_u64()] }).collect();
        let sites: Vec<*const u32> = (0..traces.len())
            .map(|i| mutex_sites.get(i).and_then(|m| m.as_ref()).map_or(ptr::null(), |m| m.as_ptr()))
            .collect();
        let mut rep = core::mem::MaybeUninit::<MdnBalanceReport>::zeroed();
        let rc = unsafe {
            mdn_check_trace_balance(self.session.raw, &mdn_st, mats.as_ptr(), rnd.as_ptr(), bnd.as_ptr(), boundary.emissions.len(),
                                    sites.as_ptr(), max_contributions, 0, rep.as_mut_ptr())
        };
        assert_eq!(rc, MDN_OK, "check_trace_balance failed: {}", last_error(self.session.raw));
        let rep = unsafe { rep.assume_init() };
        // interaction index -> insert name; boundary emissions keep their eval_boundary name
        let name = |inst: u32, k: u32| -> String {
            if inst == u32::MAX {
                return format!("[boundary:{}]", boundary.emissions.get(k as usize).map_or("?", |e| e.0));
            }
            site_names.get(inst as usize).and_then(|n| n.get(k as usize)).map_or(format!("interaction {k}"), |s| s.to_string())
        };
        let unmatched = unsafe { core::slice::from_raw_parts(rep.unmatched, rep.n_unmatched as usize) };
        let pushes: &[MdnBalancePush] =
            if rep.contributions_complete != 0 { unsafe { core::slice::from_raw_parts(rep.contributions, rep.n_contributions as usize) } } else { &[] };
        let mut out = GpuBalanceReport::default();
        let mut c = 0usize;
        for u in unmatched {
            let n = if rep.contributions_complete != 0 { u.n_pushes as usize } else { 0 };
            let contributions = pushes[c..c + n]
                .iter()
                .map(|p| GpuPush { instance: p.instance, row: p.row, column: p.column, interaction: p.interaction, multiplicity: p.multiplicity, site: name(p.instance, p.interaction) })
                .collect();
            c += n;
            out.unmatched.push(GpuUnmatched {
                denom: u.denom,
                net_multiplicity: u.net_multiplicity,
                n_pushes: u.n_pushes,
                first: GpuPush { instance: u.first_instance, row: u.first_row, column: u32::MAX, interaction: u.first_interaction, multiplicity: 0, site: name(u.first_instance, u.first_interaction) },
                contributions,
            });
        }
        out.mutex_violations = unsafe { core::slice::from_raw_parts(rep.mutex_violations, rep.n_mutex_listed as usize) }.to_vec();
        out.n_mutex_violations = rep.n_mutex_violations;
        out
    }
}

/// A `BoundaryBuilder` that records `eval_boundary`'s emissions (name, encoded denominator, multiplicity) for
/// [`GpuStarkProver::check_trace_balance`], as the reference's `DebugBoundaryEmitter` (builder.rs:382-415) feeds its walk.
pub struct RecordingBoundary<'a> {
    pub challenges: &'a miden_air::lookup::Challenges<QuadFelt>,
    pub public_values: &'a [Felt],
    pub var_len_public_inputs: &'a [&'a [Felt]],
    pub emissions: Vec<(&'static str, QuadFelt, Felt)>,
}

impl<'a> miden_air::lookup::BoundaryBuilder for RecordingBoundary<'a> {
    type F = Felt;
    type EF = QuadFelt;
    fn public_values(&self) -> &[Felt] {
        self.public_values
    }
    fn var_len_public_inputs(&self) -> &[&[Felt]] {
        self.var_len_public_inputs
    }
    fn insert<M>(&mut self, name: &'static str, multiplicity: Felt, msg: M)
    where
        M: miden_air::lookup::LookupMessage<Felt, QuadFelt>,
    {
        self.emissions.push((name, msg.encode(self.challenges), multiplicity));
    }
}

/// One push of an unmatched denominator; `site` names its insert (or `[boundary:<name>]`).
#[derive(Clone, Debug)]
pub struct GpuPush {
    pub instance: u32,
    pub row: u64,
    pub column: u32,
    pub interaction: u32,
    pub multiplicity: u64,
    pub site: String,
}

#[derive(Clone, Debug)]
pub struct GpuUnmatched {
    pub denom: [u64; 2],
    pub net_multiplicity: u64,
    pub n_pushes: u64,
    pub first: GpuPush,
    /// every push in emission order, empty when there were more than `max_contributions` in all
    pub contributions: Vec<GpuPush>,
}

/// `BalanceReport` (air/src/lookup/debug/trace/mod.rs:84-95) as the device reports it.
#[derive(Clone, Debug, Default)]
pub struct GpuBalanceReport {
    pub unmatched: Vec<GpuUnmatched>,
    pub mutex_violations: Vec<MdnMutexViolation>,
    pub n_mutex_violations: u64,
}

impl GpuBalanceReport {
    pub fn is_ok(&self) -> bool {
        self.unmatched.is_empty() && self.n_mutex_violations == 0
    }
}

/// `StarkProofData`'s three streams as the C ABI returns them; a commitment is four u64 whatever the hash configuration.
struct RawProof {
    log_trace_heights: Vec<u8>,
    fields: Vec<Felt>,
    commitments: Vec<[u64; 4]>,
}

fn serialize_wire<T: Serialize>(wire: &T) -> Result<Vec<u8>, ExecutionError> {
    let cfg = wincode::config::Configuration::default();
    <wincode::SerdeCompat<T> as wincode::config::Serialize<_>>::serialize(wire, cfg).map_err(|e| ExecutionError::ProvingError(e.to_string()))
}

/// Serde mirror of `StarkProofData<Felt, QuadFelt, SC>` for the Poseidon2 configuration (`Commitment = [Felt; 4]`
/// digests, air/src/config.rs:204-223): same field names, order and types, hence the same wincode bytes.
#[derive(Serialize)]
struct ProofWire {
    log_trace_heights: Vec<u8>,
    transcript: TranscriptData<Felt, [Felt; 4]>,
}
/// The same for the Blake3_256 configuration (`Commitment = [u8; 32]`, air/src/config.rs:282-289) ...
#[derive(Serialize)]
struct ProofWireBytes {
    log_trace_heights: Vec<u8>,
    transcript: TranscriptData<Felt, [u8; 32]>,
}
/// ... and for the Keccak configuration (`Commitment = [u64; 4]`, air/src/config.rs:325-332).
#[derive(Serialize)]
struct ProofWireLanes {
    log_trace_heights: Vec<u8>,
    transcript: TranscriptData<Felt, [u64; 4]>,
}

// CALLBACKS
// ================================================================================================

/// `LiftedAir::build_aux_trace(main, air_inputs, aux_inputs, challenges)` for instance `instance`
/// (prover/mod.rs:357-381), EF flattened to base exactly like `flatten_to_base` (:403-409).
unsafe extern "C" fn aux_trampoline<MA: MultiAir<Felt, QuadFelt>>(
    ctx: *mut c_void,
    instance: u32,
    _main: *const MdnMatrix,
    randomness: *const u64,
    aux_out: *mut u64,
    aux_values: *mut u64,
) -> c_int {
    let result = std::panic::catch_unwind(|| {
        let ctx = unsafe { &*(ctx as *const CallbackCtx<'_, MA>) };
        let st = ctx.statement.statement();
        let air = &st.airs()[instance as usize];
        let main = &ctx.statement.traces()[instance as usize];
        let nr = air.num_randomness();
        let r = unsafe { core::slice::from_raw_parts(randomness, 2 * nr) };
        let challenges: Vec<QuadFelt> = r.chunks_exact(2).map(|c| quad(c[0], c[1])).collect();
        let (aux, values) = air.build_aux_trace(main, st.air_inputs(), st.aux_inputs(), &challenges);
        let n = main.height() * air.aux_width();
        let out = unsafe { core::slice::from_raw_parts_mut(aux_out, 2 * n) };
        for (i, e) in aux.values.iter().enumerate() {
            let c: &[Felt] = e.as_basis_coefficients_slice();
            out[2 * i] = c[0].as_canonical_u64();
            out[2 * i + 1] = c[1].as_canonical_u64();
        }
        let vals = unsafe { core::slice::from_raw_parts_mut(aux_values, 2 * air.num_aux_values()) };
        for (i, e) in values.iter().enumerate() {
            let c: &[Felt] = e.as_basis_coefficients_slice();
            vals[2 * i] = c[0].as_canonical_u64();
            vals[2 * i + 1] = c[1].as_canonical_u64();
        }
    });
    if result.is_ok() { 0 } else { 1 }
}

/// `Statement::eval_external(randomness, aux_values, log_trace_heights)` (crates/lifted-air/src/statement.rs:94-110),
/// called by the backend once the aux values exist -- including the finals of aux traces built on the device -- and
/// before the aux commitment, where the reference evaluates it (prover/mod.rs:383-395).
unsafe extern "C" fn external_trampoline<MA: MultiAir<Felt, QuadFelt>>(
    ctx: *mut c_void,
    challenges: *const u64,
    n_challenges: u32,
    aux_values: *const *const u64,
    n_aux_values: *const u32,
    log_trace_heights: *const u8,
    n_airs: u32,
    failed_assertion: *mut u32,
) -> c_int {
    let result = std::panic::catch_unwind(|| {
        let ctx = unsafe { &*(ctx as *const CallbackCtx<'_, MA>) };
        let ch = unsafe { core::slice::from_raw_parts(challenges, 2 * n_challenges as usize) };
        let randomness: Vec<QuadFelt> = ch.chunks_exact(2).map(|c| quad(c[0], c[1])).collect();
        let k = n_airs as usize;
        let ptrs = unsafe { core::slice::from_raw_parts(aux_values, k) };
        let lens = unsafe { core::slice::from_raw_parts(n_aux_values, k) };
        let owned: Vec<Vec<QuadFelt>> = (0..k)
            .map(|i| unsafe { core::slice::from_raw_parts(ptrs[i], 2 * lens[i] as usize) }.chunks_exact(2).map(|c| quad(c[0], c[1])).collect())
            .collect();
        let views: Vec<&[QuadFelt]> = owned.iter().map(Vec::as_slice).collect();
        let heights = unsafe { core::slice::from_raw_parts(log_trace_heights, k) };
        match ctx.statement.statement().eval_external(&randomness, &views, heights) {
            Err(_) => -1,                                            // ProverError::Reduction
            Ok(assertions) => match assertions.iter().position(|a| *a != QuadFelt::ZERO) {
                None => 0,
                Some(i) => {
                    unsafe { *failed_assertion = i as u32 };
                    1                                                // ProverError::ExternalAssertionFailed { assertion: i }
                },
            },
        }
    });
    result.unwrap_or(-1)
}

fn quad(c0: u64, c1: u64) -> QuadFelt {
    QuadFelt::from_basis_coefficients_slice(&[Felt::new_unchecked(c0), Felt::new_unchecked(c1)]).expect("two coefficients")
}

// PINNING
// ================================================================================================

/// `cudaHostRegister` / `cudaHostUnregister` around a proof: a Rust `Vec<Felt>` is pageable, and a pageable 0.75 GB
/// trace set is uploaded more slowly than pinned memory (tools/e2e_pageable.py times both).
#[cfg(feature = "host-register")]
mod pin {
    use core::ffi::{c_int, c_uint, c_void};
    unsafe extern "C" {
        fn cudaHostRegister(ptr: *mut c_void, size: usize, flags: c_uint) -> c_int;
        fn cudaHostUnregister(ptr: *mut c_void) -> c_int;
    }
    pub struct Registration(*mut c_void, bool);
    impl Registration {
        pub fn new<T>(v: &[T]) -> Self {
            let p = v.as_ptr() as *mut c_void;
            let ok = unsafe { cudaHostRegister(p, core::mem::size_of_val(v), 0) } == 0;
            Self(p, ok)
        }
    }
    impl Drop for Registration {
        fn drop(&mut self) {
            if self.1 {
                unsafe { cudaHostUnregister(self.0) };
            }
        }
    }
}

// THE ONE-LINE CHANGE IN `prove_stark`
// ================================================================================================

/// What `miden_prover::prove_stark` (prover/src/lib.rs:317-355) becomes for `HashFunction::Poseidon2` when this backend
/// is enabled: identical up to the `ProverInstance::prove` line.
pub fn prove_stark_b200(
    session: &mut GpuSession,
    config: &MidenStarkConfig<impl Sized, DuplexChallenger<Felt, miden_crypto::hash::poseidon2::Poseidon2Permutation256, 12, 8>>,
    core_trace: RowMajorMatrix<Felt>,
    chiplets_trace: RowMajorMatrix<Felt>,
    poseidon2_trace: RowMajorMatrix<Felt>,
    public_values: &[Felt],
    aux_inputs: &[Felt],
) -> Result<Vec<u8>, ExecutionError> {
    use miden_air::{MidenMultiAir, config};
    use miden_crypto::stark::air::Statement;

    let mut challenger = config.challenger();
    config::observe_protocol_params(&mut challenger);

    let multi_air = MidenMultiAir::new();
    // aux traces on the device: all three Miden AIRs use build_logup_aux_trace (air/src/lib.rs:671-685)
    let lookups = multi_air
        .airs()
        .iter()
        .map(|air| Some(lookup::lower_lookup(air.air_layout(), air)))
        .collect();
    let statement = Statement::new(multi_air, public_values.to_vec(), aux_inputs.to_vec())
        .map_err(|e| ExecutionError::ProvingError(e.to_string()))?;
    let prover_statement = ProverStatement::new(statement, vec![core_trace, chiplets_trace, poseidon2_trace])
        .map_err(|e| ExecutionError::ProvingError(e.to_string()))?;

    let mut prover = GpuStarkProver::new(session, prover_statement.statement().multi_air(), lookups);
    prover.prove(&prover_statement, &challenger)
}
