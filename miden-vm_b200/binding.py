"""ctypes view of include/miden_b200.h.  No fallback: importing works without the library (so the
CPU test-suite can check the header/export surface), but every compute entry point raises if
`libmiden_b200.so` cannot be loaded."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MDN_LIB_PATH") or os.path.join(HERE, "csrc", "libmiden_b200.so")   # override only for A/B kernel experiments
u64p = C.POINTER(C.c_uint64)
u32p = C.POINTER(C.c_uint32)


class PcsParams(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("log_blowup", "log_folding_arity", "log_final_degree",
                                          "folding_pow_bits", "deep_pow_bits", "num_queries", "query_pow_bits")]


class Challenger(C.Structure):
    _fields_ = [("sponge_state", C.c_uint64 * 12), ("input_buffer", C.c_uint64 * 8),
                ("input_len", C.c_uint32), ("output_len", C.c_uint32)]


class Lookup(C.Structure):
    _fields_ = [("num_columns", C.c_uint32), ("program_words", C.c_uint32), ("program", u32p)]


class Air(C.Structure):
    _fields_ = [("width", C.c_uint32), ("aux_width", C.c_uint32), ("num_aux_values", C.c_uint32),
                ("num_randomness", C.c_uint32), ("log_quotient_degree", C.c_uint32),
                ("program_words", C.c_uint32), ("program", u32p),
                ("periodic_values", u64p), ("num_periodic_columns", C.c_uint32), ("log_max_period", C.c_uint32),
                ("preprocessed_width", C.c_uint32), ("lookup", C.POINTER(Lookup))]


class HashChallenger(C.Structure):
    _fields_ = [("input_buffer", C.POINTER(C.c_uint8)), ("input_len", C.c_size_t),
                ("output_buffer", C.POINTER(C.c_uint8)), ("output_len", C.c_size_t)]


HASH_POSEIDON2, HASH_BLAKE3, HASH_KECCAK, HASH_RPO, HASH_RPX = 0, 1, 2, 3, 4
# Session.info(INFO_JIT_LOOKUP_CHECK): per AIR (instance order) of the last check_trace_balance / check_lookup_folds /
# lookup_fold_census call, 1 where the row passes ran on the NVRTC kernel, 0 on the interpreter (mdn_get_info 12)
INFO_JIT_LOOKUP_CHECK = 12


class Matrix(C.Structure):
    _fields_ = [("values", u64p), ("log_height", C.c_uint32), ("width", C.c_uint32)]


class Statement(C.Structure):
    _fields_ = [("airs", C.POINTER(Air)), ("n_airs", C.c_uint32),
                ("public_values", u64p), ("n_public_values", C.c_uint32),
                ("observe_felts", u64p), ("n_observe_felts", C.c_uint32)]


class Proof(C.Structure):
    _fields_ = [("log_trace_heights", C.POINTER(C.c_uint8)), ("n_heights", C.c_size_t),
                ("fields", u64p), ("n_fields", C.c_size_t),
                ("commitments", u64p), ("n_commitments", C.c_size_t)]


class Timings(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("h2d_transpose", "commit_main", "commit_aux", "evaluate_constraints",
                                         "commit_quotient", "open", "total", "lde_main", "hash_main")] + \
               [("kernel_ms", C.c_float * 10), ("kernel_regions", C.c_uint * 10), ("kernel_launches", C.c_ulonglong),
                ("permutations", C.c_ulonglong), ("leaf_hash_bytes", C.c_double), ("ntt_bytes", C.c_double)]


class ConstraintReport(C.Structure):
    """`mdn_constraint_report`: the outcome of mdn_check_constraints (kind 1 = AIR constraint, 2 = external assertion)."""
    _fields_ = [("holds", C.c_uint32), ("kind", C.c_uint32), ("instance", C.c_uint32), ("constraint", C.c_uint32),
                ("row", C.c_uint64), ("value", C.c_uint64 * 2), ("failing_rows", C.c_uint64)]


class ConstraintFailure(C.Structure):
    """`mdn_constraint_failure`: constraint `constraint` of instance `instance` is non-zero at `row`."""
    _fields_ = [("instance", C.c_uint32), ("constraint", C.c_uint32), ("row", C.c_uint64), ("value", C.c_uint64 * 2)]


class ConstraintTally(C.Structure):
    """`mdn_constraint_tally`: one (instance, constraint) that is non-zero on at least one row."""
    _fields_ = [("instance", C.c_uint32), ("constraint", C.c_uint32), ("failing_rows", C.c_uint64), ("first_row", C.c_uint64),
                ("last_row", C.c_uint64), ("first_value", C.c_uint64 * 2)]


class ConstraintCensus(C.Structure):
    """`mdn_constraint_census`: the counts of mdn_constraint_census; `first` is mdn_check_constraints' report."""
    _fields_ = [("first", ConstraintReport), ("violations", C.c_uint64), ("n_failures", C.c_uint64),
                ("failing_constraints", C.c_uint64), ("n_tallies", C.c_uint64)]


class Unmatched(C.Structure):
    """`mdn_unmatched`: a denominator whose multiplicities do not sum to zero, with its least push."""
    _fields_ = [("denom", C.c_uint64 * 2), ("net_multiplicity", C.c_uint64), ("n_pushes", C.c_uint64), ("first_row", C.c_uint64),
                ("first_instance", C.c_uint32), ("first_interaction", C.c_uint32)]


class BalancePush(C.Structure):
    """`mdn_balance_push`: one push of an unmatched denominator (instance / column 0xFFFFFFFF: a boundary emission)."""
    _fields_ = [("row", C.c_uint64), ("multiplicity", C.c_uint64), ("instance", C.c_uint32), ("column", C.c_uint32),
                ("interaction", C.c_uint32), ("reserved", C.c_uint32)]


class MutexViolation(C.Structure):
    _fields_ = [("row", C.c_uint64), ("instance", C.c_uint32), ("column", C.c_uint32), ("group", C.c_uint32), ("active_flags", C.c_uint32)]


class BalanceReport(C.Structure):
    """`mdn_balance_report`: the outcome of mdn_check_trace_balance.  Its arrays are owned by the session."""
    _fields_ = [("holds", C.c_uint32), ("contributions_complete", C.c_uint32), ("n_pushes", C.c_uint64),
                ("n_denominators", C.c_uint64), ("n_unmatched", C.c_uint64), ("n_mutex_violations", C.c_uint64),
                ("n_contributions", C.c_uint64), ("n_skipped_airs", C.c_uint32), ("reserved", C.c_uint32),
                ("unmatched", C.POINTER(Unmatched)), ("contributions", C.POINTER(BalancePush)),
                ("mutex_violations", C.POINTER(MutexViolation)), ("n_mutex_listed", C.c_uint64)]


class FoldReport(C.Structure):
    """`mdn_fold_report`: the outcome of mdn_check_lookup_folds (kind 1 = fraction column, 2 = accumulator, 3 = zero U)."""
    _fields_ = [("holds", C.c_uint32), ("kind", C.c_uint32), ("instance", C.c_uint32), ("column", C.c_uint32),
                ("row", C.c_uint64), ("fold", C.c_uint64 * 4), ("expected", C.c_uint64 * 2), ("actual", C.c_uint64 * 2),
                ("failing_rows", C.c_uint64), ("zero_u", C.c_uint64), ("n_skipped_airs", C.c_uint32), ("reserved", C.c_uint32)]


def fold_report_dict(rep: FoldReport) -> dict:
    """A FoldReport as plain Python values."""
    return dict(holds=rep.holds, kind=rep.kind, instance=rep.instance, column=rep.column, row=rep.row, fold=tuple(rep.fold),
                expected=tuple(rep.expected), actual=tuple(rep.actual), failing_rows=rep.failing_rows, zero_u=rep.zero_u,
                n_skipped_airs=rep.n_skipped_airs)


class FoldFailure(C.Structure):
    """`mdn_fold_failure`: one (instance, row, column) where the aux trace departs from the fold (kind as FoldReport)."""
    _fields_ = [("instance", C.c_uint32), ("column", C.c_uint32), ("kind", C.c_uint32), ("reserved", C.c_uint32),
                ("row", C.c_uint64), ("fold", C.c_uint64 * 4), ("expected", C.c_uint64 * 2), ("actual", C.c_uint64 * 2)]


class FoldTally(C.Structure):
    """`mdn_fold_tally`: one (instance, column) that disagrees on at least one row."""
    _fields_ = [("instance", C.c_uint32), ("column", C.c_uint32), ("failing_rows", C.c_uint64), ("zero_u_rows", C.c_uint64),
                ("first_row", C.c_uint64), ("last_row", C.c_uint64), ("first_kind", C.c_uint32), ("reserved", C.c_uint32),
                ("first_expected", C.c_uint64 * 2), ("first_actual", C.c_uint64 * 2)]


class FoldCensus(C.Structure):
    """`mdn_fold_census_report`: the counts of mdn_lookup_fold_census; `first` is mdn_check_lookup_folds' report."""
    _fields_ = [("first", FoldReport), ("disagreements", C.c_uint64), ("n_failures", C.c_uint64),
                ("failing_columns", C.c_uint64), ("n_tallies", C.c_uint64)]


BOUNDARY = 0xFFFFFFFF     # instance / column of a boundary emission in a balance report (row = 2^64 - 1)


def balance_report_dict(rep: BalanceReport) -> dict:
    """A BalanceReport as plain Python values (copied out of the session's memory): every field, lists of tuples
    unmatched (denom, net, n_pushes, (first instance, first row, first interaction)), contributions (instance, row,
    column, interaction, multiplicity) and mutex_violations (instance, row, column, group, active_flags)."""
    um = [((u.denom[0], u.denom[1]), u.net_multiplicity, u.n_pushes, (u.first_instance, u.first_row, u.first_interaction))
          for u in (rep.unmatched[i] for i in range(rep.n_unmatched))]
    co = [(c.instance, c.row, c.column, c.interaction, c.multiplicity)
          for c in (rep.contributions[i] for i in range(rep.n_contributions if rep.contributions_complete else 0))]
    mv = [(m.instance, m.row, m.column, m.group, m.active_flags) for m in (rep.mutex_violations[i] for i in range(rep.n_mutex_listed))]
    return dict(holds=rep.holds, contributions_complete=rep.contributions_complete, n_pushes=rep.n_pushes,
                n_denominators=rep.n_denominators, n_unmatched=rep.n_unmatched, n_mutex_violations=rep.n_mutex_violations,
                n_contributions=rep.n_contributions, n_skipped_airs=rep.n_skipped_airs, unmatched=um, contributions=co,
                mutex_violations=mv)


AUX_BUILDER = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint32, C.POINTER(Matrix), u64p, u64p, u64p)
ALLGATHER = C.CFUNCTYPE(C.c_int, C.c_void_p, u64p, u64p, C.c_size_t)
EXTERNAL_CHECK = C.CFUNCTYPE(C.c_int, C.c_void_p, u64p, C.c_uint32, C.POINTER(u64p), u32p, C.POINTER(C.c_uint8), C.c_uint32, u32p)
DEVICE_AUX_BUILDER = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint32, C.POINTER(Matrix), u64p, C.c_void_p, u64p, C.c_void_p)
FLAG_DEVICE_TRACES = 1
FLAG_COLUMN_MAJOR = 2     # with FLAG_DEVICE_TRACES: device matrices are column-major, column c at values + (c << log_height)

# Every symbol include/miden_b200.h declares (checked by tests/test_abi.py).
EXPORTS = [
    "mdn_session_create", "mdn_session_destroy", "mdn_last_error", "mdn_prove", "mdn_prove_begin",
    "mdn_prove_commit_aux", "mdn_prove_finish", "mdn_proof_serialize", "mdn_coset_lde_batch",
    "mdn_lmcs_commit", "mdn_poseidon2_permute", "mdn_get_info", "mdn_get_timings",
    "mdn_challenger_observe", "mdn_challenger_sample", "mdn_set_debug", "mdn_session_set_shard",
    "mdn_session_set_preprocessed", "mdn_session_set_jit", "mdn_jit_compile_check", "mdn_jit_status", "mdn_abi_layout",
    "mdn_session_set_external_check", "mdn_session_set_hash", "mdn_session_set_hash_challenger",
    "mdn_check_constraints", "mdn_session_set_device_aux_builder", "mdn_check_trace_balance",
    "mdn_check_lookup_folds", "mdn_constraint_census", "mdn_session_set_constraint_guard", "mdn_last_constraint_report",
    "mdn_lookup_fold_census",
]
ERR_CONSTRAINT_VIOLATED = -8

_lib = None


def jit_compile_check(program: np.ndarray) -> int:
    """Lower + NVRTC-compile a constraint program without touching a device; returns the cubin size."""
    err = C.c_char_p()
    prog = np.ascontiguousarray(program, dtype=np.uint32)
    n = lib().mdn_jit_compile_check(prog.ctypes.data_as(u32p), len(prog), C.byref(err))
    if n < 0:
        raise ProverError(n, (err.value or b"").decode())
    return n


class BackendMissing(RuntimeError):
    pass


def lib():
    """Load libmiden_b200.so.  Raises BackendMissing (never falls back) when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise BackendMissing(f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(LIB_PATH)
        if hasattr(L, "mdn_emulated_build") and os.environ.get("MDN_ALLOW_EMULATOR") != "1":
            # tests/emu builds the kernels for the CPU (one fiber per CUDA thread) so that host logic can be tested
            # without a GPU; it is test infrastructure and must never stand in for the product
            raise BackendMissing(f"{LIB_PATH} is the CPU kernel emulator of tests/emu, not the CUDA backend "
                                 "(there is no CPU fallback; only tests/test_emulated.py may load it)")
        L.mdn_last_error.restype = C.c_char_p
        L.mdn_last_error.argtypes = [C.c_void_p]
        L.mdn_session_create.argtypes = [C.POINTER(PcsParams), C.c_int, C.POINTER(C.c_void_p)]
        L.mdn_session_destroy.argtypes = [C.c_void_p]
        L.mdn_prove.argtypes = [C.c_void_p, C.POINTER(Statement), C.POINTER(Matrix), C.POINTER(Challenger),
                                AUX_BUILDER, C.c_void_p, C.c_uint32, C.POINTER(Proof)]
        L.mdn_check_constraints.argtypes = [C.c_void_p, C.POINTER(Statement), C.POINTER(Matrix), C.POINTER(Matrix),
                                            C.POINTER(Challenger), AUX_BUILDER, C.c_void_p, C.c_uint32, u64p,
                                            C.POINTER(ConstraintReport)]
        L.mdn_constraint_census.argtypes = [C.c_void_p, C.POINTER(Statement), C.POINTER(Matrix), C.POINTER(Matrix),
                                            C.POINTER(Challenger), AUX_BUILDER, C.c_void_p, C.c_uint32, u64p,
                                            C.POINTER(ConstraintFailure), C.c_uint64, C.POINTER(ConstraintTally), C.c_uint64,
                                            C.POINTER(ConstraintCensus)]
        L.mdn_check_trace_balance.argtypes = [C.c_void_p, C.POINTER(Statement), C.POINTER(Matrix), u64p, u64p, C.c_size_t,
                                              C.POINTER(u32p), C.c_uint64, C.c_uint32, C.POINTER(BalanceReport)]
        L.mdn_check_lookup_folds.argtypes = [C.c_void_p, C.POINTER(Statement), C.POINTER(Matrix), u64p, C.POINTER(u32p),
                                             C.POINTER(Matrix), C.POINTER(u64p), C.POINTER(u64p), C.c_uint32,
                                             C.POINTER(FoldReport)]
        L.mdn_lookup_fold_census.argtypes = [C.c_void_p, C.POINTER(Statement), C.POINTER(Matrix), u64p, C.POINTER(u32p),
                                             C.POINTER(Matrix), C.POINTER(u64p), C.c_uint32, C.POINTER(FoldFailure), C.c_uint64,
                                             C.POINTER(FoldTally), C.c_uint64, C.POINTER(FoldCensus)]
        L.mdn_prove_begin.argtypes = [C.c_void_p, C.POINTER(Statement), C.POINTER(Matrix), C.POINTER(Challenger),
                                      C.c_uint32, u64p, u64p]
        L.mdn_prove_commit_aux.argtypes = [C.c_void_p, C.POINTER(Matrix), C.POINTER(u64p), u64p]
        L.mdn_prove_finish.argtypes = [C.c_void_p, C.POINTER(Proof)]
        L.mdn_proof_serialize.restype = C.c_size_t
        L.mdn_proof_serialize.argtypes = [C.POINTER(Proof), C.POINTER(C.c_uint8), C.c_size_t]
        L.mdn_coset_lde_batch.argtypes = [C.c_void_p, C.POINTER(Matrix), C.c_uint32, C.c_uint64, u64p]
        L.mdn_lmcs_commit.argtypes = [C.c_void_p, C.POINTER(Matrix), C.c_uint32, u64p]
        L.mdn_poseidon2_permute.argtypes = [C.c_void_p, u64p, C.c_size_t]
        L.mdn_get_info.restype = C.c_longlong
        L.mdn_get_info.argtypes = [C.c_void_p, C.c_int, u64p, C.c_size_t]
        L.mdn_set_debug.argtypes = [C.c_void_p, C.c_int]
        L.mdn_session_set_shard.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, ALLGATHER, C.c_void_p]
        L.mdn_session_set_hash.argtypes = [C.c_void_p, C.c_int]
        L.mdn_session_set_hash_challenger.argtypes = [C.c_void_p, C.POINTER(HashChallenger)]
        L.mdn_session_set_external_check.argtypes = [C.c_void_p, EXTERNAL_CHECK, C.c_void_p]
        L.mdn_session_set_device_aux_builder.argtypes = [C.c_void_p, DEVICE_AUX_BUILDER, C.c_void_p]
        L.mdn_session_set_preprocessed.argtypes = [C.c_void_p, C.POINTER(Statement), C.POINTER(Matrix), u64p]
        L.mdn_abi_layout.restype = C.c_size_t
        L.mdn_abi_layout.argtypes = [u32p, C.c_size_t]
        L.mdn_session_set_jit.argtypes = [C.c_void_p, C.c_uint32]
        L.mdn_session_set_constraint_guard.argtypes = [C.c_void_p, C.c_uint32]
        L.mdn_last_constraint_report.argtypes = [C.c_void_p, C.POINTER(ConstraintReport)]
        L.mdn_jit_status.restype = C.c_char_p
        L.mdn_jit_status.argtypes = [C.c_void_p]
        L.mdn_jit_compile_check.restype = C.c_longlong
        L.mdn_jit_compile_check.argtypes = [u32p, C.c_uint32, C.POINTER(C.c_char_p)]
        L.mdn_get_timings.argtypes = [C.c_void_p, C.POINTER(Timings)]
        L.mdn_challenger_observe.argtypes = [C.POINTER(Challenger), u64p, C.c_size_t]
        L.mdn_challenger_sample.restype = C.c_uint64
        L.mdn_challenger_sample.argtypes = [C.POINTER(Challenger)]
        _lib = L
    return _lib


def ptr(a: np.ndarray):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(u64p)


class ProverError(RuntimeError):
    """Mirrors `ExecutionError::ProvingError(String)` (reference prover/src/lib.rs:336-345)."""


class ConstraintViolation(ProverError):
    """The constraint guard refused the proof (MDN_ERR_CONSTRAINT_VIOLATED); `report` is its ConstraintReport."""

    def __init__(self, message: str, report: "ConstraintReport"):
        super().__init__(message)
        self.report = report


class Session:
    """One proving session bound to one CUDA device (`mdn_session`)."""

    def __init__(self, params: PcsParams, device: int = 0):
        self._h = C.c_void_p()
        rc = lib().mdn_session_create(C.byref(params), device, C.byref(self._h))
        if rc != 0:
            raise ProverError(f"mdn_session_create failed ({rc}): {lib().mdn_last_error(None).decode()}")

    def close(self):
        if self._h:
            lib().mdn_session_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc == ERR_CONSTRAINT_VIOLATED:
            raise ConstraintViolation(f"[{rc}] {lib().mdn_last_error(self._h).decode()}", self.last_constraint_report())
        if rc != 0:
            raise ProverError(f"[{rc}] {lib().mdn_last_error(self._h).decode()}")

    @property
    def handle(self):
        return self._h

    def set_shard(self, rank: int, world: int, allgather_cb):
        """Split every proof of this session over `world` ranks (mdn_session_set_shard); collective."""
        self._allgather_cb = allgather_cb      # keep the ctypes trampoline alive
        self._check(lib().mdn_session_set_shard(self._h, rank, world, allgather_cb, None))

    def set_external_check(self, fn):
        """`Statement::eval_external`: fn(challenges u64[2n], aux_values [per AIR u64[]], log_heights bytes) ->
        None / -1 when every assertion holds, else the index of the first failing assertion."""
        if fn is None:
            self._ext_cb = C.cast(None, EXTERNAL_CHECK)
        else:
            def tramp(ctx, ch, n_ch, vals, n_vals, lh, n_airs, failed):
                try:
                    chal = np.ctypeslib.as_array(ch, shape=(2 * n_ch,)).copy() if n_ch else np.zeros(0, np.uint64)
                    av = [np.ctypeslib.as_array(vals[i], shape=(2 * n_vals[i],)).copy() if n_vals[i] else np.zeros(0, np.uint64) for i in range(n_airs)]
                    k = fn(chal, av, bytes(lh[:n_airs]))
                    if k is None or k < 0:
                        return 0
                    failed[0] = k
                    return 1
                except Exception:
                    import traceback
                    traceback.print_exc()
                    return -1
            self._ext_cb = EXTERNAL_CHECK(tramp)
        self._check(lib().mdn_session_set_external_check(self._h, self._ext_cb, None))

    def set_device_aux_builder(self, fn):
        """Aux traces of FLAG_DEVICE_TRACES | FLAG_COLUMN_MAJOR calls (mdn_session_set_device_aux_builder):
        fn(instance, main Matrix, randomness (u64 pointer, 2 * num_randomness words), aux_out device address (int, None
        when aux_width is 0), stream handle (int)) -> the aux values, a sequence of 2 * num_aux_values ints.  aux_out
        holds 2 * aux_width columns of 2^log_height rows, column-major; fn enqueues its writes on `stream` or finishes
        them before returning.  None removes the builder."""
        if fn is None:
            self._dev_aux_cb = C.cast(None, DEVICE_AUX_BUILDER)
        else:
            def tramp(ctx, instance, main, randomness, aux_out, aux_values, stream):
                try:
                    vals = fn(instance, main.contents, randomness, aux_out, stream or 0)
                    for i, v in enumerate(vals if vals is not None else ()):
                        aux_values[i] = int(v)
                    return 0
                except Exception:
                    import traceback
                    traceback.print_exc()
                    return -1
            self._dev_aux_cb = DEVICE_AUX_BUILDER(tramp)
        self._check(lib().mdn_session_set_device_aux_builder(self._h, self._dev_aux_cb, None))

    def set_hash(self, kind: int, challenger_input: bytes = b"", challenger_output: bytes = b""):
        """`blake3_256_config` / `keccak_config` instead of `poseidon2_config` (mdn_session_set_hash) + the pre-bound HashChallenger state."""
        self._check(lib().mdn_session_set_hash(self._h, kind))
        if kind in (HASH_BLAKE3, HASH_KECCAK):
            a = (C.c_uint8 * max(1, len(challenger_input))).from_buffer_copy(challenger_input or b"\0")
            b = (C.c_uint8 * max(1, len(challenger_output))).from_buffer_copy(challenger_output or b"\0")
            hc = HashChallenger(a, len(challenger_input), b, len(challenger_output))
            self._check(lib().mdn_session_set_hash_challenger(self._h, C.byref(hc)))

    def set_jit(self, min_nodes: int):
        """Node threshold above which constraint programs are NVRTC-compiled (0 = interpreter only)."""
        self._check(lib().mdn_session_set_jit(self._h, min_nodes))

    def set_constraint_guard(self, enable: bool):
        """Check every constraint on every row inside each later proof, with the proof's own challenges, and refuse a
        statement that does not hold with ConstraintViolation (mdn_session_set_constraint_guard)."""
        self._check(lib().mdn_session_set_constraint_guard(self._h, 1 if enable else 0))

    def last_constraint_report(self) -> ConstraintReport:
        """The report of the last guard run (mdn_last_constraint_report)."""
        rep = ConstraintReport()
        rc = lib().mdn_last_constraint_report(self._h, C.byref(rep))
        if rc != 0:
            raise ProverError(f"[{rc}] {lib().mdn_last_error(self._h).decode()}")
        return rep

    def jit_status(self) -> str:
        return lib().mdn_jit_status(self._h).decode()

    def set_preprocessed(self, statement: Statement, preprocessed):
        """`Preprocessed::build(statement, config)` on the device; returns the commitment (u64[4]).
        `preprocessed` = Matrix array in instance order (width 0 = none), or None to remove the bundle."""
        out = np.zeros(4, dtype=np.uint64)
        self._check(lib().mdn_session_set_preprocessed(self._h, C.byref(statement) if statement is not None else None,
                                                       preprocessed, out.ctypes.data_as(u64p)))
        return out

    def prove(self, statement: Statement, traces, challenger: Challenger, aux_builder=None, flags=0):
        """`ProverInstance::new(config, statement, None)?.prove(challenger)`; returns
        (log_trace_heights bytes, fields u64[], commitments u64[n,4])."""
        proof = Proof()
        cb = aux_builder if aux_builder is not None else C.cast(None, AUX_BUILDER)
        self._check(lib().mdn_prove(self._h, C.byref(statement), traces, C.byref(challenger) if challenger is not None else None, cb, None, flags,
                                    C.byref(proof)))
        return proof_to_numpy(proof)

    def check_constraints(self, statement: Statement, traces, challenger: Challenger, aux_builder=None, preprocessed=None,
                          flags=0):
        """`debug::check_constraints(prover_statement, challenger)` on the device: every constraint of every AIR on
        every trace row, without proving.  `preprocessed` = Matrix array in instance order (width 0 = none) or None; the
        row checks and the device LogUp build both read it.
        Returns (ConstraintReport, randomness u64[2 * max num_randomness])."""
        rep = ConstraintReport()
        n_rand = max((statement.airs[i].num_randomness for i in range(statement.n_airs)), default=0)
        rnd = np.zeros(max(1, 2 * n_rand), dtype=np.uint64)
        cb = aux_builder if aux_builder is not None else C.cast(None, AUX_BUILDER)
        self._check(lib().mdn_check_constraints(self._h, C.byref(statement), traces, preprocessed,
                                                C.byref(challenger) if challenger is not None else None, cb, None, flags,
                                                ptr(rnd), C.byref(rep)))
        return rep, rnd[: 2 * n_rand]

    def constraint_census(self, statement: Statement, traces, challenger: Challenger, aux_builder=None, preprocessed=None,
                          flags=0, max_failures: int = 1 << 16, max_tallies: int = 1 << 16):
        """check_constraints without stopping at the first failure: every (instance, row, constraint) that is non-zero.
        Returns (ConstraintCensus, failures, tallies, randomness u64[2 * max num_randomness]), with `failures` the
        first min(violations, max_failures) ConstraintFailure in (instance, row, constraint) order and `tallies` the
        first min(failing_constraints, max_tallies) ConstraintTally in (instance, constraint) order."""
        out = ConstraintCensus()
        n_rand = max((statement.airs[i].num_randomness for i in range(statement.n_airs)), default=0)
        rnd = np.zeros(max(1, 2 * n_rand), dtype=np.uint64)
        fails = (ConstraintFailure * max(1, max_failures))()
        tallies = (ConstraintTally * max(1, max_tallies))()
        cb = aux_builder if aux_builder is not None else C.cast(None, AUX_BUILDER)
        self._check(lib().mdn_constraint_census(self._h, C.byref(statement), traces, preprocessed,
                                                C.byref(challenger) if challenger is not None else None, cb, None, flags,
                                                ptr(rnd), fails if max_failures else None, max_failures,
                                                tallies if max_tallies else None, max_tallies, C.byref(out)))
        return out, list(fails[: out.n_failures]), list(tallies[: out.n_tallies]), rnd[: 2 * n_rand]

    def check_trace_balance(self, statement: Statement, traces, randomness, boundary=(), mutex_sites=None,
                            max_contributions: int = 1 << 16, flags=0) -> dict:
        """`check_trace_balance` (air/src/lookup/debug/trace/mod.rs:169) on the device, jointly over every AIR of the
        statement with a lowered lookup program; programs that read preprocessed columns read the installed bundle
        (set_preprocessed).  randomness: 2 * max num_randomness words (e.g. the randomness of
        check_constraints); boundary: (c0, c1, multiplicity) triples of eval_boundary; mutex_sites: per AIR None or the
        annotation array of LookupProgramBuilder.mutex_sites().  Returns balance_report_dict of the report."""
        rnd = np.ascontiguousarray(np.asarray(randomness, dtype=np.uint64).reshape(-1))
        bnd = np.ascontiguousarray(np.asarray([[int(x) for x in t] for t in boundary], dtype=np.uint64).reshape(-1))
        keep, sites = [], None
        if mutex_sites is not None:
            sites = (u32p * statement.n_airs)()
            for i, m in enumerate(mutex_sites):
                if m is not None:
                    keep.append(np.ascontiguousarray(m, dtype=np.uint32))
                    sites[i] = keep[-1].ctypes.data_as(u32p)
        rep = BalanceReport()
        self._check(lib().mdn_check_trace_balance(self._h, C.byref(statement), traces, ptr(rnd) if rnd.size else None,
                                                  ptr(bnd) if bnd.size else None, len(bnd) // 3, sites, max_contributions,
                                                  flags, C.byref(rep)))
        return balance_report_dict(rep)

    def check_lookup_folds(self, statement: Statement, traces, randomness, fold_marks=None, aux=None, aux_finals=None,
                           folds_out=None, flags=0) -> dict:
        """`collect_column_oracle_folds` (air/src/lookup/debug/trace/mod.rs:196) on the device, compared with an aux trace
        as `assert_prover_matches_oracle` compares them.  fold_marks: per AIR None or LookupProgramBuilder.fold_marks();
        aux: Matrix array in instance order (host row-major, or device as `flags` say) with aux_finals, per AIR None or
        (c0, c1) -- or None for the device LogUp build of the same call; preprocessed columns come from the installed
        bundle, as in check_trace_balance; folds_out: per AIR None, a uint64 numpy array of
        rows * num_columns * 4 words to fill, or a device address (int) with FLAG_DEVICE_TRACES.  A lookup program with
        registers (LookupProgramBuilder(num_columns, num_registers)) is compared on its num_columns LogUp columns only: its
        aux trace keeps every aux column, and check_constraints checks the registers.  Returns fold_report_dict."""
        rnd, marks, fins, keep = _fold_inputs(statement, randomness, fold_marks, aux_finals)
        n, outs = statement.n_airs, None
        if folds_out is not None:
            outs = (u64p * n)()
            for i, o in enumerate(folds_out):
                if o is not None:
                    outs[i] = ptr(o) if isinstance(o, np.ndarray) else C.cast(C.c_void_p(int(o)), u64p)
        rep = FoldReport()
        self._check(lib().mdn_check_lookup_folds(self._h, C.byref(statement), traces, ptr(rnd) if rnd.size else None, marks,
                                                 aux, fins, outs, flags, C.byref(rep)))
        return fold_report_dict(rep)

    def lookup_fold_census(self, statement: Statement, traces, randomness, fold_marks=None, aux=None, aux_finals=None,
                           flags=0, max_failures: int = 1 << 16, max_tallies: int = 1 << 16):
        """check_lookup_folds without stopping at the first disagreement: every (instance, row, column) of non-zero kind.
        The arguments are those of check_lookup_folds without folds_out.  Returns (FoldCensus, failures, tallies), with
        `failures` the first min(disagreements, max_failures) FoldFailure in (instance, row, column) order and `tallies`
        the first min(failing_columns, max_tallies) FoldTally in (instance, column) order."""
        rnd, marks, fins, keep = _fold_inputs(statement, randomness, fold_marks, aux_finals)
        out = FoldCensus()
        fails = (FoldFailure * max(1, max_failures))()
        tallies = (FoldTally * max(1, max_tallies))()
        self._check(lib().mdn_lookup_fold_census(self._h, C.byref(statement), traces, ptr(rnd) if rnd.size else None, marks,
                                                 aux, fins, flags, fails if max_failures else None, max_failures,
                                                 tallies if max_tallies else None, max_tallies, C.byref(out)))
        return out, list(fails[: out.n_failures]), list(tallies[: out.n_tallies])

    def info(self, what: int, cap: int = 0) -> np.ndarray:
        n = lib().mdn_get_info(self._h, what, None, 0)
        if n < 0:
            raise ProverError(f"mdn_get_info({what}) failed")
        out = np.zeros(n, dtype=np.uint64)
        if n:
            lib().mdn_get_info(self._h, what, ptr(out), n)
        return out

    def timings(self) -> Timings:
        t = Timings()
        self._check(lib().mdn_get_timings(self._h, C.byref(t)))
        return t


def _fold_inputs(statement, randomness, fold_marks, aux_finals):
    """(randomness, fold marks, aux finals, arrays to keep alive) as the two lookup fold checks take them."""
    rnd = np.ascontiguousarray(np.asarray(randomness, dtype=np.uint64).reshape(-1))
    n, keep = statement.n_airs, []
    marks = fins = None
    if fold_marks is not None:
        marks = (u32p * n)()
        for i, m in enumerate(fold_marks):
            if m is not None:
                keep.append(np.ascontiguousarray(m, dtype=np.uint32))
                marks[i] = keep[-1].ctypes.data_as(u32p)
    if aux_finals is not None:
        fins = (u64p * n)()
        for i, f in enumerate(aux_finals):
            if f is not None:
                keep.append(np.array([int(f[0]), int(f[1])], dtype=np.uint64))
                fins[i] = ptr(keep[-1])
    return rnd, marks, fins, keep


def device_matrices(tensors):
    """mdn_matrix array (instance order) over CUDA tensors of shape (width, N), 64-bit, contiguous: column-major
    device traces for FLAG_DEVICE_TRACES | FLAG_COLUMN_MAJOR.  The tensors must outlive every call that uses the array
    (the array keeps references to them)."""
    mats = (Matrix * len(tensors))()
    for i, t in enumerate(tensors):
        if not t.is_cuda or t.dim() != 2 or t.element_size() != 8 or not t.is_contiguous():
            raise ValueError(f"tensor {i}: need a contiguous 64-bit CUDA tensor of shape (width, N)")
        width, n = t.shape
        if n < 1 or n & (n - 1):
            raise ValueError(f"tensor {i}: the height {n} is not a power of two")
        mats[i] = Matrix(C.cast(C.c_void_p(t.data_ptr()), u64p), n.bit_length() - 1, width)
    mats._keep = list(tensors)
    return mats


def proof_to_numpy(proof: Proof):
    heights = bytes(proof.log_trace_heights[: proof.n_heights])
    fields = np.ctypeslib.as_array(proof.fields, shape=(proof.n_fields,)).copy() if proof.n_fields else np.zeros(0, np.uint64)
    comms = (np.ctypeslib.as_array(proof.commitments, shape=(proof.n_commitments * 4,)).copy().reshape(-1, 4)
             if proof.n_commitments else np.zeros((0, 4), np.uint64))
    return heights, fields, comms
