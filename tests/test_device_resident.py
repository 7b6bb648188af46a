"""Traces that already live on the GPU, column-major (MDN_FLAG_DEVICE_TRACES | MDN_FLAG_COLUMN_MAJOR), with their aux
traces from a device aux builder (mdn_session_set_device_aux_builder).

Every case proves the same statement twice -- from host row-major traces with a host aux builder, and from column-major
device traces with the equivalent device aux builder -- and the two proofs must be equal byte for byte and accepted by
the oracle verifier.  The device builder computes the aux columns with the host builder and copies them into `aux_out`
on the session's stream: what is under test is the library's side (ingest, in-place LogUp build, aux slots, checks).

On the CPU kernel emulator of tests/emu (MDN_ALLOW_EMULATOR=1, tests/test_device_resident_emulated.py) device memory
is host memory, so "device" buffers are numpy arrays there; on the H100 they are CUDA tensors."""
import ctypes as C
import os

import numpy as np
import pytest

import helpers as H
import oracle_binding as ob
import pkgload
import test_airs as TA
import test_check_constraints as TC

pkg = pkgload.load_pkg()
W, B = pkg.workload, pkg.binding
P = W.P
pytestmark = pytest.mark.gpu
EMU = os.environ.get("MDN_ALLOW_EMULATOR") == "1"
CM = B.FLAG_DEVICE_TRACES | B.FLAG_COLUMN_MAJOR


# ---------------------------------------------------------------------------------------------------------------------
# device buffers: CUDA tensors on the GPU, numpy arrays on the emulator
# ---------------------------------------------------------------------------------------------------------------------
def to_device(a):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    if EMU:
        return a.copy()
    import torch
    return torch.from_numpy(a.view(np.int64)).cuda()


def addr(buf):
    return buf.ctypes.data if EMU else buf.data_ptr()


def from_device(buf):
    return buf.copy() if EMU else buf.cpu().numpy().view(np.uint64)


class _CudaArray:
    """`aux_out` as a CUDA array (the __cuda_array_interface__ torch.as_tensor reads)."""
    def __init__(self, address, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "<i8", "data": (address, False), "version": 3,
                                         "strides": None}


def write_device(address, a, stream):
    """Copy host array `a` to device address `address`, ordered on the session's stream."""
    a = np.ascontiguousarray(a, dtype=np.uint64)
    if EMU:
        C.memmove(address, a.ctypes.data, a.nbytes)
        return
    import torch
    with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
        dst = torch.as_tensor(_CudaArray(address, a.shape), device="cuda")
        dst.copy_(torch.from_numpy(a.view(np.int64)))


def column_major_traces(wl):
    """(mdn_matrix array, device buffers) of the workload's traces, column-major: shape (width, N)."""
    bufs = [to_device(t.T) for t in wl.traces]
    if not EMU:
        return B.device_matrices(bufs), bufs
    mats = (B.Matrix * wl.k)()
    for i, b in enumerate(bufs):
        mats[i] = B.Matrix(C.cast(C.c_void_p(addr(b)), B.u64p), wl.log_heights[i], wl.widths[i])
    return mats, bufs


def row_major_device_traces(wl):
    bufs = [to_device(t) for t in wl.traces]
    mats = (B.Matrix * wl.k)()
    for i, b in enumerate(bufs):
        mats[i] = B.Matrix(C.cast(C.c_void_p(addr(b)), B.u64p), wl.log_heights[i], wl.widths[i])
    return mats, bufs


def host_aux(wl, host_builder, instance, randomness):
    """The host builder's aux trace (row-major N x 2*aux_width) and values for one instance."""
    a = wl._airs[instance]
    n = 1 << wl.log_heights[instance]
    aux = np.zeros(max(1, n * 2 * a.aux_width), dtype=np.uint64)
    vals = np.zeros(2 * a.num_aux_values + 1, dtype=np.uint64)
    if host_builder is not None:
        m = B.Matrix(wl.traces[instance].ctypes.data_as(B.u64p), wl.log_heights[instance], wl.widths[instance])
        assert host_builder(None, instance, C.pointer(m), randomness, B.ptr(aux), B.ptr(vals)) == 0
    return aux[: n * 2 * a.aux_width].reshape(n, 2 * a.aux_width), vals[: 2 * a.num_aux_values]


def device_builder(wl, host_builder, bufs, calls=None, corrupt=None):
    """The device aux builder equivalent to `host_builder` (None: zeros); checks that `main` is the caller's matrix."""
    def fn(instance, main, randomness, aux_out, stream):
        assert C.cast(main.values, C.c_void_p).value == addr(bufs[instance])
        assert (main.log_height, main.width) == (wl.log_heights[instance], wl.widths[instance])
        if calls is not None:
            calls.append(instance)
        aux, vals = host_aux(wl, host_builder, instance, randomness)
        if corrupt is not None:
            aux = corrupt(aux)
        if aux.shape[1]:
            write_device(aux_out, aux.T, stream)
        else:
            assert aux_out is None
        return vals
    return fn


def dummy_case(log_heights, widths, aux_widths, seed=11):
    """The dummy Miden AIR (it does not constrain its aux trace) with a host builder writing canonical pseudo-random
    aux columns and values that depend on the randomness."""
    wl = W.Workload(log_heights, widths=widths, aux_widths=aux_widths)

    def fn(ctx, instance, main, randomness, aux_out, aux_values):
        n, a = 1 << main.contents.log_height, 2 * wl._airs[instance].aux_width
        v = W.splitmix64(np.arange(n * a + 2, dtype=np.uint64) ^ np.uint64(seed + 1000 * instance)) % np.uint64(P)
        if a:
            np.ctypeslib.as_array(aux_out, shape=(n * a,))[:] = v[: n * a]
        for q in range(2 * wl._airs[instance].num_aux_values):
            aux_values[q] = (int(v[-2 + q % 2]) ^ int(randomness[q % 2])) % P
        return 0
    return wl, fn


# ---------------------------------------------------------------------------------------------------------------------
# one statement, proved both ways
# ---------------------------------------------------------------------------------------------------------------------
def prod_observe(c, felts):
    B.lib().mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(felts, dtype=np.uint64)), len(felts))


def session(params, hash_kind=B.HASH_POSEIDON2):
    s = B.Session(params, 0)
    if hash_kind != B.HASH_POSEIDON2:
        s.set_hash(hash_kind, W.initial_hash_challenger(params) if hash_kind in (B.HASH_BLAKE3, B.HASH_KECCAK) else b"")
    return s


def oracle_verify(params, wl, hash_kind, proof, prep_commitment=None):
    L = TC._orc()
    init = W.initial_hash_challenger(params) if hash_kind in (B.HASH_BLAKE3, B.HASH_KECCAK) else b""
    ch = TC.seed(params, hash_kind) or B.Challenger()
    assert L.orc_set_hash(hash_kind, init or None, len(init)) == 0
    try:
        return H.oracle_verify(params, wl, ch, *proof, prep_commitment=prep_commitment)
    finally:
        L.orc_set_hash(0, None, 0)


def same(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def prove_both(s, params, wl, host_builder=None, hash_kind=B.HASH_POSEIDON2, prep_commitment=None, verify=True):
    """Host row-major + host builder vs column-major device traces + device builder: equal, verified, inputs intact."""
    ch = TC.seed(params, hash_kind)
    ref = s.prove(wl.statement, wl.matrices, ch, B.AUX_BUILDER(host_builder) if host_builder else None)
    mats, bufs = column_major_traces(wl)
    calls = []
    s.set_device_aux_builder(device_builder(wl, host_builder, bufs, calls))
    try:
        got = s.prove(wl.statement, mats, ch, None, CM)
    finally:
        s.set_device_aux_builder(None)
    assert same(ref, got), "the column-major device proof differs from the host proof"
    assert calls == [i for i in range(wl.k) if not wl._airs[i].lookup]       # instance order, no LogUp AIR
    for t, b in zip(wl.traces, bufs):
        assert np.array_equal(from_device(b), t.T), "the caller's device trace changed"
    if verify:
        rc, err = oracle_verify(params, wl, hash_kind, got, prep_commitment)
        assert rc == 0, err
    return got


@pytest.fixture(scope="module")
def sess_fast():
    s = B.Session(W.fast_pcs_params(), 0)
    yield s
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# proofs
# ---------------------------------------------------------------------------------------------------------------------
def test_every_small_height(sess_fast):
    """Every height the host path accepts up to 2^12 (one-row traces of odd width take the ingest's scalar tail)."""
    params, accepted = W.fast_pcs_params(), []
    for lh in range(0, 13):
        wl, fn = dummy_case([lh], (9,), (1,), seed=lh)
        try:
            sess_fast.prove(wl.statement, wl.matrices, TC.seed(params), B.AUX_BUILDER(fn))
        except B.ProverError as e:
            host_err = str(e)
            mats, bufs = column_major_traces(wl)
            with pytest.raises(B.ProverError) as ei:
                sess_fast.prove(wl.statement, mats, TC.seed(params), None, CM)
            assert str(ei.value) == host_err
            continue
        accepted.append(lh)
        prove_both(sess_fast, params, wl, fn)
    assert accepted and accepted[0] <= 3 and accepted == list(range(accepted[0], 13)), accepted


def test_mixed_heights(sess_fast):
    params = W.fast_pcs_params()
    prove_both(sess_fast, params, *dummy_case([6, 8, 5], (11, 9, 10), (2, 0, 1)))
    prove_both(sess_fast, params, *dummy_case([0, 3, 7, 7], (9, 13, 9, 10), (1, 2, 0, 3)))
    prove_both(sess_fast, params, *TA.fib_product_workload([6, 4]))


def test_aux_width_zero(sess_fast):
    params = W.fast_pcs_params()
    prove_both(sess_fast, params, TA.periodic_workload(6, lqd=3))
    prove_both(sess_fast, params, *dummy_case([5, 7], (9, 12), (0, 0)))


def test_no_device_builder_means_zero_aux(sess_fast):
    """Without a device builder the aux traces and values are zero, as with a NULL host builder."""
    params = W.fast_pcs_params()
    wl = W.Workload([6, 5], widths=(9, 10), aux_widths=(2, 1))
    ch = TC.seed(params)
    ref = sess_fast.prove(wl.statement, wl.matrices, ch)
    mats, bufs = column_major_traces(wl)
    assert same(ref, sess_fast.prove(wl.statement, mats, ch, None, CM))


@pytest.mark.parametrize("log_h", [6, 12])
def test_logup_reads_the_callers_trace(sess_fast, log_h):
    """A LogUp AIR built from the caller's column-major buffer in place: its aux root equals the one of the row-major
    device path (which builds from a copy of the trace), and the proofs are equal."""
    params = W.fast_pcs_params()
    wl, _ = TA.logup_workload(log_h, device=True)
    ch = TC.seed(params)
    rm, rm_bufs = row_major_device_traces(wl)
    ref = sess_fast.prove(wl.statement, rm, ch, None, B.FLAG_DEVICE_TRACES)
    ref_aux_root = sess_fast.info(1)
    got = prove_both(sess_fast, params, wl)
    assert same(ref, got)
    assert np.array_equal(sess_fast.info(1), ref_aux_root)


def test_logup_next_to_a_device_built_aux(sess_fast):
    """A LogUp AIR next to the fib/product AIR whose aux comes from the device builder (called for instance 1 only)."""
    params = W.fast_pcs_params()
    wl_l, _ = TA.logup_workload(6, device=True)
    wl_f, fib_builder = TA.fib_product_workload([7])
    wl = W.Workload([6, 7], widths=[6, 3], aux_widths=[3, 1], programs=[wl_l.programs[0], wl_f.programs[0]],
                    traces=[wl_l.traces[0], wl_f.traces[0]], public_values=[int(v) for v in wl_f.public_values],
                    log_quotient_degrees=[2, 1], num_aux_values=[1, 1],
                    periodic=[np.array([[1], [0], [0], [1]], dtype=np.uint64), None], lookups=[(3, wl_l._lookups[0][1]), None])

    def builder(ctx, instance, main, randomness, aux_out, aux_values):
        assert instance == 1
        return fib_builder(ctx, 0, main, randomness, aux_out, aux_values)

    prove_both(sess_fast, params, wl, builder)


def test_preprocessed_bundle():
    params = W.fast_pcs_params()
    s = B.Session(params, 0)
    try:
        wl = TA.preprocessed_workload((6, 8), (True, True))
        commitment = s.set_preprocessed(wl.statement, wl.preprocessed_matrices)
        prove_both(s, params, wl, prep_commitment=commitment)
    finally:
        s.close()


def test_jit_sized_program():
    """A constraint program large enough for the NVRTC kernel."""
    params = W.fast_pcs_params()
    s = B.Session(params, 0)
    try:
        prove_both(s, params, TA.big_program_workload(8))
        assert list(s.info(8)) == [1], s.jit_status()
    finally:
        s.close()


@pytest.mark.parametrize("hash_kind", [B.HASH_BLAKE3, B.HASH_KECCAK, B.HASH_RPO])
def test_hash_configurations(hash_kind):
    params = W.fast_pcs_params()
    s = session(params, hash_kind)
    try:
        prove_both(s, params, *TA.fib_product_workload([6, 5]), hash_kind=hash_kind)
        prove_both(s, params, *dummy_case([5, 7], (9, 17), (1, 2)), hash_kind=hash_kind)
    finally:
        s.close()


def test_benchmark_statement_2_20():
    """The 2^20 x (51, 22, 16) statement of bench.py, with an aux builder."""
    params = W.miden_pcs_params()
    s = B.Session(params, 0)
    try:
        prove_both(s, params, *dummy_case([20] * 3, W.MIDEN_WIDTHS, W.MIDEN_AUX_WIDTHS))
    finally:
        s.close()


def test_narrow_2_22():
    """A narrow 2^22 trace: the (11, 11) NTT split."""
    params = W.miden_pcs_params()
    s = B.Session(params, 0)
    try:
        prove_both(s, params, *dummy_case([22], (9,), (1,)))
    finally:
        s.close()


def test_staged_api_with_device_aux_matrices(sess_fast):
    """begin / commit_aux / finish with column-major device traces and column-major device aux matrices."""
    params = W.fast_pcs_params()
    wl, builder = TA.fib_product_workload([6, 4])
    ch = TC.seed(params)
    ref = sess_fast.prove(wl.statement, wl.matrices, ch, B.AUX_BUILDER(builder))
    lib, h = B.lib(), sess_fast.handle
    mats, bufs = column_major_traces(wl)
    root, rnd = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64)
    assert lib.mdn_prove_begin(h, C.byref(wl.statement), mats, C.byref(ch), CM, B.ptr(root), B.ptr(rnd)) == 0, lib.mdn_last_error(h)
    aux_bufs, vals = [], []
    aux_mats = (B.Matrix * wl.k)()
    r = np.concatenate([rnd, np.zeros(1, dtype=np.uint64)])
    for i in range(wl.k):
        aux, v = host_aux(wl, builder, i, B.ptr(r))
        aux_bufs.append(to_device(aux.T))
        vals.append(np.ascontiguousarray(v))
        aux_mats[i] = B.Matrix(C.cast(C.c_void_p(addr(aux_bufs[-1])), B.u64p), wl.log_heights[i], aux.shape[1])
    vptrs = (B.u64p * wl.k)(*[B.ptr(v) for v in vals])
    assert lib.mdn_prove_commit_aux(h, aux_mats, vptrs, None) == 0, lib.mdn_last_error(h)
    proof = B.Proof()
    assert lib.mdn_prove_finish(h, C.byref(proof)) == 0, lib.mdn_last_error(h)
    assert same(ref, B.proof_to_numpy(proof))
    for t, b in zip(wl.traces, bufs):
        assert np.array_equal(from_device(b), t.T)


# ---------------------------------------------------------------------------------------------------------------------
# mdn_check_constraints
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", TC.VALID + TC.VIOLATIONS)
def test_check_constraints_matches_the_host_path(sess_fast, name):
    """Same report and randomness as the host path, on valid statements and on single-fault statements."""
    params = W.fast_pcs_params()
    wl, bld = TC.valid_case(name) if name in TC.VALID else TC.violation_case(name)
    ch = TC.seed(params)
    prep = wl.preprocessed_matrices if wl.preprocessed is not None else None
    rep, rnd = sess_fast.check_constraints(wl.statement, wl.matrices, ch, aux_builder=B.AUX_BUILDER(bld) if bld else None,
                                           preprocessed=prep)
    mats, bufs = column_major_traces(wl)
    sess_fast.set_device_aux_builder(device_builder(wl, bld, bufs))
    try:
        rep2, rnd2 = sess_fast.check_constraints(wl.statement, mats, ch, preprocessed=prep, flags=CM)
    finally:
        sess_fast.set_device_aux_builder(None)
    assert TC.report_dict(rep2) == TC.report_dict(rep)
    assert np.array_equal(rnd2, rnd)
    for t, b in zip(wl.traces, bufs):
        assert np.array_equal(from_device(b), t.T), "the caller's device trace changed"


# ---------------------------------------------------------------------------------------------------------------------
# error paths: refused, and the session proves correctly afterwards
# ---------------------------------------------------------------------------------------------------------------------
def _refused(s, fn, code, text):
    with pytest.raises(B.ProverError) as ei:
        fn()
    assert str(ei.value).startswith(f"[{code}]") and text in str(ei.value), str(ei.value)


def test_error_paths_leave_the_session_usable():
    params = W.fast_pcs_params()
    s = B.Session(params, 0)
    try:
        wl, builder = TA.fib_product_workload([6, 4])
        ch = TC.seed(params)
        ref = s.prove(wl.statement, wl.matrices, ch, B.AUX_BUILDER(builder))

        def good():
            assert same(prove_both(s, params, wl, builder, verify=False), ref)

        mats, bufs = column_major_traces(wl)
        _refused(s, lambda: s.prove(wl.statement, mats, ch, None, B.FLAG_COLUMN_MAJOR), -1, "MDN_FLAG_DEVICE_TRACES")
        _refused(s, lambda: s.check_constraints(wl.statement, mats, ch, flags=B.FLAG_COLUMN_MAJOR), -1, "MDN_FLAG_DEVICE_TRACES")
        good()
        # a misaligned base pointer
        bad = (B.Matrix * wl.k)(*[mats[i] for i in range(wl.k)])
        big = to_device(np.concatenate([[0], wl.traces[1].T.reshape(-1)]))
        bad[1] = B.Matrix(C.cast(C.c_void_p(addr(big) + 8), B.u64p), wl.log_heights[1], wl.widths[1])
        _refused(s, lambda: s.prove(wl.statement, bad, ch, None, CM), -1, "16-byte aligned")
        _refused(s, lambda: s.check_constraints(wl.statement, bad, ch, flags=CM), -1, "16-byte aligned")
        good()
        # a non-canonical cell
        t = wl.traces[1].T.copy()
        t[4, 9] = P
        nc = to_device(t)
        bad[1] = B.Matrix(C.cast(C.c_void_p(addr(nc)), B.u64p), wl.log_heights[1], wl.widths[1])
        _refused(s, lambda: s.prove(wl.statement, bad, ch, None, CM), -1, "a main trace contains a non-canonical")
        _refused(s, lambda: s.check_constraints(wl.statement, bad, ch, flags=CM), -1, "a main trace contains a non-canonical")
        good()
        # a non-canonical word written by the device builder
        def corrupt(aux):
            aux = aux.copy()
            aux[3, 1] = P + 5
            return aux
        s.set_device_aux_builder(device_builder(wl, builder, bufs, corrupt=corrupt))
        _refused(s, lambda: s.prove(wl.statement, mats, ch, None, CM), -1, "an aux trace contains a non-canonical")
        _refused(s, lambda: s.check_constraints(wl.statement, mats, ch, flags=CM), -1, "an aux trace contains a non-canonical")
        good()
        # a device builder returning non-zero
        def failing(instance, main, randomness, aux_out, stream):
            raise RuntimeError("builder failure on purpose")
        s.set_device_aux_builder(failing)
        _refused(s, lambda: s.prove(wl.statement, mats, ch, None, CM), -5, "device aux builder failed for instance 0")
        _refused(s, lambda: s.check_constraints(wl.statement, mats, ch, flags=CM), -5, "device aux builder failed for instance 0")
        s.set_device_aux_builder(None)
        good()
        # a host builder passed with COLUMN_MAJOR
        _refused(s, lambda: s.prove(wl.statement, mats, ch, B.AUX_BUILDER(builder), CM), -1, "device aux builder")
        _refused(s, lambda: s.check_constraints(wl.statement, mats, ch, aux_builder=B.AUX_BUILDER(builder), flags=CM), -1,
                 "device aux builder")
        good()
        # row-major device traces keep their refusal of a host builder
        rm, rm_bufs = row_major_device_traces(wl)
        _refused(s, lambda: s.prove(wl.statement, rm, ch, B.AUX_BUILDER(builder), B.FLAG_DEVICE_TRACES), -4,
                 "an aux builder needs host-resident main traces")
        good()
        for t, b in zip(wl.traces, bufs):
            assert np.array_equal(from_device(b), t.T)
    finally:
        s.close()


# ---------------------------------------------------------------------------------------------------------------------
# the C++ host layer with a CUDA aux-builder kernel (tests/cpp_device, built by build())
# ---------------------------------------------------------------------------------------------------------------------
def test_cpp_host_layer_with_a_cuda_aux_builder_kernel():
    import subprocess
    if EMU:
        pytest.skip("a CUDA kernel: H100 only")
    d = os.path.join(pkgload.ROOT, "tests", "cpp_device")
    subprocess.check_call(["make", "-s", "-C", d])
    r = subprocess.run([os.path.join(d, "test_device_api")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "DEVICE_API_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
