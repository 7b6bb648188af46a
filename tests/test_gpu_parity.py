"""GPU parity tests (run on an H100): every stage of the CUDA path, called through the C ABI,
against the CPU oracle on identical seeded inputs; bit-exact (integer arithmetic)."""
import ctypes as C

import numpy as np
import pytest

import helpers as H
import oracle_binding as ob
import pkgload

pkg = pkgload.load_pkg()
W, B = pkg.workload, pkg.binding
P = W.P
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    return B.lib()


def prod_observe(c, felts):
    B.lib().mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(felts, dtype=np.uint64)), len(felts))


@pytest.fixture(scope="module")
def sess():
    s = B.Session(W.miden_pcs_params(), 0)
    B.lib().mdn_set_debug(s.handle, 1)
    yield s
    s.close()


@pytest.fixture(scope="module")
def sess_fast():
    s = B.Session(W.fast_pcs_params(), 0)
    B.lib().mdn_set_debug(s.handle, 1)
    yield s
    s.close()


def rand_felts(shape, seed):
    rng = np.random.default_rng(seed)
    v = rng.integers(0, 2**63, shape, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, shape, dtype=np.uint64)
    v = np.where(v >= np.uint64(P), v - np.uint64(P), v)
    return np.ascontiguousarray(v.astype(np.uint64))


def test_poseidon2_permutation_device(lib, sess, oracle):
    st = rand_felts((1000, 12), 1)
    st[0] = np.arange(12)
    st[1] = P - 1
    st[2] = 0
    a, b = st.copy(), st.copy()
    assert lib.mdn_poseidon2_permute(sess.handle, B.ptr(a.reshape(-1)), len(a)) == 0
    oracle.orc_poseidon2_permute(ob.ptr(b.reshape(-1)), len(b))
    assert np.array_equal(a, b)
    assert int(a[0, 0]) == 0xF292AB67C0F14B03   # reference KAT poseidon2/test.rs:27


@pytest.mark.parametrize("log_n,width", [(3, 1), (4, 5), (7, 9), (10, 3), (11, 2), (12, 3), (13, 2), (15, 1)])
def test_coset_lde_batch(lib, sess, oracle, log_n, width):
    m = rand_felts((1 << log_n, width), log_n)
    if log_n == 4:
        m[:, 0] = 0; m[:, 1] = P - 1
    shift = oracle.orc_lde_shift(log_n + 3)
    got = np.zeros(((1 << log_n) << 3, width), dtype=np.uint64)
    exp = np.zeros_like(got)
    mat = B.Matrix(B.ptr(m), log_n, width)
    assert lib.mdn_coset_lde_batch(sess.handle, C.byref(mat), 3, shift, B.ptr(got.reshape(-1))) == 0, lib.mdn_last_error(sess.handle)
    omat = ob.Matrix(ob.ptr(m), log_n, width)
    oracle.orc_coset_lde_batch(C.byref(omat), 3, shift, ob.ptr(exp.reshape(-1)))
    assert np.array_equal(got, exp)


@pytest.mark.parametrize("shapes", [[(5, 9)], [(4, 3), (4, 8), (6, 17)], [(3, 16), (5, 1), (8, 51), (8, 22)], [(12, 10), (13, 4)]])
def test_lmcs_commit_root(lib, sess, oracle, shapes):
    mats = [rand_felts((1 << lh, w), 100 + i) for i, (lh, w) in enumerate(shapes)]
    # oracle: LDE each matrix (domain order), then build_aligned_tree
    ldes, omats = [], (ob.Matrix * len(shapes))()
    for i, ((lh, w), m) in enumerate(zip(shapes, mats)):
        out = np.zeros(((1 << lh) << 3, w), dtype=np.uint64)
        om = ob.Matrix(ob.ptr(m), lh, w)
        oracle.orc_coset_lde_batch(C.byref(om), 3, oracle.orc_lde_shift(lh + 3), ob.ptr(out.reshape(-1)))
        # orc_lmcs_commit takes DOMAIN-order matrices: undo the bit reversal
        n = out.shape[0]; bits = lh + 3
        idx = np.array([int(format(i, "0%db" % bits)[::-1], 2) for i in range(n)])
        nat = np.ascontiguousarray(out[idx])
        ldes.append(nat)
        omats[i] = ob.Matrix(ob.ptr(nat.reshape(-1)), lh + 3, w)
    exp = np.zeros(4, dtype=np.uint64)
    oracle.orc_lmcs_commit(omats, len(shapes), ob.ptr(exp), None)
    pm = (B.Matrix * len(shapes))()
    for i, ((lh, w), m) in enumerate(zip(shapes, mats)):
        pm[i] = B.Matrix(B.ptr(m.reshape(-1)), lh, w)
    got = np.zeros(4, dtype=np.uint64)
    assert lib.mdn_lmcs_commit(sess.handle, pm, len(shapes), B.ptr(got)) == 0, lib.mdn_last_error(sess.handle)
    assert np.array_equal(got, exp)


def _compare_proofs(s, params, wl, aux_builder=None):
    ch = W.initial_challenger(params, prod_observe)
    cb = B.AUX_BUILDER(aux_builder) if aux_builder else None
    heights, fields, comms = s.prove(wl.statement, wl.matrices, ch, cb)
    ocb = aux_builder
    h, oh, of, oc = H.oracle_prove(params, wl, ch, ocb)
    try:
        # stage-by-stage first, so a failure names the first diverging phase
        names = ["main_root", "aux_root", "quotient_root", "ood_point", "quotient_acc", "deep_evals", "fri_roots", "query_indices"]
        for what, name in enumerate(names):
            g, e = s.info(what), H.oracle_info(h, what)
            assert np.array_equal(g, e), f"stage {name} differs"
        assert heights == oh
        assert np.array_equal(comms, oc)
        assert np.array_equal(fields, of)
    finally:
        ob.lib().orc_prove_free(h)
    rc, err = H.oracle_verify(params, wl, ch, heights, fields, comms)
    assert rc == 0, err
    return heights, fields, comms


def test_prove_bit_exact_single_air(sess_fast):
    _compare_proofs(sess_fast, W.fast_pcs_params(), W.Workload([5], widths=(9,), aux_widths=(1,)))


def test_prove_bit_exact_mixed_heights(sess_fast):
    _compare_proofs(sess_fast, W.fast_pcs_params(), W.Workload([6, 8, 5], widths=(11, 9, 10), aux_widths=(2, 0, 1)))


def test_prove_many_airs_of_one_height(sess_fast):
    # more equal-height matrices than one leaf-sponge launch takes (8): the states are handed on between launches;
    # 11 + 2 AIRs, so both the main and the aux tree chain launches and a second height group follows
    k = 13
    lhs = [5] * 11 + [7, 7]
    _compare_proofs(sess_fast, W.fast_pcs_params(), W.Workload(lhs, widths=(9,) * k, aux_widths=(1,) * k))


def test_prove_bit_exact_miden_shape_small(sess):
    _compare_proofs(sess, W.miden_pcs_params(), W.Workload([8, 7, 6]))


def test_prove_bit_exact_two_pass_ntt(sess):
    # heights above 2^11 exercise the strided + contiguous NTT passes
    _compare_proofs(sess, W.miden_pcs_params(), W.Workload([12, 13], widths=(12, 9), aux_widths=(1, 2)))


def test_prove_with_aux_selectors_transitions(sess_fast):
    import test_airs
    wl, builder = test_airs.fib_product_workload([6, 4], lqd=3)
    _compare_proofs(sess_fast, W.fast_pcs_params(), wl, builder)


def test_prove_mixed_quotient_degrees(sess_fast):
    # fib/product AIR with its native log_quotient_degree 1 next to a degree-9 AIR (log 3): the
    # reference evaluates the first on gJ_j and upsamples (quotient.rs:45-56)
    import test_airs
    wl, builder = test_airs.fib_product_workload([6, 4], lqd=1)
    _compare_proofs(sess_fast, W.fast_pcs_params(), wl, builder)
    wl, builder = test_airs.fib_product_workload([4, 7], lqd=1)
    _compare_proofs(sess_fast, W.fast_pcs_params(), wl, builder)


def test_prove_low_max_quotient_degree(sess_fast):
    # every AIR below the blowup: D_max = 2 < B = 8 quotient chunks
    import test_airs
    wl, builder = test_airs.fib_product_workload([5], lqd=1)
    _compare_proofs(sess_fast, W.fast_pcs_params(), wl, builder)
    _compare_proofs(sess_fast, W.fast_pcs_params(), test_airs.periodic_workload(6, lqd=1))


@pytest.mark.parametrize("log_blowup", [1, 2, 4])
def test_prove_other_blowups(log_blowup):
    # PcsParams are generic (pcs/params.rs:53-99); the Miden value is 3
    import test_airs
    params = B.PcsParams(log_blowup, 2, 1, 1, 2, 6, 3)
    s = B.Session(params, 0)
    B.lib().mdn_set_debug(s.handle, 1)
    try:
        wl, builder = test_airs.fib_product_workload([6], lqd=1)
        _compare_proofs(s, params, wl, builder)
        _compare_proofs(s, params, test_airs.periodic_workload(5, lqd=1))
    finally:
        s.close()


@pytest.mark.parametrize("log_arity", [1, 3])
def test_prove_other_fri_arities(log_arity):
    # FriFold::new accepts log_arity 1, 2, 3 (pcs/fri/fold/mod.rs:38-46); Miden uses 2
    import test_airs
    params = B.PcsParams(3, log_arity, 2, 2, 3, 7, 4)
    s = B.Session(params, 0)
    B.lib().mdn_set_debug(s.handle, 1)
    try:
        _compare_proofs(s, params, W.Workload([7, 9], widths=(9, 12), aux_widths=(1, 2)))
        wl, builder = test_airs.fib_product_workload([8], lqd=1)
        _compare_proofs(s, params, wl, builder)
    finally:
        s.close()


@pytest.mark.parametrize("pcs,lhs", [((3, 2, 7, 4, 12, 27, 16), [3]),        # 2^6-point LDE < final degree * blowup: zero FRI rounds
                                     ((3, 2, 7, 4, 12, 27, 16), [4, 6]),     # still zero rounds, two heights
                                     ((3, 2, 7, 4, 12, 27, 16), [7]),        # exactly at the boundary
                                     ((1, 1, 0, 0, 0, 3, 0), [2]),           # 4-row trace, blowup 2, no proof-of-work at all
                                     ((2, 3, 1, 1, 1, 4, 2), [3, 5])])       # arity 8 on tiny domains
def test_prove_edge_configurations(pcs, lhs):
    import test_airs
    params = B.PcsParams(*pcs)
    s = B.Session(params, device=0)
    B.lib().mdn_set_debug(s.handle, 1)
    builder = None
    if params.log_blowup >= 3:
        wl = W.Workload(lhs, widths=(9,) * len(lhs), aux_widths=(1,) * len(lhs))
    elif len(lhs) == 1:
        wl, builder = test_airs.fib_product_workload(lhs, lqd=1)
    else:
        wl = W.Workload(lhs, widths=(9,) * len(lhs), aux_widths=(1,) * len(lhs), log_quotient_degrees=[params.log_blowup] * len(lhs),
                        programs=[AP_degree(1 + (1 << params.log_blowup)) for _ in lhs])
    _compare_proofs(s, params, wl, builder)
    s.close()


def test_prove_periodic_columns(sess_fast):
    import test_airs
    _compare_proofs(sess_fast, W.fast_pcs_params(), test_airs.periodic_workload(6, lqd=3))


@pytest.mark.parametrize("log_hs,with_prep", [((6, 8), (True, True)), ((5, 7), (True, False)), ((5, 7), (False, True)),
                                              ((6, 6, 4), (True, False, True)), ((12, 13), (True, True))])
def test_prove_preprocessed_columns(log_hs, with_prep):
    # Preprocessed::build on the device, commitment == oracle's, then bit-exact proofs with the
    # preprocessed group first in the opening batch (shorter than the max LDE in case 2)
    import test_airs
    wl = test_airs.preprocessed_workload(log_hs, with_prep)
    params = W.fast_pcs_params()
    s = B.Session(params, device=0)
    B.lib().mdn_set_debug(s.handle, 1)
    commitment = s.set_preprocessed(wl.statement, wl.preprocessed_matrices)
    _compare_proofs(s, params, wl)
    assert np.array_equal(commitment, wl.oracle_prep_commitment)
    # the bundle is borrowed across proofs: a second proof is identical
    _compare_proofs(s, params, wl)
    # presence parity (PreprocessedValidationError::PresenceMismatch)
    ch = W.initial_challenger(params, prod_observe)
    plain = W.Workload([5], widths=(9,), aux_widths=(1,))
    with pytest.raises(B.ProverError):
        s.prove(plain.statement, plain.matrices, ch)
    s.set_preprocessed(None, None)
    with pytest.raises(B.ProverError):
        s.prove(wl.statement, wl.matrices, ch)
    _compare_proofs(s, params, plain)
    # height mismatch between the bundle and the main traces
    wl_short = test_airs.preprocessed_workload(tuple(h - 1 for h in log_hs), with_prep)
    s.set_preprocessed(wl_short.statement, wl_short.preprocessed_matrices)
    with pytest.raises(B.ProverError):
        s.prove(wl.statement, wl.matrices, ch)


@pytest.mark.parametrize("log_h", [5, 13])
def test_prove_logup_aux_built_on_device(sess_fast, log_h):
    # mdn_air.lookup: fraction collection, per-row sums and the EF prefix sum run on the device; the proof is
    # bit-exact against the oracle and against a host aux builder using Python integers (small case)
    import test_airs
    params = W.fast_pcs_params()
    wl_dev, _ = test_airs.logup_workload(log_h, device=True)
    h1, f1, c1 = _compare_proofs(sess_fast, params, wl_dev)
    if log_h <= 8:
        wl_host, builder = test_airs.logup_workload(log_h, device=False)
        ch = W.initial_challenger(params, prod_observe)
        h2, f2, c2 = sess_fast.prove(wl_host.statement, wl_host.matrices, ch, B.AUX_BUILDER(builder))
        assert h1 == h2 and np.array_equal(f1, f2) and np.array_equal(c1, c2)


def test_logup_mixed_with_host_built_aux(sess_fast):
    # one AIR with a lowered LookupAir (device aux) next to the fib/product AIR whose aux comes from the host callback
    import test_airs
    params = W.fast_pcs_params()
    wl_l, _ = test_airs.logup_workload(6, device=True)
    wl_f, fib_builder = test_airs.fib_product_workload([7])
    progs = [wl_l.programs[0], wl_f.programs[0]]
    wl = W.Workload([6, 7], widths=[6, 3], aux_widths=[3, 1], programs=progs, traces=[wl_l.traces[0], wl_f.traces[0]],
                    public_values=[int(v) for v in wl_f.public_values], log_quotient_degrees=[2, 1], num_aux_values=[1, 1],
                    periodic=[np.array([[1], [0], [0], [1]], dtype=np.uint64), None],
                    lookups=[(3, wl_l._lookups[0][1]), None])

    def builder(ctx, instance, main, randomness, aux_out, aux_values):
        assert instance == 1            # the lookup AIR never reaches the host callback
        return fib_builder(ctx, 0, main, randomness, aux_out, aux_values)

    _compare_proofs(sess_fast, params, wl, builder)


def test_logup_zero_denominator_is_an_error(sess_fast):
    import test_airs
    AP = test_airs.AP
    lb = AP.LookupProgramBuilder(1)
    lb.insert(0, None, lb.const(1), lb.main(0, 0) + lb.challenge(0) - lb.challenge(0))
    b = AP.ProgramBuilder()
    b.assert_zero(b.main(0, 0) - b.main(0, 0))
    t = W.synthetic_trace(3, 5, 2)
    t[7, 0] = 0
    wl = W.Workload([5], widths=[2], aux_widths=[1], programs=[b.serialize()], traces=[t], log_quotient_degrees=[1],
                    num_aux_values=[1], lookups=[(1, lb.serialize())])
    ch = W.initial_challenger(W.fast_pcs_params(), prod_observe)
    with pytest.raises(B.ProverError, match="denominator"):
        sess_fast.prove(wl.statement, wl.matrices, ch)
    # the session stays usable
    _compare_proofs(sess_fast, W.fast_pcs_params(), W.Workload([5], widths=(9,), aux_widths=(1,)))


def _jit_session(params, min_nodes):
    s = B.Session(params, device=0)
    B.lib().mdn_set_debug(s.handle, 1)
    s.set_jit(min_nodes)
    return s


@pytest.mark.parametrize("case", ["fib_aux_selectors", "periodic", "logup", "mixed_degrees", "big_program", "preprocessed"])
def test_jit_constraint_kernels_match_oracle(case):
    # every AIR forced through the NVRTC-specialised kernel (threshold 1 node): proofs stay bit-exact
    import test_airs
    params = W.fast_pcs_params()
    s = _jit_session(params, 1)
    builder = None
    if case == "fib_aux_selectors":
        wl, builder = test_airs.fib_product_workload([6, 4])
    elif case == "periodic":
        wl = test_airs.periodic_workload(6, lqd=3)
    elif case == "logup":
        wl, _ = test_airs.logup_workload(7, device=True)
    elif case == "mixed_degrees":
        wl = W.Workload([5, 7, 6], widths=(9, 9, 9), aux_widths=(1, 1, 1), log_quotient_degrees=[3, 1, 2],
                        programs=[AP_degree(9), AP_degree(3), AP_degree(5)])
    elif case == "big_program":
        wl = test_airs.big_program_workload(5, n_terms=300)        # 10 k nodes: 21 chunk functions
    else:
        wl = test_airs.preprocessed_workload((6, 8), (True, True))
        s.set_preprocessed(wl.statement, wl.preprocessed_matrices)
    _compare_proofs(s, params, wl, builder)
    assert list(s.info(8)) == [1] * wl.k, "the JIT kernel was not used"
    assert "disagreed" not in s.jit_status() and "nvrtc 1" in s.jit_status(), s.jit_status()   # incl. the generated LogUp row kernel
    # and the interpreter on the same session gives the same bytes
    s.set_jit(0)
    _compare_proofs(s, params, wl, builder)
    assert list(s.info(8)) == [0] * wl.k


def test_jit_kernels_with_tiny_chunks(monkeypatch):
    # 5-node chunk functions force cross-chunk spills in both generated kernels (constraints and LogUp rows)
    import test_airs
    monkeypatch.setenv("MDN_JIT_CHUNK", "5")
    params = W.fast_pcs_params()
    s = _jit_session(params, 1)
    wl, _ = test_airs.logup_workload(7, device=True)
    _compare_proofs(s, params, wl)
    assert list(s.info(8)) == [1] and "disagreed" not in s.jit_status(), s.jit_status()
    wl, builder = test_airs.fib_product_workload([6, 4])
    _compare_proofs(s, params, wl, builder)
    assert "disagreed" not in s.jit_status(), s.jit_status()
    s.close()


def test_jit_self_check_catches_a_miscompiling_nvrtc():
    import subprocess, sys, os
    r = subprocess.run([sys.executable, os.path.join(os.path.dirname(__file__), "run_jit_old_nvrtc.py")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "SELF-CHECK OK" in r.stdout or "NOTE" in r.stdout or "SKIP" in r.stdout, r.stdout


def AP_degree(d):
    b = H.pkg.air_program.ProgramBuilder()
    acc = b.const(1)
    for j in range(d):
        acc = acc * b.main(0, j)
    b.assert_zero(acc)
    return b.serialize()


def test_prove_big_constraint_program(sess_fast):
    # ~2.4k nodes per constraint pair: far above the old 256-node interpreter limit
    import test_airs
    _compare_proofs(sess_fast, W.fast_pcs_params(), test_airs.big_program_workload(5, n_terms=300))


def test_config2_synthetic_2_16_roots(sess):
    """BASELINE config 2: synthetic 2^16 x (51, 22, 16): NTT + Poseidon2 commit, bit-exact root."""
    wl = W.Workload([16, 16, 16])
    lib = B.lib()
    got = np.zeros(4, dtype=np.uint64)
    assert lib.mdn_lmcs_commit(sess.handle, wl.matrices, 3, B.ptr(got)) == 0
    ch = W.initial_challenger(W.miden_pcs_params(), prod_observe)
    h, oh, of, oc = H.oracle_prove(W.miden_pcs_params(), wl, ch)
    try:
        assert np.array_equal(got, H.oracle_info(h, 0))
        heights, fields, comms = sess.prove(wl.statement, wl.matrices, ch)
        assert np.array_equal(comms, oc) and np.array_equal(fields, of)
    finally:
        ob.lib().orc_prove_free(h)


def test_full_size_2_20_verifies():
    """BASELINE config 4 shape on one GPU: the 2^20 proof must be accepted by the oracle verifier
    (size-independent property; the oracle prover would take minutes here), and proving twice gives
    identical bytes."""
    s = B.Session(W.miden_pcs_params(), 0)
    wl = W.Workload([20, 20, 20])
    ch = W.initial_challenger(W.miden_pcs_params(), prod_observe)
    a = s.prove(wl.statement, wl.matrices, ch)
    b = s.prove(wl.statement, wl.matrices, ch)
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    rc, err = H.oracle_verify(W.miden_pcs_params(), wl, ch, *a)
    assert rc == 0, err
    s.close()


def _bit_exact_vs_oracle_prover(s, params, wl, prep_commitment=None):
    """Full streams + the stage values that are recorded without the debug copies (roots, OOD point, FRI roots, query
    indices) against the ORACLE PROVER on the same inputs."""
    ch = W.initial_challenger(params, prod_observe)
    heights, fields, comms = s.prove(wl.statement, wl.matrices, ch)
    h, oh, of, oc = H.oracle_prove(params, wl, ch)
    try:
        for what, name in ((0, "main_root"), (1, "aux_root"), (2, "quotient_root"), (3, "ood_point"), (6, "fri_roots"), (7, "query_indices")):
            assert np.array_equal(s.info(what), H.oracle_info(h, what)), f"stage {name} differs"
        assert heights == oh
        assert np.array_equal(comms, oc), "commitment stream differs"
        assert np.array_equal(fields, of), "field stream differs"
    finally:
        ob.lib().orc_prove_free(h)
    return heights, fields, comms


def test_full_size_2_20_bit_exact_vs_oracle_prover():
    """The metric's own configuration -- synthetic 2^20 x (51,22,16), 96-bit parameters -- bit for bit against the oracle
    PROVER (not only its verifier): every root, the OOD point, the FRI roots, the query indices and the complete
    `fields` / `commitments` streams.  The oracle needs tens of seconds on the GPU box's host cores."""
    ob.lib().orc_set_threads(0)
    params = W.miden_pcs_params()
    s = B.Session(params, 0)
    try:
        _bit_exact_vs_oracle_prover(s, params, W.Workload([20, 20, 20]))
    finally:
        s.close()


def test_config5_width_mixed_heights_preprocessed_2_20_bit_exact():
    """BASELINE config 5's features at Miden widths: 51 + 3 + 22 main columns (aux 4 / 0 / 3 EF columns) on mixed heights
    2^20 / 2^18 / 2^19, the 2^18 AIR with preprocessed columns (a tree shorter than the max LDE, virtually lifted),
    production parameters with full FRI -- bit-exact against the oracle prover."""
    import test_airs
    ob.lib().orc_set_threads(0)
    params = W.miden_pcs_params()
    lhs = (20, 18, 19)
    prep_prog = test_airs.preprocessed_workload((6,), (True,)).programs[0]
    t1 = W.synthetic_trace(71, lhs[1], 3)
    pm = W.synthetic_trace(72, lhs[1], 2)
    t1[:, 0] = _mulmod(pm[:, 0], t1[:, 1])
    t1[:, 2] = _addmod(np.roll(pm[:, 1], -1), t1[:, 1])
    traces = [W.synthetic_trace(70, lhs[0], 51), t1, W.synthetic_trace(73, lhs[2], 22)]
    wl = W.Workload(list(lhs), widths=[51, 3, 22], aux_widths=[4, 0, 3], traces=traces,
                    programs=[pkg.air_program.dummy_miden_air(), prep_prog, pkg.air_program.dummy_miden_air()],
                    log_quotient_degrees=[3, 1, 3], num_aux_values=[4, 0, 3], preprocessed=[None, pm, None])
    s = B.Session(params, 0)
    try:
        commitment = s.set_preprocessed(wl.statement, wl.preprocessed_matrices)
        _bit_exact_vs_oracle_prover(s, params, wl)
        assert np.array_equal(commitment, wl.oracle_prep_commitment)
    finally:
        s.close()


def test_config5_shape_2_22_with_preprocessed_verifies():
    """BASELINE config 5 shape (tallest trace 2^22, mixed heights, a preprocessed tree, full FRI with the
    production parameters): the proof must be accepted by the oracle verifier.  Narrower than the Miden widths so
    the host-side trace generation stays in seconds; the maximum supported height and the 11+11 NTT split are what
    is exercised."""
    import test_airs
    params = W.miden_pcs_params()
    s = B.Session(params, 0)
    lhs = (22, 18, 20)
    base = test_airs.preprocessed_workload((6, 6, 6), (True, False, True))       # programs only
    traces, preps = [], []
    for i, lh in enumerate(lhs):
        n = 1 << lh
        t = W.synthetic_trace(50 + i, lh, 3)
        if i != 1:
            pm = W.synthetic_trace(60 + i, lh, 2)
            t[:, 0] = _mulmod(pm[:, 0], t[:, 1])
            t[:, 2] = _addmod(np.roll(pm[:, 1], -1), t[:, 1])
            preps.append(pm)
        else:
            t[:, 0] = _mulmod(t[:, 1], t[:, 2])
            preps.append(None)
        traces.append(t)
    wl = W.Workload(list(lhs), widths=[3, 3, 3], aux_widths=[0, 0, 0], programs=base.programs, traces=traces,
                    log_quotient_degrees=[1, 1, 1], num_aux_values=[0, 0, 0], preprocessed=preps)
    commitment = s.set_preprocessed(wl.statement, wl.preprocessed_matrices)
    ch = W.initial_challenger(params, prod_observe)
    proof = s.prove(wl.statement, wl.matrices, ch)
    rc, err = H.oracle_verify(params, wl, ch, *proof, prep_commitment=commitment)
    assert rc == 0, err
    s.close()


def _mulmod(a, b):
    """Vectorised Goldilocks product of two uint64 arrays (Python-int object arrays would take minutes at 2^22)."""
    P = int(W.P)
    a = a.astype(np.uint64); b = b.astype(np.uint64)
    a0, a1 = a & np.uint64(0xFFFFFFFF), a >> np.uint64(32)
    b0, b1 = b & np.uint64(0xFFFFFFFF), b >> np.uint64(32)
    # 128-bit product limbs via float-free 32x32 partials
    p00 = a0 * b0; p01 = a0 * b1; p10 = a1 * b0; p11 = a1 * b1
    mid = (p00 >> np.uint64(32)) + (p01 & np.uint64(0xFFFFFFFF)) + (p10 & np.uint64(0xFFFFFFFF))
    lo = (p00 & np.uint64(0xFFFFFFFF)) | ((mid & np.uint64(0xFFFFFFFF)) << np.uint64(32))
    hi = p11 + (p01 >> np.uint64(32)) + (p10 >> np.uint64(32)) + (mid >> np.uint64(32))
    # reduce: lo - hh + hl * (2^32 - 1)   (2^64 = 2^32 - 1, 2^96 = -1 mod p); one pass of Python ints for the final mod
    hh, hl = hi >> np.uint64(32), hi & np.uint64(0xFFFFFFFF)
    res = (lo.astype(object) - hh.astype(object) + hl.astype(object) * 0xFFFFFFFF) % P
    return res.astype(np.uint64)


def _addmod(a, b):
    res = (a.astype(object) + b.astype(object)) % int(W.P)
    return res.astype(np.uint64)


def test_large_height_2_21_commit_root(lib, sess, oracle):
    """Heights above 2^20 (n1 = 10, n2 = 11 NTT split; BASELINE config 5 is 2^22): LMCS root of a narrow
    2^21-row matrix against the oracle."""
    lh, w = 21, 3
    m = rand_felts((1 << lh, w), 77)
    out = np.zeros(((1 << lh) << 3, w), dtype=np.uint64)
    om = ob.Matrix(ob.ptr(m.reshape(-1)), lh, w)
    oracle.orc_coset_lde_batch(C.byref(om), 3, oracle.orc_lde_shift(lh + 3), ob.ptr(out.reshape(-1)))
    bits = lh + 3
    idx = np.arange(1 << bits, dtype=np.uint64)
    rev = np.zeros_like(idx)
    for b in range(bits):
        rev |= ((idx >> np.uint64(b)) & np.uint64(1)) << np.uint64(bits - 1 - b)
    nat = np.ascontiguousarray(out[rev.astype(np.int64)])
    omat = (ob.Matrix * 1)(ob.Matrix(ob.ptr(nat.reshape(-1)), bits, w))
    exp = np.zeros(4, dtype=np.uint64)
    oracle.orc_lmcs_commit(omat, 1, ob.ptr(exp), None)
    pm = (B.Matrix * 1)(B.Matrix(B.ptr(m.reshape(-1)), lh, w))
    got = np.zeros(4, dtype=np.uint64)
    assert lib.mdn_lmcs_commit(sess.handle, pm, 1, B.ptr(got)) == 0, lib.mdn_last_error(sess.handle)
    assert np.array_equal(got, exp)


def test_non_canonical_input_rejected(lib, sess):
    wl = W.Workload([5], widths=(9,), aux_widths=(1,))
    wl.traces[0][7, 3] = np.uint64(P)          # not a canonical Felt
    ch = W.initial_challenger(W.miden_pcs_params(), prod_observe)
    with pytest.raises(B.ProverError) as e:
        sess.prove(wl.statement, wl.matrices, ch)
    assert "non-canonical" in str(e.value)
    # the session stays usable afterwards
    wl = W.Workload([5], widths=(9,), aux_widths=(1,))
    sess.prove(wl.statement, wl.matrices, ch)


def test_error_paths(lib, sess):
    wl = W.Workload([5], widths=(9,), aux_widths=(1,))
    wl._airs[0].width = 10   # trace width mismatch -> InstanceError
    ch = W.initial_challenger(W.miden_pcs_params(), prod_observe)
    with pytest.raises(B.ProverError):
        sess.prove(wl.statement, wl.matrices, ch)
    wl = W.Workload([5], widths=(9,), aux_widths=(1,), log_quotient_degrees=[4])   # > log_blowup: DomainError
    with pytest.raises(B.ProverError):
        sess.prove(wl.statement, wl.matrices, ch)
    # height above the supported maximum (2^22): rejected before any upload
    big = np.zeros((1 << 23, 1), dtype=np.uint64)
    wl = W.Workload([23], widths=(1,), aux_widths=(0,), traces=[big], programs=[AP_degree(1)], log_quotient_degrees=[1], num_aux_values=[0])
    with pytest.raises(B.ProverError, match="2\\^22"):
        sess.prove(wl.statement, wl.matrices, ch)
    # malformed constraint programs
    good = W.Workload([5], widths=(9,), aux_widths=(1,))
    for mutate in (lambda p: p.__setitem__(0, 0x12345678),            # magic
                   lambda p: p.__setitem__(5, 99),                    # unknown op
                   lambda p: p.__setitem__(6, 1000),                  # constant index out of range (node 0 is CONST)
                   lambda p: p.__setitem__(2, int(p[2]) + 1)):        # node count / length mismatch
        wl = W.Workload([5], widths=(9,), aux_widths=(1,))
        mutate(wl.programs[0])
        with pytest.raises(B.ProverError):
            sess.prove(wl.statement, wl.matrices, ch)
    # no AIRs at all
    empty = B.Statement(None, 0, None, 0, None, 0)
    with pytest.raises(B.ProverError):
        sess.prove(empty, good.matrices, ch)
    # a lookup program whose column count disagrees with aux_width
    import test_airs
    wl, _ = test_airs.logup_workload(5)
    wl._airs[0].aux_width = 2
    with pytest.raises(B.ProverError):
        sess.prove(wl.statement, wl.matrices, ch)
    # the session is still usable afterwards
    _compare_proofs(sess, W.miden_pcs_params(), good)


def test_gpu_matches_committed_golden_proofs():
    """The CUDA path against the committed fixtures (tests/golden/oracle_proofs.json), without
    running the oracle prover."""
    import importlib.util, json, os
    gdir = os.path.join(os.path.dirname(__file__), "golden")
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(gdir, "make_golden.py"))
    mg = importlib.util.module_from_spec(spec); spec.loader.exec_module(mg)
    gold = json.load(open(os.path.join(gdir, "oracle_proofs.json")))
    for name, params, wl, builder in mg.cases():
        s = B.Session(params, 0)
        try:
            ch = W.initial_challenger(params, prod_observe)
            cb = B.AUX_BUILDER(builder) if builder else None
            heights, fields, comms = s.prove(wl.statement, wl.matrices, ch, cb)
            g = gold[name]
            assert [int(x) for x in s.info(0)] == g["main_root"], name
            assert [int(x) for x in s.info(2)] == g["quotient_root"], name
            assert [int(x) for x in s.info(7)] == g["query_indices"], name
            assert mg.digest(heights, fields, comms) == g["proof_sha256"], name
        finally:
            s.close()


def test_staged_api_matches_one_shot(sess_fast):
    """mdn_prove_begin / _commit_aux / _finish (host drives the aux build itself) must give the same
    bytes as mdn_prove with a callback."""
    import test_airs
    lib = B.lib()
    params = W.fast_pcs_params()
    wl, builder = test_airs.fib_product_workload([6, 4], lqd=3)
    ch = W.initial_challenger(params, prod_observe)
    ref = sess_fast.prove(wl.statement, wl.matrices, ch, B.AUX_BUILDER(builder))
    root = np.zeros(4, dtype=np.uint64)
    rnd = np.zeros(4, dtype=np.uint64)
    h = sess_fast.handle
    assert lib.mdn_prove_begin(h, C.byref(wl.statement), wl.matrices, C.byref(ch), 0, B.ptr(root), B.ptr(rnd)) == 0, lib.mdn_last_error(h)
    # the host-side aux build, exactly what the callback does
    aux_bufs, val_bufs = [], []
    for i in range(wl.k):
        n = 1 << wl.log_heights[i]
        ab = np.zeros(n * 2 * wl.aux_widths[i], dtype=np.uint64)
        vb = np.zeros(2, dtype=np.uint64)
        assert builder(None, i, C.pointer(wl.matrices[i]), rnd.ctypes.data_as(B.u64p), ab.ctypes.data_as(B.u64p), vb.ctypes.data_as(B.u64p)) == 0
        aux_bufs.append(ab); val_bufs.append(vb)
    aux_m = (B.Matrix * wl.k)()
    vals = (B.u64p * wl.k)()
    for i in range(wl.k):
        aux_m[i] = B.Matrix(B.ptr(aux_bufs[i]), wl.log_heights[i], 2 * wl.aux_widths[i])
        vals[i] = B.ptr(val_bufs[i])
    aux_root = np.zeros(4, dtype=np.uint64)
    assert lib.mdn_prove_commit_aux(h, aux_m, vals, B.ptr(aux_root)) == 0, lib.mdn_last_error(h)
    proof = B.Proof()
    assert lib.mdn_prove_finish(h, C.byref(proof)) == 0, lib.mdn_last_error(h)
    got = B.proof_to_numpy(proof)
    assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2])
    assert np.array_equal(root, sess_fast.info(0)) and np.array_equal(aux_root, sess_fast.info(1))
    # out-of-order calls are rejected, not crashed
    assert lib.mdn_prove_finish(h, C.byref(proof)) != 0


def test_external_assertions_hook(sess_fast):
    """`Statement::eval_external` (mdn_session_set_external_check): called once per proof, after the aux traces exist --
    here the LogUp aux trace is built ON THE DEVICE, so its committed final reaches the host only through this call --
    and before the aux commitment; a failing assertion aborts the proof with MDN_ERR_EXTERNAL_ASSERTION
    (`ProverError::ExternalAssertionFailed`, prover/mod.rs:383-395) and the session stays usable."""
    import test_airs
    params = W.fast_pcs_params()
    wl, _ = test_airs.logup_workload(6, device=True)
    ch = W.initial_challenger(params, prod_observe)
    calls = []

    def ok(chal, aux_values, heights):
        calls.append((chal.copy(), [a.copy() for a in aux_values], heights))
        return None
    sess_fast.set_external_check(ok)
    try:
        heights, fields, comms = sess_fast.prove(wl.statement, wl.matrices, ch)
        assert len(calls) == 1
        chal, aux_values, hs = calls[0]
        assert len(chal) == 4 and hs == bytes(wl.log_heights) and len(aux_values) == 1 and len(aux_values[0]) == 2
        assert np.array_equal(aux_values[0], fields[:2])        # the device-built final is what gets committed next
        sess_fast.set_external_check(lambda c, a, h: 0)         # assertion 0 evaluates to non-zero
        with pytest.raises(B.ProverError, match=r"\[-7\] external assertion 0 failed"):
            sess_fast.prove(wl.statement, wl.matrices, ch)
    finally:
        sess_fast.set_external_check(None)
    again = sess_fast.prove(wl.statement, wl.matrices, ch)
    assert np.array_equal(again[1], fields) and np.array_equal(again[2], comms)


def test_non_canonical_statement_values_rejected(sess_fast):
    """Public values and observed statement felts must be canonical (< p), like every other input (ADVICE r1)."""
    params = W.fast_pcs_params()
    ch = W.initial_challenger(params, prod_observe)
    wl = W.Workload([5], widths=(9,), aux_widths=(1,), public_values=(1, 2))
    wl.public_values[1] = np.uint64(P)
    with pytest.raises(B.ProverError, match=r"\[-1\] public value 1"):
        sess_fast.prove(wl.statement, wl.matrices, ch)
    wl.public_values[1] = 2
    wl.observe_felts[0] = np.uint64(2**64 - 1)
    with pytest.raises(B.ProverError, match=r"\[-1\] observed statement felt 0"):
        sess_fast.prove(wl.statement, wl.matrices, ch)


def test_two_sessions_are_independent():
    params = W.fast_pcs_params()
    a, b = B.Session(params, 0), B.Session(params, 0)
    try:
        wl1 = W.Workload([6], widths=(9,), aux_widths=(1,), seed=1)
        wl2 = W.Workload([5, 7], widths=(9, 10), aux_widths=(1, 2), seed=2)
        ch = W.initial_challenger(params, prod_observe)
        p1 = a.prove(wl1.statement, wl1.matrices, ch)
        p2 = b.prove(wl2.statement, wl2.matrices, ch)
        q2 = a.prove(wl2.statement, wl2.matrices, ch)      # sessions are reusable across statements
        q1 = b.prove(wl1.statement, wl1.matrices, ch)
        assert np.array_equal(p1[1], q1[1]) and np.array_equal(p2[1], q2[1])
        assert np.array_equal(p1[2], q1[2]) and np.array_equal(p2[2], q2[2])
    finally:
        a.close(); b.close()


def test_split_proof_matches_single_gpu():
    """mdn_session_set_shard: the same proof split over 2 GPUs (LDE cosets + Merkle sub-trees per rank, peer-memory
    stores over NVLink, device barrier) must be byte-identical.  Needs two visible GPUs; skips on a one-GPU machine."""
    import os, subprocess, sys, torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", "29533", os.path.join(root, "tests", "run_sharded.py")],
                         capture_output=True, text=True, timeout=900)
    assert "SHARDED_OK world 2" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]

