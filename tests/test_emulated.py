"""The -m gpu parity tests, small cases, on the CPU kernel emulator of tests/emu (TEST INFRASTRUCTURE).

tests/emu compiles the product's kernels.cu and session.cu with g++ against a stand-in <cuda_runtime.h>; every CUDA
thread of a block is a cooperative fiber, __syncthreads() and warp shuffles go through a block scheduler, device memory
is host memory.  The same launch geometry, shared-memory tiles, barriers and host orchestration run as on the GPU, so
these tests cover what the oracle tests cannot reach without a device: session.cu (phases, arena, tables, openings,
staged API, error paths) and the index arithmetic of every kernel, against the oracle, bit for bit.  What they cannot
show is listed in tests/emu/cuda_runtime.h (PTX carry primitives, hardware limits, races, speed); the real parity
gate stays `-m gpu` on an H100.  binding.py refuses the emulator library unless MDN_ALLOW_EMULATOR=1."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
# too large for fibers (2^20 and up), need the CUDA driver (NVRTC kernels), or need several processes.  The 2^16 case of
# BASELINE config 2 (two-pass NTT, 8.4 M permutations) takes two more minutes and runs with MDN_EMU_FULL=1.
SKIP = "not 2_20 and not 2_21 and not 2_22 and not full_size and not sharded and not split_proof and not jit" + ("" if os.environ.get("MDN_EMU_FULL") else " and not 2_16")


def _build():
    subprocess.check_call(["make", "-s", "-C", EMU])
    return os.path.join(EMU, "libmiden_b200_emu.so")


# The four single-process suites are started together by whichever of their tests runs first and collected by each test
# (they are independent python processes; running them side by side keeps the CPU suite within a few minutes).
_SUITES = {
    "parity": ["test_gpu_parity.py", SKIP, "300"],
    "blake3": ["test_blake3.py", "not 2_16", "600"],
    "keccak": ["test_keccak.py", "not 2_16", "600"],
    # every RPO case; RPX differs in the permutation only: one proof case and the hash-switch test (the GPU suite runs all of them)
    "rescue": ["test_rescue.py", "rpo or two_heights or switch", "900"],
}
_jobs = {}


def _suite(name):
    if not _jobs:
        lib = _build()
        env = dict(os.environ, MDN_LIB_PATH=lib, MDN_ALLOW_EMULATOR="1")
        for key, (file, expr, tmo) in _SUITES.items():
            _jobs[key] = subprocess.Popen([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", file), "-q", "-m", "gpu", "-k", expr,
                                           "-p", "no:cacheprovider", "--timeout", tmo], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, cwd=ROOT)
    out, err = _jobs[name].communicate(timeout=2400)
    assert _jobs[name].returncode == 0 and " passed" in out and "failed" not in out, out[-3000:] + err[-1000:]


def test_binding_refuses_the_emulator_without_opt_in():
    lib = _build()
    env = dict(os.environ, MDN_LIB_PATH=lib)
    env.pop("MDN_ALLOW_EMULATOR", None)
    code = ("import sys; sys.path.insert(0, %r); import pkgload; B = pkgload.load_pkg().binding\n"
            "try:\n    B.lib(); print('LOADED')\nexcept B.BackendMissing as e:\n    print('REFUSED', e)\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert "REFUSED" in r.stdout and "no CPU fallback" in r.stdout, r.stdout + r.stderr


def test_gpu_parity_suite_on_the_emulator():
    """tests/test_gpu_parity.py (-m gpu, the sizes fibers can run) on the emulator."""
    _suite("parity")


def test_blake3_configuration_on_the_emulator():
    """The Blake3_256 configuration (chaining-hasher LMCS, blake3 nodes, hash challenger, PoW through the hash challenger):
    the -m gpu cases of tests/test_blake3.py on the emulator, bit-exact against the oracle in Blake3 mode."""
    _suite("blake3")


def test_keccak_configuration_on_the_emulator():
    """The Keccak configuration (stateful sponge with rate 17 / alignment 17 and 25 lanes of state between height groups,
    PaddingFreeSponge nodes, Keccak-256 hash challenger and proof-of-work): the -m gpu cases of tests/test_keccak.py on the
    emulator, bit-exact against the oracle in Keccak mode."""
    _suite("keccak")


def test_rpo_rpx_configurations_on_the_emulator():
    """`rpo_config` / `rpx_config`: the Poseidon2 kernels instantiated with the Rescue permutations (leaf sponge, nodes, FRI
    leaves, proof-of-work) and the duplex challenger with them: the -m gpu cases of tests/test_rescue.py on the emulator."""
    _suite("rescue")


@pytest.mark.parametrize("world,min_log", [(2, None), (4, 2), (8, None)])
def test_one_proof_split_over_ranks_on_the_emulator(world, min_log):
    """ONE proof split over `world` ranks (mdn_session_set_shard: LDE cosets, leaf sponge, constraints, quotient chunks,
    DEEP and FRI folds per coset; Merkle sub-trees per leaf range; peer-memory stores ordered by the device barrier) is
    byte-identical to the unsplit proof -- the product's N>1 path, here with one emulated device per process, gloo as
    the bootstrap transport and POSIX shared memory standing in for the CUDA IPC mappings (on the GPU box:
    test_split_proof_matches_single_gpu).  min_log = 2 keeps even tiny FRI layers split, so the rank-local folds, the
    split FRI trees and the first-replicated-layer store are exercised at every round of a small proof; the stage
    outputs (roots, quotient accumulator, DEEP evaluations, FRI roots, query indices) are compared as well."""
    lib = _build()
    env = dict(os.environ, MDN_LIB_PATH=lib, MDN_ALLOW_EMULATOR="1", MDN_EMU_SHM="1", SHARD_LOG_H="9", OMP_NUM_THREADS="1")
    env.pop("SHARD_BENCH", None)
    if min_log is not None:
        env.update(MDN_SHARD_MIN_LOG=str(min_log), SHARD_DEBUG_STAGES="1")
    else:
        env["SHARD_SUBSET"] = "1"      # the full case list runs at world 4 (and on the GPU box); worlds 2 and 8 run one case per feature
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29711 + world),
                        os.path.join(ROOT, "tests", "run_sharded.py")],
                       env=env, capture_output=True, text=True, timeout=1200, cwd=ROOT)
    assert r.returncode == 0 and f"SHARDED_OK world={world}" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def test_cpp_host_layer_prove_verify_tamper_on_the_emulator():
    """miden-vm_b200/host/miden_prover.hpp (the reference's prover interface restated in C++ above the C ABI) through its
    parity program tests/cpp/test_host_api.cpp, linked against the emulator: StarkConfig / ProverStatement /
    Preprocessed / ProverInstance::prove, verified by the oracle, tampered proofs rejected."""
    _build()
    cpp = os.path.join(ROOT, "tests", "cpp")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])
    subprocess.check_call(["make", "-s", "-C", cpp, "test_host_api_emu"])
    r = subprocess.run([os.path.join(cpp, "test_host_api_emu")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "HOST_API_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_graft_entry_smoke_on_the_emulator():
    """__graft_entry__.smoke() (one small proof through the C ABI, checked against the oracle) runs unchanged."""
    lib = _build()
    env = dict(os.environ, MDN_LIB_PATH=lib, MDN_ALLOW_EMULATOR="1")
    r = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.smoke()"], env=env, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "smoke ok" in r.stdout, r.stdout[-1500:] + r.stderr[-1500:]
