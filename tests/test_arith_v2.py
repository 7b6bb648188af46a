"""The device arithmetic (miden-vm_b200/csrc/poseidon2_fast2.cuh) is written as
__host__ __device__ code whose only device-specific parts are five carry-flag primitives.  This test
compiles THAT header for the CPU (tests/cpp/test_arith_v2.cpp) and checks multiplication, the wide
accumulators, exact division by 2^k, the external layer and the whole permutation against 128-bit integer
arithmetic, the canonical p2::permute and the reference KAT (poseidon2/test.rs:7-39), on canonical and
non-canonical representatives.  The GPU side of the same header is what the -m gpu parity tests run."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")


def test_arith_v2_on_host():
    """The product build (lanes 1..11 of the 22 internal rounds kept as unreduced 96-bit values) and the same with the
    bound instrumentation (largest lane value tracked)."""
    for target in ("test_arith_v2", "test_arith_v2_lazy"):
        subprocess.check_call(["make", "-s", "-C", CPP, target])
        r = subprocess.run([os.path.join(CPP, target)], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and "ARITH_V2_OK" in r.stdout, target + ": " + r.stdout + r.stderr
        if target == "test_arith_v2_lazy":
            assert "largest lane high word seen" in r.stdout


def test_ntt_v2_block_functions_on_host():
    """ntt2.cuh (the bodies of the product's NTT kernels) run on the CPU with the tables of ntt_tables.hpp: inverse
    transform and all cosets of the LDE for 2^1 .. 2^16 (both the single-pass and the two-pass split) against a
    textbook transform; also pins the table layout ntt_tables.hpp builds."""
    subprocess.check_call(["make", "-s", "-C", CPP, "test_ntt_v2"])
    r = subprocess.run([os.path.join(CPP, "test_ntt_v2"), "19"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "NTT_V2_OK" in r.stdout, r.stdout + r.stderr
