"""Register columns of version-2 lookup programs on the CPU kernel emulator of tests/emu (TEST INFRASTRUCTURE; see
tests/test_emulated.py): the -m gpu cases of tests/test_lookup_registers.py -- proofs against the host builder and the
oracle, the trace layouts, the staged API, the guard, the wrong lowering, the three lookup checks and the refusals --
with device memory being host memory, and proofs split over 2 and 4 ranks (tests/run_lookup_registers_sharded.py over
gloo and POSIX shared memory).  The NVRTC, 2^17 and 2^20 cases are left to the GPU."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")


def _env(**extra):
    subprocess.check_call(["make", "-s", "-C", EMU])
    return dict(os.environ, MDN_LIB_PATH=os.path.join(EMU, "libmiden_b200_emu.so"), MDN_ALLOW_EMULATOR="1", **extra)


def test_lookup_register_cases_on_the_emulator():
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_lookup_registers.py"), "-q", "-m", "gpu",
                        "-k", "not 2_20 and not 2_17 and not jit", "-p", "no:cacheprovider"],
                       env=_env(), capture_output=True, text=True, timeout=2400, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]


@pytest.mark.parametrize("world", [2, 4])
def test_split_proofs_on_the_emulator(world):
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29781 + world),
                        os.path.join(ROOT, "tests", "run_lookup_registers_sharded.py")],
                       env=_env(MDN_EMU_SHM="1", OMP_NUM_THREADS="1"), capture_output=True, text=True, timeout=1200, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.count("LOOKUP_REGISTERS_SHARDED_OK") == world, r.stdout[-2000:] + r.stderr[-3000:]
