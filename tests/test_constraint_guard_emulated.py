"""The constraint guard on the CPU kernel emulator of tests/emu (TEST INFRASTRUCTURE; see tests/test_emulated.py): the
small -m gpu cases of tests/test_constraint_guard.py -- identical proofs with the guard on every trace source and hash
configuration, the refusals and their reports, the staged API and the error paths -- with device memory being host
memory, and proofs split over 2 and 4 ranks (tests/run_guard_sharded.py over gloo and POSIX shared memory).  The 2^20
case is left to the GPU."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")


def _env(**extra):
    subprocess.check_call(["make", "-s", "-C", EMU])
    return dict(os.environ, MDN_LIB_PATH=os.path.join(EMU, "libmiden_b200_emu.so"), MDN_ALLOW_EMULATOR="1", **extra)


def test_constraint_guard_cases_on_the_emulator():
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_constraint_guard.py"), "-q", "-m", "gpu",
                        "-k", "not h100", "-p", "no:cacheprovider"],
                       env=_env(), capture_output=True, text=True, timeout=2400, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]


@pytest.mark.parametrize("world", [2, 4])
def test_split_proofs_on_the_emulator(world):
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29751 + world),
                        os.path.join(ROOT, "tests", "run_guard_sharded.py")],
                       env=_env(MDN_EMU_SHM="1", OMP_NUM_THREADS="1"), capture_output=True, text=True, timeout=1200, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.count("GUARD_SHARDED_OK") == world, r.stdout[-2000:] + r.stderr[-3000:]
