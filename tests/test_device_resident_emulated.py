"""Column-major device traces and the device aux builder on the CPU kernel emulator of tests/emu (TEST INFRASTRUCTURE;
see tests/test_emulated.py): the small cases of tests/test_device_resident.py -- proofs, the constraint check, the error
paths -- with device memory being host memory, and one proof split over two ranks."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")


def _build():
    subprocess.check_call(["make", "-s", "-C", EMU])
    return os.path.join(EMU, "libmiden_b200_emu.so")


def test_device_resident_cases_on_the_emulator():
    """The -m gpu cases of tests/test_device_resident.py that fibers can run (no 2^20 / 2^22, no NVRTC, no CUDA kernel)."""
    env = dict(os.environ, MDN_LIB_PATH=_build(), MDN_ALLOW_EMULATOR="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_device_resident.py"), "-q", "-m", "gpu",
                        "-k", "not 2_20 and not 2_22 and not jit and not cpp", "-p", "no:cacheprovider"],
                       env=env, capture_output=True, text=True, timeout=2400, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]


def test_split_proof_from_column_major_device_traces_on_the_emulator():
    """ONE proof split over two ranks, each ingesting its own whole copy of the column-major traces, is byte-identical to
    the unsplit proof from host traces (tests/run_sharded_device.py over gloo and POSIX shared memory)."""
    env = dict(os.environ, MDN_LIB_PATH=_build(), MDN_ALLOW_EMULATOR="1", MDN_EMU_SHM="1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29741", os.path.join(ROOT, "tests", "run_sharded_device.py")],
                       env=env, capture_output=True, text=True, timeout=1200, cwd=ROOT)
    assert r.returncode == 0 and "SHARDED_DEVICE_OK world=2" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
