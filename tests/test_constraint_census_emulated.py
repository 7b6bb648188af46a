"""The constraint census on the CPU kernel emulator of tests/emu (TEST INFRASTRUCTURE; see tests/test_emulated.py): the
small -m gpu cases of tests/test_constraint_census.py -- every valid, single-fault and multi-fault statement against both
references, the three trace layouts, repeat calls, truncation, the error paths and the proofs around a census -- with
device memory being host memory.  The 2^20 cases are left to the GPU."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")


def test_constraint_census_cases_on_the_emulator():
    subprocess.check_call(["make", "-s", "-C", EMU])
    env = dict(os.environ, MDN_LIB_PATH=os.path.join(EMU, "libmiden_b200_emu.so"), MDN_ALLOW_EMULATOR="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_constraint_census.py"), "-q", "-m", "gpu",
                        "-k", "not h100", "-p", "no:cacheprovider"],
                       env=env, capture_output=True, text=True, timeout=2400, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]
