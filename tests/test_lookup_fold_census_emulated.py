"""The LogUp fold census on the CPU kernel emulator of tests/emu (TEST INFRASTRUCTURE; see tests/test_emulated.py): the
small -m gpu cases of tests/test_lookup_fold_census.py -- every single and multi-fault trace against both references in
host row-major, row-major device and column-major device layout, without fold marks, truncation, `first` against the
fold check, repeated calls, the error paths and the proof afterwards -- with device memory being host memory.  The 2^20
case is left to the GPU."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")


def test_lookup_fold_census_cases_on_the_emulator():
    subprocess.check_call(["make", "-s", "-C", EMU])
    env = dict(os.environ, MDN_LIB_PATH=os.path.join(EMU, "libmiden_b200_emu.so"), MDN_ALLOW_EMULATOR="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_lookup_fold_census.py"), "-q", "-m", "gpu",
                        "-k", "not 2_20", "-p", "no:cacheprovider"],
                       env=env, capture_output=True, text=True, timeout=2400, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]
