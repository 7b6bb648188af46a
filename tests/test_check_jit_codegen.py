"""The trace-check mode of the constraint JIT (jit.hpp MODE_CHECK) on the host: tests/cpp_jitcheck generates the source
of k_jit_check / k_jit_census for a constraint program and compiles it with NVRTC for sm_90a, with no device.  Every
leaf kind, a chunked program and a program past the census's shared-tally bound must compile to a cubin holding both
entry points with no local memory.  Execution against the interpreter is in tests/test_check_jit.py."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import pkgload
import test_airs as TA
import test_constraint_census as TCC

ROOT = pkgload.ROOT
D = os.path.join(ROOT, "tests", "cpp_jitcheck")


def programs():
    wl, _ = TA.fib_product_workload([5])
    logup, _ = TA.logup_workload(5)
    return {
        "fib_product": wl.programs[0],                               # aux, challenges, publics, selectors, aux values
        "periodic": TA.periodic_workload(5).programs[0],
        "preprocessed": TA.preprocessed_workload().programs[0],
        "logup_main": logup.programs[0],                             # mixed base / extension arithmetic
        "chunked_2k": TA.big_program_workload(5, n_terms=60).programs[0],
        "constraints_300": TCC._wide_program(300),                   # > CENSUS_SHARED_K: the global tally
    }


@pytest.fixture(scope="module")
def driver():
    subprocess.check_call(["make", "-s", "-C", D, "test_jitcheck"])
    return os.path.join(D, "test_jitcheck")


@pytest.mark.parametrize("name", list(programs()))
def test_check_kernels_compile(driver, tmp_path, name):
    prog = programs()[name]
    src = tmp_path / "prog.bin"
    np.ascontiguousarray(prog, dtype=np.uint32).tofile(src)
    r = subprocess.run([driver, str(src), "check", str(tmp_path / "out")], capture_output=True, text=True, timeout=900)
    if "NVRTC unavailable" in r.stdout:
        pytest.skip(r.stdout.strip())
    assert r.returncode == 0 and r.stdout.startswith("JITCHECK "), r.stdout + r.stderr
    info = dict(kv.split("=") for kv in r.stdout.split()[1:])
    if name == "chunked_2k":
        assert int(info["chunks"]) > 1 and int(info["spill_base"]) + int(info["spill_ext"]) > 0
    source = (tmp_path / "out.cu").read_text()
    for entry in ("k_jit_check", "k_jit_census"):
        assert f'extern "C" __global__ void __launch_bounds__(128) {entry}(' in source
    assert source.count(" tally(a, sh, (u32)pos, ") == int(prog[3])     # one non-zero test per constraint
    assert "finv(" not in source.split("struct Ctx")[1]                  # exact selectors: no Lagrange evaluation
    cubin = (tmp_path / "out.cubin").read_bytes()
    assert b"k_jit_check" in cubin and b"k_jit_census" in cubin
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        return
    usage = subprocess.run([cuobjdump, "--dump-resource-usage", str(tmp_path / "out.cubin")], capture_output=True,
                           text=True, timeout=300).stdout
    for entry in ("k_jit_check", "k_jit_census"):
        m = re.search(r"Function %s:\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)" % entry, usage)
        assert m, usage
        assert int(m.group(4)) == 0, usage                               # only the chunk calls' stack frames
        assert (int(m.group(3)) >= 4 * 3 * 256 + 4) if entry == "k_jit_census" else int(m.group(3)) == 0   # the block's tallies
