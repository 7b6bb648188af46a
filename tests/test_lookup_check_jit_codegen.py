"""The lookup-check mode of the JIT (jit.hpp MODE_LOOKUP_CHECK) on the host: tests/cpp_jitlookup generates the source of
k_jit_balance / k_jit_fold / k_jit_fold_census for a lowered lookup program and compiles it with NVRTC for sm_90a, with
no device.  A program with every leaf kind, a chunked program whose values cross chunk boundaries and a 16-column
program must compile to a cubin holding the three entry points with no local memory, and call the interaction hook once
per interaction.  Execution against the interpreter is in tests/test_lookup_check_jit.py."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import pkgload
import test_trace_balance as TB

pkg = pkgload.load_pkg()
AP, P = pkg.air_program, pkg.workload.P
ROOT = pkgload.ROOT
D = os.path.join(ROOT, "tests", "cpp_jitlookup")
ENTRIES = ("k_jit_balance", "k_jit_fold", "k_jit_fold_census")


def every_leaf():
    """main rows r and r + 1, a public value, challenges, base and extension constants, a periodic column and
    preprocessed rows r and r + 1; flagged and flag-free interactions over two columns, one cached group."""
    lb = AP.LookupProgramBuilder(2)
    with lb.group(0):
        lb.insert(0, lb.main(0, 0), lb.const(1), lb.encode(0, 4, [lb.main(1, 1), lb.public(0), lb.periodic(0)]))
    with lb.group(1, cached=True):
        lb.insert(1, lb.main(0, 2), lb.const(P - 1), lb.encode(1, 4, [lb.preprocessed(0, 0), lb.preprocessed(1, 1)]))
        lb.insert(1, lb.const(1) - lb.main(0, 2), lb.main(0, 3), lb.ext_const(5, 9) + lb.challenge(1))
    lb.insert(1, None, lb.main(1, 3), lb.main(0, 4))
    return lb.serialize()


def sixteen_columns():
    lb = AP.LookupProgramBuilder(16)
    for c in range(16):
        with lb.group(c):
            lb.insert(c, lb.main(0, c), lb.const(c + 1), lb.encode(c % 4, 16, [lb.main(1, (c + i) % 16) for i in range(16)]))
    return lb.serialize()


def programs():
    return {"every_leaf": (every_leaf(), None), "bus_sender": (TB.sender_lookup().serialize(), None),
            "bus_sender_chunked": (TB.sender_lookup().serialize(), "6"), "sixteen_columns": (sixteen_columns(), None)}


@pytest.fixture(scope="module")
def driver():
    subprocess.check_call(["make", "-s", "-C", D, "test_jitlookup"])
    return os.path.join(D, "test_jitlookup")


@pytest.mark.parametrize("name", list(programs()))
def test_lookup_check_kernels_compile(driver, tmp_path, name):
    prog, chunk = programs()[name]
    src = tmp_path / "prog.bin"
    np.ascontiguousarray(prog, dtype=np.uint32).tofile(src)
    env = dict(os.environ)
    env.pop("MDN_JIT_CHUNK", None)
    if chunk:
        env["MDN_JIT_CHUNK"] = chunk
    r = subprocess.run([driver, str(src), "lookup-check", str(tmp_path / "out")], capture_output=True, text=True,
                       timeout=900, env=env)
    if "NVRTC unavailable" in r.stdout:
        pytest.skip(r.stdout.strip())
    assert r.returncode == 0 and r.stdout.startswith("JITLOOKUP "), r.stdout + r.stderr
    info = dict(kv.split("=") for kv in r.stdout.split()[1:])
    if chunk:
        assert int(info["chunks"]) > 1 and int(info["spill_base"]) + int(info["spill_ext"]) > 0
    assert int(info["cols"]) == 1 + max(int(prog[5 + 3 * int(prog[2]) + 4 * q]) for q in range(int(prog[3])))
    source = (tmp_path / "out.cu").read_text()
    for entry in ENTRIES:
        assert f'extern "C" __global__ void __launch_bounds__(128) {entry}(' in source
    # one hook call per interaction, in interaction order, each with its literal index
    calls = [int(k) for k in re.findall(r"  lk_hook\(a, pos, st, (\d+)u, ", source)]
    assert calls == list(range(int(prog[3])))
    cubin = (tmp_path / "out.cubin").read_bytes()
    assert all(e.encode() in cubin for e in ENTRIES)
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        return
    usage = subprocess.run([cuobjdump, "--dump-resource-usage", str(tmp_path / "out.cubin")], capture_output=True,
                           text=True, timeout=300).stdout
    for entry in ENTRIES:
        m = re.search(r"Function %s:\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)" % entry, usage)
        assert m, usage
        assert int(m.group(4)) == 0, usage                               # only the chunk calls' stack frames
        if entry == "k_jit_fold_census":                                 # the block's per-column tallies
            assert int(m.group(3)) >= 4 * 4 * int(info["cols"]) + 4, usage


def test_other_modes_do_not_emit_the_lookup_check_code(driver, tmp_path):
    """The LogUp mode's source of the same program carries none of the lookup-check prelude or entry points."""
    prog = TB.sender_lookup().serialize()
    src = tmp_path / "prog.bin"
    np.ascontiguousarray(prog, dtype=np.uint32).tofile(src)
    r = subprocess.run([driver, str(src), "lookup-source", str(tmp_path / "lk")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    text = (tmp_path / "lk.cu").read_text()
    assert "LookupCheckJitArgs" not in text and "lk_hook" not in text and "k_jit_balance" not in text
