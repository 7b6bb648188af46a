"""The persistent NVRTC cubin cache (mdn_jit_set_cache_dir, mdn_get_info(NULL, MDN_INFO_JIT_CACHE)).

Every process here is a fresh subprocess (tests/run_jit_cache.py) on a tmp_path directory, so that nothing comes from
the in-memory cubin cache.  The CPU tests compile through mdn_jit_compile_check, which needs no device, on a constraint
program and a lookup program just over 256 nodes.  The GPU test runs every kind of NVRTC row pass in a cold process,
a warm one and a warm one under MDN_JIT_FORCE_DISAGREE=1."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import pkgload
import test_airs as TA

pkg = pkgload.load_pkg()
W, B, AP = pkg.workload, pkg.binding, pkg.air_program
RUN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "run_jit_cache.py")
HEADER = 88      # jit.hpp DiskHeader: magic[8], format, reserved, key[8], cubin bytes, cubin hash[8]


def constraint_program():
    p = TA.big_program_workload(5, n_terms=7).programs[0]
    assert p[2] > 256
    return p


def lookup_program():
    lb = AP.LookupProgramBuilder(2)
    acc = lb.main(0, 0)
    for i in range(60):
        acc = acc * lb.main(i % 2, i % 4) + lb.const(i + 1)
    lb.insert(0, lb.main(0, 4), lb.const(1), lb.encode(0, 2, [acc, lb.main(0, 1)]))
    lb.insert(1, None, -lb.main(0, 5), lb.encode(0, 2, [lb.main(0, 2), lb.main(0, 3)]))
    p = lb.serialize()
    assert p[2] > 256
    return p


def save(tmp_path, name, prog):
    path = tmp_path / f"{name}.npy"
    np.save(path, np.ascontiguousarray(prog, dtype=np.uint32))
    return str(path)


def start(args, env=None):
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.Popen([sys.executable, RUN] + [str(a) for a in args], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                            text=True, env=e)


def finish(p):
    out, err = p.communicate(timeout=1800)
    assert p.returncode == 0, out + err
    return json.loads(out.strip().splitlines()[-1])


def run(args, env=None):
    return finish(start(args, env))


def compile_in(d, progs, env=None):
    r = run(["compile", d] + progs, env)
    for v in r["results"]:
        if isinstance(v, str) and "NVRTC unavailable" in v:
            pytest.skip(v)
    return r


def entries(d):
    return {f: (d / f).read_bytes() for f in os.listdir(d)}


def counts(r):
    s = r["stats"]
    return s["disk_hits"], s["disk_misses"], s["rejected"], s["write_failures"], s["compiles"]


@pytest.fixture
def progs(tmp_path):
    return [save(tmp_path, "constraints", constraint_program()), save(tmp_path, "lookup", lookup_program())]


@pytest.fixture
def cache(tmp_path):
    d = tmp_path / "cache"
    d.mkdir()
    return d


def test_cold_then_warm(cache, progs):
    cold = compile_in(cache, progs)
    assert counts(cold) == (0, 2, 0, 0, 2)
    assert all(isinstance(v, int) and v > 1000 for v in cold["results"]), cold
    files = entries(cache)
    assert len(files) == 2 and all(f.endswith(".cubin") and len(f) == 64 + 6 for f in files)
    warm = compile_in(cache, progs)
    assert counts(warm) == (2, 0, 0, 0, 0) and warm["stats"]["compile_ms"] == 0
    assert warm["results"] == cold["results"]
    assert entries(cache) == files


@pytest.mark.parametrize("change", ["ptxas", "chunk", "program"])
def test_key_follows_what_nvrtc_is_given(cache, progs, tmp_path, change):
    base = compile_in(cache, progs[:1])
    assert counts(base) == (0, 1, 0, 0, 1)
    before = entries(cache)
    env, prog = {}, progs[:1]
    if change == "ptxas":
        env = {"MDN_JIT_PTXAS": "-O2"}
    elif change == "chunk":
        env = {"MDN_JIT_CHUNK": "64"}
    else:
        p = constraint_program().copy()
        consts = 5 + 3 * int(p[2]) + int(p[3])        # the first constant's low word
        p[consts] ^= 1
        prog = [save(tmp_path, "changed", p)]
    r = compile_in(cache, prog, env)
    assert counts(r) == (0, 1, 0, 0, 1)
    after = entries(cache)
    assert len(after) == 2 and all(after[f] == before[f] for f in before)
    again = compile_in(cache, prog, env)              # the new entry is found under the same inputs
    assert counts(again) == (1, 0, 0, 0, 0)


def _flip_payload(b):
    b = bytearray(b); b[HEADER + len(b[HEADER:]) // 2] ^= 0x40; return bytes(b)


def _wrong_key(b):
    b = bytearray(b); b[16] ^= 1; return bytes(b)


DAMAGE = {
    "flipped_payload_byte": _flip_payload,
    "truncated": lambda b: b[: len(b) - 17],
    "wrong_magic": lambda b: b"X" + b[1:],
    "key_not_its_name": _wrong_key,
}


@pytest.mark.parametrize("damage", list(DAMAGE))
def test_damaged_file_is_rejected_and_replaced(cache, progs, damage):
    compile_in(cache, progs[:1])
    (name, good), = entries(cache).items()
    (cache / name).write_bytes(DAMAGE[damage](good))
    r = compile_in(cache, progs[:1])
    assert counts(r) == (0, 1, 1, 0, 1)
    assert entries(cache) == {name: good}


def test_off_by_default(tmp_path, progs):
    r = compile_in("-", progs)
    s = r["stats"]
    assert (s["disk_hits"], s["disk_misses"], s["rejected"], s["write_failures"]) == (0, 0, 0, 0)
    assert s["compiles"] == 2
    assert sorted(os.listdir(tmp_path)) == ["constraints.npy", "lookup.npy"]


def test_bad_directory_is_refused(tmp_path):
    regular = tmp_path / "file"
    regular.write_text("x")
    for bad in (tmp_path / "missing", regular):
        with pytest.raises(B.ProverError) as e:
            B.set_jit_cache_dir(str(bad))
        assert "[-1]" in str(e.value) and str(bad) in str(e.value)
    assert B.lib().mdn_jit_set_cache_dir(str(regular).encode()) == -1       # MDN_ERR_INVALID_ARG
    B.set_jit_cache_dir(None)
    B.set_jit_cache_dir("")
    assert B.jit_cache_stats()["disk_hits"] == 0


def test_stats_need_no_session():
    s = B.jit_cache_stats()
    assert set(s) == {"disk_hits", "disk_misses", "rejected", "write_failures", "compiles", "compile_ms"}
    assert B.lib().mdn_get_info(None, 8, None, 0) == -1      # MDN_INFO_JIT: every other kind still needs a session


@pytest.mark.skipif(hasattr(os, "geteuid") and os.geteuid() == 0, reason="root ignores directory permissions")
def test_unwritable_directory(cache, progs):
    want = compile_in("-", progs[:1])["results"]
    os.chmod(cache, 0o555)
    try:
        r = compile_in(cache, progs[:1])
    finally:
        os.chmod(cache, 0o755)
    assert counts(r) == (0, 1, 0, 1, 1)
    assert r["results"] == want and os.listdir(cache) == []


def test_concurrent_writers(cache, progs):
    ps = [start(["compile", cache] + progs[:1]) for _ in range(2)]
    rs = [finish(p) for p in ps]
    assert rs[0]["results"] == rs[1]["results"]
    files = os.listdir(cache)
    assert len(files) == 1 and files[0].endswith(".cubin") and not files[0].startswith(".")
    warm = compile_in(cache, progs[:1])
    assert counts(warm) == (1, 0, 0, 0, 0) and warm["results"] == rs[0]["results"]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: three fresh processes on one directory
# ---------------------------------------------------------------------------------------------------------------------
PROOF = "NVRTC kernel disagreed with the interpreter on its first use; interpreter kept"
LOGUP = "NVRTC lookup kernel disagreed with the interpreter on its first use; interpreter kept"
CHECK = "NVRTC check kernel disagreed with the interpreter on its first use; interpreter kept"
LOOKUP_CHECK = "NVRTC lookup-check kernel disagreed with the interpreter on its first use; interpreter kept"


@pytest.mark.gpu
def test_warm_process_loads_every_kernel_from_disk(cache, tmp_path):
    def gpu_run(name, env=None):
        out = tmp_path / f"{name}.json"
        run(["gpu", cache, out], env)
        return json.loads(out.read_text())

    cold = gpu_run("cold")
    c = cold["stats"]
    assert c["disk_misses"] > 0 and c["compiles"] == c["disk_misses"] and c["disk_hits"] == 0, c
    assert c["rejected"] == 0 and c["write_failures"] == 0
    assert len(os.listdir(cache)) == c["disk_misses"]
    files = entries(cache)

    warm = gpu_run("warm")
    w = warm["stats"]
    assert w["compiles"] == 0 and w["disk_misses"] == 0 and w["disk_hits"] == c["disk_misses"], w
    fl = warm["flags"]
    assert fl == cold["flags"]
    for k in ("guarded_proof", "guarded_proof_check", "proof", "census"):
        assert fl[k] and all(v == 1 for v in fl[k]), fl
    for k in ("balance", "fold_census"):
        assert fl[k] == fl[k + "_lookups"] and any(fl[k]), fl
    assert all(n == "" for n in warm["notes"].values()), warm["notes"]
    assert warm["outputs"] == cold["outputs"] == warm["interpreter_outputs"]
    assert warm["outputs"]["guarded_proof"] == warm["outputs"]["proof"]
    assert entries(cache) == files

    forced = gpu_run("forced", {"MDN_JIT_FORCE_DISAGREE": "1"})
    f = forced["stats"]
    assert f["compiles"] == 0 and f["disk_hits"] == c["disk_misses"], f
    assert all(all(v == 0 for v in fl) for k, fl in forced["flags"].items() if not k.endswith("_lookups")), forced["flags"]
    n = forced["notes"]
    assert n["proof_commit_aux"] == LOGUP and n["proof"] == PROOF and n["guarded_proof"] == PROOF
    assert n["guarded_proof_commit_aux"] in (LOGUP, CHECK)
    assert n["census"] == CHECK and n["balance"] == LOOKUP_CHECK and n["fold_census"] == LOOKUP_CHECK
    assert forced["outputs"] == forced["interpreter_outputs"] == cold["outputs"]
