"""The device arithmetic, Poseidon2 and NTT kernels, operation by operation, against plain integer references.

tests/cuda/libmdn_devtest.so compiles the product's __host__ __device__ headers and kernels.cu for sm_90a.  Each of its
entry points runs one named operation either on the device (the PTX carry-chain branches, the bulk-copy table loads, the
thread-strided loops) or, from the same source, on the host (the unsigned __int128 branches).  A device case checks:

  1. device == host, bit for bit, including the non-canonical representatives the lazy arithmetic chooses;
  2. host == a Python-integer reference (mod p, or exactly where the function promises an exact value);
  3. the function's contract: canonical results where promised, the documented bounds of the lazy ones.

The inputs are the cross product of an edge set, directed inputs for every carry, borrow and fold branch (each case
asserts in Python that its branch is taken), and random words biased towards high words of all ones.  The NTT cases go
through the product's own launchers at every size 2^1 .. 2^22, so the seven kernels specialised for 2^16 .. 2^22 run
here on their own instead of only inside proofs.

The host-half tests (not marked gpu) run the same references, edge sets and branch assertions on any machine."""
import ctypes as C
import functools
import itertools
import json
import os
import subprocess

import numpy as np
import pytest

import oracle_binding as ob
import pkgload

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_DIR = os.path.join(ROOT, "tests", "cuda")
P = 0xFFFFFFFF00000001
EPS = 0xFFFFFFFF
M32 = (1 << 32) - 1
M64 = (1 << 64) - 1
u64p = C.POINTER(C.c_uint64)


# ---------------------------------------------------------------------------------------------------------------------
# The library
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def dt():
    subprocess.check_call(["make", "-s", "-C", CUDA_DIR])
    L = C.CDLL(os.path.join(CUDA_DIR, "libmdn_devtest.so"))
    L.dt_op_name.restype = C.c_char_p
    L.dt_op_name.argtypes = [C.c_int]
    L.dt_scalar.argtypes = [C.c_int, u64p, u64p, C.c_size_t, C.c_int]
    L.dt_p2.argtypes = [C.c_int, u64p, C.c_size_t, C.c_int]
    L.dt_p2_chain.argtypes = [u64p, C.c_uint32, u64p, C.c_int]
    L.dt_intt.argtypes = [u64p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_int]
    L.dt_fwd.argtypes = [u64p, C.c_uint32, C.c_uint32, u64p, C.c_uint32, u64p, C.c_int]
    return L


def ptr(a):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(u64p)


@functools.lru_cache(maxsize=None)
def ops():
    """operation name -> id, as the library names them"""
    L = dt()
    return {L.dt_op_name(i).decode(): i for i in range(L.dt_op_count())}


def run_scalar(name, rows, device):
    """rows: list of argument tuples (<= 6 ints) -> uint64 array [n, 4]"""
    a = np.zeros((len(rows), 6), dtype=np.uint64)
    for i, r in enumerate(rows):
        a[i, : len(r)] = r
    out = np.zeros((len(rows), 4), dtype=np.uint64)
    rc = dt().dt_scalar(ops()[name], ptr(a), ptr(out), len(rows), int(device))
    assert rc == 0, f"dt_scalar({name}) returned {rc}"
    return out


def run_p2(op, states, device):
    s = np.ascontiguousarray(states, dtype=np.uint64).copy()
    assert dt().dt_p2(op, ptr(s.reshape(-1)), len(s), int(device)) == 0
    return s


P2_FAST_PERMUTE, P2_FAST_EXTERNAL, P2_CANONICAL_PERMUTE = 0, 1, 2


# ---------------------------------------------------------------------------------------------------------------------
# Inputs
# ---------------------------------------------------------------------------------------------------------------------
def edge_values():
    """0..8; 2^k and 2^k +- 1 for k < 64; p +- k, 2^64 - k, 2^32 +- k, 2^63 +- k, 2^64 - 2^32 +- k for k < 4."""
    s = set(range(9))
    for k in range(64):
        s.update(((1 << k) + d) & M64 for d in (-1, 0, 1))
    for k in range(4):
        for base in (P, 1 << 32, 1 << 63, (1 << 64) - (1 << 32)):
            s.update(((base + k) & M64, (base - k) & M64))
        s.add((1 << 64) - 1 - k)
    return sorted(s)


EDGES = edge_values()
CANON_EDGES = [v for v in EDGES if v < P]
HI_WORDS = [0, 1, 2, 3, 7, 8, 0xFF, (1 << 31) - 1, 1 << 31, M32 - 8, M32 - 1, M32]
SMALL = [0, 1, 2, 3, EPS, 1 << 32, (1 << 63) - 1, 1 << 63, P - 2, P - 1, P, P + 1, (1 << 64) - (1 << 32), M64 - 1, M64]
SMALL_CANON = [v for v in SMALL if v < P] + [0x123456789ABCDEF0 % P, 0xDEADBEEF00000001]
ACC_WORDS = [0, 1, EPS, 1 << 63, (1 << 64) - (1 << 32), M64 - 1, M64]
ACC_HI = [0, 1, 1 << 31, M32 - 1, M32]
EXPONENTS = [0, 1, 2, 3, 7, 1 << 32, EPS, P - 2, P - 1, M64, 0x9E3779B97F4A7C15]
KINDS = {"u": EDGES, "c": CANON_EDGES, "h": HI_WORDS, "us": SMALL, "cs": SMALL_CANON, "aw": ACC_WORDS, "ah": ACC_HI,
         "e": EXPONENTS, "k1": [1, 2, 3, 16, 31, 32], "k96l": [1, 2], "k96r": [1, 2, 3]}


def wv(lo, hi):
    return lo + (hi << 64)


def div_exact(v, k):
    """(v + n p) >> k with n = -v mod 2^k: the exact quotient of the representative v + n p"""
    n = (-v) % (1 << k)
    return (v + n * P) >> k, n


# ---------------------------------------------------------------------------------------------------------------------
# Operations: argument kinds, precondition, check (None = pass) and the branches the directed cases target
# ---------------------------------------------------------------------------------------------------------------------
def eq(got, want, what="value"):
    return None if got == want else f"{what} {got:#x} != {want:#x}"


def congruent(got, want):
    return None if (got - want) % P == 0 else f"{got:#x} is not {want % P:#x} mod p"


def canonical(got, want):
    if got >= P:
        return f"{got:#x} is not canonical"
    return eq(got, want % P)


def red128_path(lo, hi):
    """the branches red128 takes on (lo, hi): borrow of lo - hi[63:32], carry of + hi[31:0] * (2^32 - 1)"""
    x3, x2 = hi >> 32, hi & M32
    borrow = lo < x3
    t = (lo - x3) & M64
    if borrow:
        t -= EPS
    carry = t + x2 * EPS > M64
    return borrow, carry


def e2_mul(x, y):
    return ((x[0] * y[0] + 7 * x[1] * y[1]) % P, (x[0] * y[1] + x[1] * y[0]) % P)


def e2_pow(x, e):
    r = (1, 0)
    while e:
        if e & 1:
            r = e2_mul(r, x)
        x = e2_mul(x, x)
        e >>= 1
    return r


def e2_inv(x):
    n = (x[0] * x[0] - 7 * x[1] * x[1]) % P
    ni = pow(n, P - 2, P)
    return (x[0] * ni % P, (-x[1] * ni) % P)


def wide_out(o):
    if o[1] > M32:
        return None, f"high word {o[1]:#x} >= 2^32"
    return wv(o[0], o[1]), None


def chk_wide_exact(want):
    def f(a, o):
        v, err = wide_out(o)
        return err or eq(v, want(a))
    return f


def chk_whalf(a, o):
    v, err = wide_out(o)
    if err:
        return err
    w = wv(a[0], a[1])
    want = (w + (w & 1) * P) >> 1
    if v > (w + P) // 2:
        return "whalf above (v + p) / 2"
    return eq(v, want) or congruent(2 * v, w)


def chk_wdiv(k):
    def f(a, o):
        v, err = wide_out(o)
        if err:
            return err
        w = wv(a[0], a[1])
        if v > (w >> k) + P:
            return f"wdiv2k<{k}> above v / 2^{k} + p"
        return eq(v, div_exact(w, k)[0]) or congruent(v << k, w)
    return f


def chk_div(k):
    def f(a, o):
        return eq(o[0], div_exact(a[0], k)[0]) or congruent(o[0] << k, a[0])
    return f


def chk_acc_exact(a, o):
    if o[2] > M32:
        return "accumulator high word >= 2^32"
    return eq(o[0] + (o[1] << 64) + (o[2] << 128), a[0] + (a[1] << 64) + (a[2] << 128) + a[3] * a[4])


def chk_acc_sum(a, o):
    want = a[0] * a[1] * a[2]
    return eq(o[0] + (o[1] << 64) + (o[2] << 128), want, "sum") or canonical(o[3], want)


def gl_mul_path(a, b):
    q = a * b
    lo, hi = q & M64, q >> 64
    borrow, carry = red128_path(lo, hi)
    x3 = hi >> 32
    t = (lo - x3) & M64
    if borrow:
        t -= EPS
    r = t + (hi & M32) * EPS
    if r > M64:
        r = (r & M64) + EPS
    return borrow, carry, r >= P


def acc_reduce_borrow(a):
    return (a[0] + (a[1] << 64)) % P < (a[2] << 32)


OPS = {
    # name: (argument kinds, precondition, check, {branch: predicate})
    "glf_addc64": ("uu", None, lambda a, o: eq(o[0] + (o[1] << 64), a[0] + a[1]), {"carry": lambda a: a[0] + a[1] > M64}),
    "glf_subb64": ("uu", None, lambda a, o: eq(o[0], (a[0] - a[1]) & M64) or eq(o[1], M32 if a[0] < a[1] else 0, "borrow mask"),
                   {"borrow": lambda a: a[0] < a[1]}),
    "glf_mul_eps": ("h", None, lambda a, o: eq(o[0], a[0] * EPS), {}),
    "glf_mul": ("uu", None, lambda a, o: congruent(o[0], a[0] * a[1]),
                {"borrow": lambda a: red128_path((a[0] * a[1]) & M64, a[0] * a[1] >> 64)[0],
                 "carry": lambda a: red128_path((a[0] * a[1]) & M64, a[0] * a[1] >> 64)[1]}),
    "glf_sqr": ("u", None, lambda a, o: congruent(o[0], a[0] * a[0]),
                {"borrow": lambda a: red128_path((a[0] * a[0]) & M64, a[0] * a[0] >> 64)[0]}),
    "glf_red128": ("uu", None, lambda a, o: congruent(o[0], wv(a[0], a[1])),
                   {"borrow": lambda a: red128_path(a[0], a[1])[0], "carry": lambda a: red128_path(a[0], a[1])[1],
                    "borrow+carry": lambda a: all(red128_path(a[0], a[1]))}),
    "glf_add_const": ("uc", None, lambda a, o: congruent(o[0], a[0] + a[1]), {"carry": lambda a: a[0] + a[1] > M64}),
    "glf_canon": ("u", None, lambda a, o: canonical(o[0], a[0]), {"x>=p": lambda a: a[0] >= P}),
    "glf_canon_cc": ("u", None, lambda a, o: canonical(o[0], a[0]), {"x>=p": lambda a: a[0] >= P, "x<p": lambda a: a[0] < P}),
    "glf_csub": ("cc", None, lambda a, o: canonical(o[0], a[0] - a[1]), {"borrow": lambda a: a[0] < a[1]}),
    "glf_cadd": ("cc", None, lambda a, o: canonical(o[0], a[0] + a[1]),
                 {"borrow": lambda a: a[0] < P - a[1], "wrap": lambda a: a[0] + a[1] >= P}),
    "glf_cmul": ("uu", None, lambda a, o: canonical(o[0], a[0] * a[1]), {}),
    "glf_half": ("u", None, lambda a, o: eq(o[0], (a[0] + (a[0] & 1) * P) >> 1) or congruent(2 * o[0], a[0]),
                 {"odd": lambda a: a[0] & 1 == 1}),
    "glf_div2k2": ("u", None, chk_div(2), {"n!=0": lambda a: a[0] % 4 != 0}),
    "glf_div2k3": ("u", None, chk_div(3), {"n!=0": lambda a: a[0] % 8 != 0}),
    "glf_wsum": ("uu", None, chk_wide_exact(lambda a: a[0] + a[1]), {"carry": lambda a: a[0] + a[1] > M64}),
    "glf_wadd_u64": (("us", "h", "u"), lambda a: wv(a[0], a[1]) + a[2] < 1 << 96, chk_wide_exact(lambda a: wv(a[0], a[1]) + a[2]),
                     {"carry": lambda a: a[0] + a[2] > M64}),
    "glf_wadd_w": (("us", "h", "us", "h"), lambda a: wv(a[0], a[1]) + wv(a[2], a[3]) < 1 << 96,
                   chk_wide_exact(lambda a: wv(a[0], a[1]) + wv(a[2], a[3])), {"carry": lambda a: a[0] + a[2] > M64}),
    "glf_wsub": (("us", "h", "us", "h"), lambda a: wv(a[0], a[1]) >= wv(a[2], a[3]),
                 chk_wide_exact(lambda a: wv(a[0], a[1]) - wv(a[2], a[3])), {"borrow": lambda a: a[0] < a[2]}),
    "glf_wshl": (("u", "k1"), None, chk_wide_exact(lambda a: a[0] << a[1]), {}),
    "glf_wtriple": ("u", None, chk_wide_exact(lambda a: 3 * a[0]), {"carry": lambda a: 3 * a[0] > M64}),
    "glf_wred": (("u", "h"), None, lambda a, o: congruent(o[0], wv(a[0], a[1])), {"carry": lambda a: a[0] + a[1] * EPS > M64}),
    "glf_wshl96": (("us", "h", "k96l"), lambda a: wv(a[0], a[1]) << a[2] < 1 << 96, chk_wide_exact(lambda a: wv(a[0], a[1]) << a[2]), {}),
    "glf_wshr96": (("us", "h", "k96r"), None, chk_wide_exact(lambda a: wv(a[0], a[1]) >> a[2]), {}),
    "glf_whalf": (("u", "h"), lambda a: wv(a[0], a[1]) + P < 1 << 96, chk_whalf, {"odd+carry": lambda a: a[0] & 1 and a[0] + P > M64}),
    "glf_wdiv2k2": (("u", "h"), lambda a: a[1] + div_exact(a[0], 2)[1] <= M32, chk_wdiv(2),
                    {"borrow": lambda a: a[0] < div_exact(a[0], 2)[1] * EPS}),
    "glf_wdiv2k3": (("u", "h"), lambda a: a[1] + div_exact(a[0], 3)[1] <= M32, chk_wdiv(3),
                    {"borrow": lambda a: a[0] < div_exact(a[0], 3)[1] * EPS}),
    "gl_fast_addc64": ("uu", None, lambda a, o: eq(o[0] + (o[1] << 64), a[0] + a[1]), {"carry": lambda a: a[0] + a[1] > M64}),
    "gl_fast_subb64": ("uu", None, lambda a, o: eq(o[0], (a[0] - a[1]) & M64) or eq(o[1], M32 if a[0] < a[1] else 0, "borrow mask"),
                       {"borrow": lambda a: a[0] < a[1]}),
    "gl_add": ("cc", None, lambda a, o: canonical(o[0], a[0] + a[1]), {"wrap": lambda a: a[0] + a[1] >= P}),
    "gl_sub": ("cc", None, lambda a, o: canonical(o[0], a[0] - a[1]), {"borrow": lambda a: a[0] < a[1]}),
    "gl_neg": ("c", None, lambda a, o: canonical(o[0], -a[0]), {}),
    "gl_mul": ("uu", None, lambda a, o: canonical(o[0], a[0] * a[1]),
               {"borrow": lambda a: gl_mul_path(*a)[0], "carry": lambda a: gl_mul_path(*a)[1],
                "r>=p": lambda a: gl_mul_path(*a)[2]}),
    "gl_half": ("c", None, lambda a, o: f"{o[0]:#x} is not canonical" if o[0] >= P else congruent(2 * o[0], a[0]), {}),
    "gl_pow": ("ue", None, lambda a, o: canonical(o[0], pow(a[0], a[1], P)), {}),
    "gl_inv": ("u", None, lambda a, o: canonical(o[0], pow(a[0], P - 2, P)), {}),
    "gl_e2_mul": (("cs",) * 4, None, lambda a, o: eq((o[0], o[1]), e2_mul(a[:2], a[2:4]), "e2"), {}),
    "gl_e2_sqr": ("cc", None, lambda a, o: eq((o[0], o[1]), e2_mul(a[:2], a[:2]), "e2"), {}),
    "gl_e2_inv": ("cc", None, lambda a, o: eq((o[0], o[1]), e2_inv(a[:2]), "e2"), {}),
    "gl_e2_pow": (("cs", "cs", "e"), None, lambda a, o: eq((o[0], o[1]), e2_pow(a[:2], a[2]), "e2"), {}),
    "acc_mul": (("aw", "aw", "ah", "us", "us"), lambda a: a[0] + (a[1] << 64) + (a[2] << 128) + a[3] * a[4] < 1 << 160,
                chk_acc_exact, {"carry lo": lambda a: a[0] + (a[3] * a[4] & M64) > M64,
                                "carry mid": lambda a: a[1] + (a[3] * a[4] >> 64) + ((a[0] + (a[3] * a[4] & M64)) >> 64) > M64}),
    "acc_reduce": (("u", "us", "h"), None, lambda a, o: canonical(o[0], a[0] + (a[1] << 64) + (a[2] << 128)),
                   {"borrow": acc_reduce_borrow}),
    "acc_sum": ((), None, chk_acc_sum, {}),
}

# Directed inputs: (operation, arguments, the branch they must take)
DIRECTED = [
    ("glf_red128", (0, 1 << 32), "borrow"),                       # the product 2^96: lo = 0, hi >> 32 = 1
    ("glf_red128", (5, 7 << 32), "borrow"),
    ("glf_red128", (M64, M32), "carry"),
    ("glf_red128", (0, (1 << 32) | M32), "borrow+carry"),
    ("glf_red128", (EPS - 1, M64), "borrow+carry"),
    ("glf_mul", (1 << 48, 1 << 48), "borrow"),
    ("glf_mul", (M64, M64), "borrow"),
    ("glf_mul", (M64, M64), "carry"),
    ("glf_sqr", (1 << 48,), "borrow"),
    ("gl_mul", (1 << 48, 1 << 48), "borrow"),
    ("gl_mul", (M64, M64), "carry"),
    ("gl_mul", (P - 1, P - 1), "r>=p"),
    ("glf_add_const", (M64, P - 1), "carry"),
    ("glf_add_const", ((1 << 64) - (1 << 32), EPS + 1), "carry"),
    ("glf_canon", (P,), "x>=p"),
    ("glf_canon", (M64,), "x>=p"),
    ("glf_canon_cc", (P + 5,), "x>=p"),
    ("glf_canon_cc", (P - 1,), "x<p"),
    ("glf_csub", (0, P - 1), "borrow"),
    ("glf_cadd", (1, 2), "borrow"),
    ("glf_cadd", (P - 1, P - 1), "wrap"),
    ("glf_half", (M64,), "odd"),
    ("glf_div2k2", (M64,), "n!=0"),
    ("glf_div2k2", (P + 2,), "n!=0"),
    ("glf_div2k3", (M64 - 2,), "n!=0"),
    ("glf_div2k3", (1,), "n!=0"),
    ("glf_wsum", (M64, M64), "carry"),
    ("glf_wadd_u64", (M64, 5, 1), "carry"),
    ("glf_wadd_w", (M64, 0, M64, M32 - 1), "carry"),
    ("glf_wsub", (0, 1, 1, 0), "borrow"),
    ("glf_wtriple", (M64,), "carry"),
    ("glf_wred", (M64, M32), "carry"),
    ("glf_whalf", (M64, 0), "odd+carry"),
    ("glf_whalf", (M64 - 2, 7), "odd+carry"),
    ("glf_wdiv2k2", (1, 1), "borrow"),                              # n = 3: n (2^32 - 1) > lo
    ("glf_wdiv2k2", (EPS - 1, 5), "borrow"),
    ("glf_wdiv2k3", (1, 0), "borrow"),
    ("glf_wdiv2k3", (3 * EPS - 1, M32 - 8), "borrow"),
    ("gl_fast_addc64", (M64, 1), "carry"),
    ("gl_fast_subb64", (0, 1), "borrow"),
    ("gl_add", (P - 1, 1), "wrap"),
    ("gl_sub", (0, P - 1), "borrow"),
    ("glf_addc64", (1 << 63, 1 << 63), "carry"),
    ("glf_subb64", (1, 2), "borrow"),
    ("acc_mul", (M64, 0, 0, 2, 1), "carry lo"),
    ("acc_mul", (M64, M64, 0, M64, M64), "carry mid"),
    ("acc_reduce", (0, 0, M32), "borrow"),
    ("acc_reduce", (5, 0, 1), "borrow"),
]


def rows_for(name, rng, n_random):
    kinds, pre, _, _ = OPS[name]
    if name == "acc_sum":   # sums of up to 2^16 products of the largest words
        return [(x, y, c) for x, y in ((P - 1, P - 1), (M64, M64), (P - 1, M64), (EPS, 1 << 63))
                for c in (0, 1, 2, 255, 256, 1 << 15, 1 << 16)]
    rows = list(itertools.product(*(KINDS[k] for k in kinds)))
    rows += [a for op, a, _ in DIRECTED if op == name]
    if n_random:   # random words, a quarter of them with the high 32 bits all ones
        r = rng.integers(0, 1 << 64, (n_random, len(kinds)), dtype=np.uint64, endpoint=False)
        r[: n_random // 4] |= np.uint64(0xFFFFFFFF00000000)
        for j, k in enumerate(kinds):
            if k in ("c", "cs"):
                r[:, j] = np.where(r[:, j] >= np.uint64(P), r[:, j] - np.uint64(P), r[:, j])
            elif k not in ("u", "us", "aw", "e"):
                choices = np.array(KINDS[k], dtype=np.uint64)
                r[:, j] = choices[rng.integers(0, len(choices), n_random)]
        rows += [tuple(int(x) for x in row) for row in r]
    if pre is not None:
        rows = [a for a in rows if pre(a)]
    return rows


# ops with a random stream (the rest see the edge cross product and the directed cases)
RANDOM_OPS = {"glf_mul": 1 << 18, "glf_red128": 1 << 17, "glf_add_const": 1 << 16, "glf_canon_cc": 1 << 16,
              "glf_cmul": 1 << 16, "glf_div2k2": 1 << 16, "glf_div2k3": 1 << 16, "glf_wred": 1 << 16,
              "glf_whalf": 1 << 16, "glf_wdiv2k2": 1 << 16, "glf_wdiv2k3": 1 << 16, "gl_mul": 1 << 18,
              "acc_mul": 1 << 16, "acc_reduce": 1 << 16}


def check_rows(name, rows, out):
    check = OPS[name][2]
    bad = []
    for a, o in zip(rows, out):
        err = check(a, [int(x) for x in o])
        if err:
            bad.append(f"{name}{tuple(hex(x) for x in a)}: {err}")
            if len(bad) >= 5:
                break
    assert not bad, "\n".join(bad)


def test_directed_cases_take_their_branches():
    """Every directed input really takes the branch it is there for, and every listed branch has a directed input."""
    covered = set()
    for name, a, branch in DIRECTED:
        assert OPS[name][3][branch](a), f"{name}{tuple(hex(x) for x in a)} does not take the {branch} branch"
        pre = OPS[name][1]
        assert pre is None or pre(a), f"{name}{a} violates the operation's precondition"
        covered.add((name, branch))
    for name, (_, _, _, branches) in OPS.items():
        for branch in branches:
            assert (name, branch) in covered, f"no directed input for {name} {branch}"


def test_every_library_operation_has_a_reference():
    assert set(ops()) == set(OPS)


@pytest.mark.parametrize("name", sorted(OPS))
def test_scalar_host_half(name):
    """The host branches of the library against the integer references, on the edge cross product and directed inputs."""
    rows = rows_for(name, np.random.default_rng(1), 1 << 12)
    check_rows(name, rows, run_scalar(name, rows, device=False))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(OPS))
def test_scalar_device(name):
    rows = rows_for(name, np.random.default_rng(2), RANDOM_OPS.get(name, 1 << 12))
    dev = run_scalar(name, rows, device=True)
    host = run_scalar(name, rows, device=False)
    diff = np.nonzero((dev != host).any(axis=1))[0]
    assert len(diff) == 0, f"{name}: device != host at {len(diff)} rows, first {tuple(hex(x) for x in rows[diff[0]])}: " \
                           f"device {[hex(int(x)) for x in dev[diff[0]]]}, host {[hex(int(x)) for x in host[diff[0]]]}"
    check_rows(name, rows, dev)


# ---------------------------------------------------------------------------------------------------------------------
# Poseidon2
# ---------------------------------------------------------------------------------------------------------------------
def p2_states(seed, n_random=4096):
    rng = np.random.default_rng(seed)
    edges = np.array(EDGES, dtype=np.uint64)
    s = [np.arange(12, dtype=np.uint64), np.zeros(12, dtype=np.uint64), np.full(12, M64, dtype=np.uint64),
         np.full(12, P - 1, dtype=np.uint64), np.full(12, P, dtype=np.uint64)]
    s = np.stack(s)
    r1 = edges[rng.integers(0, len(edges), (n_random, 12))]                          # edge lanes, [p, 2^64) included
    r2 = rng.integers(0, 1 << 64, (n_random, 12), dtype=np.uint64, endpoint=False)
    r2[: n_random // 2] |= np.uint64(0xFFFFFFFF00000000)
    return np.ascontiguousarray(np.concatenate([s, r1, r2]))


def canon(a):
    a = np.asarray(a, dtype=np.uint64)
    return np.where(a >= np.uint64(P), a - np.uint64(P), a)


def ext_layer_ref(s):
    """the external layer as integer matrix algebra mod p: M4 on each chunk, then the block-circulant [2M, M, M]"""
    m4 = [[2, 3, 1, 1], [1, 2, 3, 1], [1, 1, 2, 3], [3, 1, 1, 2]]
    y = []
    for c in range(0, 12, 4):
        y += [sum(m4[i][j] * s[c + j] for j in range(4)) for i in range(4)]
    return [(y[i] + sum(y[(i % 4) + 4 * k] for k in range(3))) % P for i in range(12)]


def kat():
    with open(os.path.join(ROOT, "tests", "golden", "poseidon2_kat.json")) as f:
        k = json.load(f)
    return np.array(k["input"], dtype=np.uint64), np.array([int(h, 16) for h in k["output_hex"]], dtype=np.uint64)


def check_p2(states, raw_perm, raw_ext, oracle):
    """raw p2f::permute / external_layer outputs against p2::permute of the canonical input, the oracle and the KAT"""
    canon_in = canon(states)
    want = run_p2(P2_CANONICAL_PERMUTE, canon_in, device=False)
    orc = canon_in.copy()
    oracle.orc_poseidon2_permute(ob.ptr(orc.reshape(-1)), len(orc))
    assert np.array_equal(want, orc), "p2::permute != oracle"
    assert np.array_equal(canon(raw_perm), want), "p2f::permute != p2::permute of the canonical input"
    for i in range(0, len(states), max(1, len(states) // 500)):
        assert [int(x) % P for x in raw_ext[i]] == ext_layer_ref([int(x) for x in states[i]]), f"external layer, state {i}"
    kin, kout = kat()
    i = [k for k in range(len(states)) if np.array_equal(states[k], kin)][0]
    assert np.array_equal(canon(raw_perm[i]), kout), "KAT"


def oracle_chain(data, oracle):
    s = np.zeros((1, 12), dtype=np.uint64)
    for j in range(len(data) // 8):
        s[0, :8] = data[8 * j: 8 * j + 8]
        oracle.orc_poseidon2_permute(ob.ptr(s.reshape(-1)), 1)
    return s[0]


def chain(data, device):
    out = np.zeros(12, dtype=np.uint64)
    assert dt().dt_p2_chain(ptr(data), len(data) // 8, ptr(out), int(device)) == 0
    return out


def chain_data(seed):
    rng = np.random.default_rng(seed)
    d = canon(rng.integers(0, 1 << 64, 64 * 8, dtype=np.uint64, endpoint=False))
    d[:8] = P - 1                                   # the bound drivers first
    d[8:16] = 0
    return np.ascontiguousarray(d)


def test_poseidon2_host_half(oracle):
    st = p2_states(3, 512)
    check_p2(st, run_p2(P2_FAST_PERMUTE, st, False), run_p2(P2_FAST_EXTERNAL, st, False), oracle)
    d = chain_data(4)
    assert np.array_equal(canon(chain(d, False)), oracle_chain(d, oracle))


@pytest.mark.gpu
def test_poseidon2_device(oracle):
    st = p2_states(5)
    perm, ext = run_p2(P2_FAST_PERMUTE, st, True), run_p2(P2_FAST_EXTERNAL, st, True)
    assert np.array_equal(perm, run_p2(P2_FAST_PERMUTE, st, False)), "p2f::permute: device != host representatives"
    assert np.array_equal(ext, run_p2(P2_FAST_EXTERNAL, st, False)), "p2f::external_layer: device != host representatives"
    c = canon(st)
    assert np.array_equal(run_p2(P2_CANONICAL_PERMUTE, c, True), run_p2(P2_CANONICAL_PERMUTE, c, False)), "p2::permute"
    check_p2(st, perm, ext, oracle)


@pytest.mark.gpu
def test_poseidon2_leaf_sponge_chain_device(oracle):
    """64 permutations with lanes 8..11 handed on as lazy representatives, as k_leaf_hash does"""
    d = chain_data(6)
    dev = chain(d, True)
    assert np.array_equal(dev, chain(d, False)), "device != host representatives"
    assert np.array_equal(canon(dev), oracle_chain(d, oracle))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 127, 128, 129, 100003])
def test_poseidon2_product_batch(oracle, n):
    """mdn_poseidon2_permute (launch_poseidon2_batch, 128-thread blocks) with partial last blocks"""
    pkg = pkgload.load_pkg()
    B, W = pkg.binding, pkg.workload
    st = canon(p2_states(7 + n, (n + 1) // 2))[:n].copy()
    if n == 1:
        st[0] = np.arange(12)
    want = st.copy()
    oracle.orc_poseidon2_permute(ob.ptr(want.reshape(-1)), n)
    s = B.Session(W.miden_pcs_params(), 0)
    try:
        assert B.lib().mdn_poseidon2_permute(s.handle, B.ptr(st.reshape(-1)), n) == 0
    finally:
        s.close()
    assert np.array_equal(st, want)


# ---------------------------------------------------------------------------------------------------------------------
# NTT
# ---------------------------------------------------------------------------------------------------------------------
def two_adic_generator(bits):
    return pow(1753635133440165772, 1 << (32 - bits), P)


def lde_shift(log_lde):
    return pow(7, 1 << (32 - log_lde), P)


def split(n):
    return (0, n) if n <= 11 else (n // 2, n - n // 2)


def npmul(a, b):
    """Goldilocks product of uint64 arrays, canonical out, without Python integers: the 128-bit product from 32-bit
    limbs, then 2^64 = 2^32 - 1 and 2^96 = -1 (mod p)."""
    a, b = np.broadcast_arrays(np.asarray(a, dtype=np.uint64), np.asarray(b, dtype=np.uint64))
    m, s32 = np.uint64(M32), np.uint64(32)
    a0, a1, b0, b1 = a & m, a >> s32, b & m, b >> s32
    p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1
    mid = (p00 >> s32) + (p01 & m) + (p10 & m)
    lo = (p00 & m) | (mid << s32)
    hi = p11 + (p01 >> s32) + (p10 >> s32) + (mid >> s32)
    x3, x2 = hi >> s32, hi & m
    t = lo - x3
    t = np.where(lo < x3, t - np.uint64(EPS), t)
    r = t + x2 * np.uint64(EPS)
    r = np.where(r < t, r + np.uint64(EPS), r)
    return canon(r)


def npadd(a, b):
    s = a + b
    s = np.where(s < a, s + np.uint64(EPS), s)      # carried: 2^64 = 2^32 - 1
    return canon(s)


def npsub(a, b):
    return np.where(a >= b, a - b, a - b + np.uint64(P))


def np_powers(g, count):
    """g^0 .. g^(count-1) as uint64"""
    lo_n = 1 << 11
    lo = np.ones(min(count, lo_n), dtype=np.uint64)
    for i in range(1, len(lo)):
        lo[i] = int(lo[i - 1]) * g % P
    if count <= lo_n:
        return lo
    gh = pow(g, lo_n, P)
    hi = np.array([pow(gh, i, P) for i in range((count + lo_n - 1) // lo_n)], dtype=np.uint64)
    return npmul(hi[:, None], lo[None, :]).reshape(-1)[:count]


def brev_idx(n):
    idx = np.arange(1 << n, dtype=np.uint64)
    rev = np.zeros_like(idx)
    for b in range(n):
        rev |= ((idx >> np.uint64(b)) & np.uint64(1)) << np.uint64(n - 1 - b)
    return rev.astype(np.int64)


def np_dft(a, w):
    """out[k] = sum_j a[j] w^(jk), natural in and out: radix-2 decimation in time on uint64 arrays"""
    n = len(a).bit_length() - 1
    x = np.asarray(a, dtype=np.uint64)[brev_idx(n)].copy()
    for s in range(n):
        h = 1 << s
        tw = np_powers(pow(w, (1 << n) >> (s + 1), P), h)
        x = x.reshape(-1, 2, h)
        u, v = x[:, 0, :], npmul(x[:, 1, :], tw[None, :])
        x = np.stack([npadd(u, v), npsub(u, v)], axis=1).reshape(-1)
    return x


def orc_dft(oracle, a):
    out = np.zeros_like(a)
    a = np.ascontiguousarray(a, dtype=np.uint64)
    oracle.orc_dft(ob.ptr(a), len(a).bit_length() - 1, 1, 0, ob.ptr(out))
    return out


def dft(oracle, a, w):
    """the transform of the definition: numpy up to 2^12, the oracle above (both run from w = the generator)"""
    n = len(a).bit_length() - 1
    if n <= 12:
        return np_dft(a, w)
    assert w == two_adic_generator(n)
    return orc_dft(oracle, a)


def idft_unscaled(oracle, col):
    """N c[j] = sum_i col[i] w^(-ij)"""
    n = len(col).bit_length() - 1
    w = two_adic_generator(n)
    if n <= 12:
        return np_dft(col, pow(w, P - 2, P))
    f = orc_dft(oracle, col)
    return f[(-np.arange(1 << n)) % (1 << n)]


def coset_eval(oracle, slots, g):
    """the forward launcher's definition: slot p holds C[bitrev(p)]; out[r] = sum_j C[j] g^j / N w^(jr)"""
    n = len(slots).bit_length() - 1
    c = slots[brev_idx(n)]
    a = npmul(npmul(c, np_powers(g, 1 << n)), pow(1 << n, P - 2, P))
    return dft(oracle, a, two_adic_generator(n))


def trace_bases(n, lb):
    s, w = lde_shift(n + lb), two_adic_generator(n + lb)
    return [s * pow(w, t, P) % P for t in range(1 << lb)]


def quotient_base(n):
    # a coset of the quotient domain: w_J^-t * w_L^t' with J = n + 3, L = n + 5
    return pow(two_adic_generator(n + 3), P - 2, P) * pow(two_adic_generator(n + 5), 3, P) % P


def base_sets(n):
    """(bases) per forward call: for n <= 11 an odd and an even count (the tab_c blocks of the odd count are not all
    16-byte aligned, so table_load takes its plain-copy path for them); above, fewer bases (2^22-point columns)."""
    q, rnd = quotient_base(n), 0x1D2C3B4A59687766 % P
    if n <= 12:
        return [trace_bases(n, 3) + [1, rnd, q], trace_bases(n, 1) + trace_bases(n, 4)]
    return [[trace_bases(n, 3)[1], 1, q]]


SAMPLE_ROWS = 48


def sample_rows(n, rng):
    N = 1 << n
    if N <= 2 * SAMPLE_ROWS:
        return list(range(N))
    return sorted({0, 1, N - 1, N // 2} | set(int(x) for x in rng.integers(0, N, SAMPLE_ROWS)))


def eval_columns(n, rng):
    """evaluation columns over H: random, zero, all p - 1, impulses at 0 and N - 1, constant, x and x^(N-1)"""
    N = 1 << n
    w = two_adic_generator(n)
    wp = np_powers(w, N)
    cols = {"random": canon(rng.integers(0, 1 << 64, N, dtype=np.uint64, endpoint=False)),
            "zero": np.zeros(N, dtype=np.uint64), "p-1": np.full(N, P - 1, dtype=np.uint64),
            "impulse0": np.zeros(N, dtype=np.uint64), "impulseN-1": np.zeros(N, dtype=np.uint64),
            "const": np.full(N, 0x0123456789ABCDEF, dtype=np.uint64), "x": wp, "x^(N-1)": wp[(-np.arange(N)) % N]}
    cols["impulse0"][0] = 0xFEDCBA9876543210 % P
    cols["impulseN-1"][N - 1] = P - 2
    return cols


def run_intt(cols, n, device):
    N = 1 << n
    stride = N + 8
    k = len(cols)
    buf = np.full((k, stride), 0x5A5A5A5A5A5A5A5A, dtype=np.uint64)
    for i, c in enumerate(cols):
        buf[i, :N] = c
    assert dt().dt_intt(ptr(buf.reshape(-1)), stride, k, n, int(device)) == 0
    assert (buf[:, N:] == np.uint64(0x5A5A5A5A5A5A5A5A)).all(), "the inverse NTT wrote outside its columns"
    return buf[:, :N].copy()


def run_fwd(src, n, bases, device):
    src = np.ascontiguousarray(src, dtype=np.uint64)
    b = np.array(bases, dtype=np.uint64)
    out = np.zeros((len(src), len(bases), 1 << n), dtype=np.uint64)
    assert dt().dt_fwd(ptr(src.reshape(-1)), len(src), n, ptr(b), len(b), ptr(out.reshape(-1)), int(device)) == 0
    return out


def check_ntt(n, oracle, device, seed):
    """inverse and forward transforms of size 2^n through the library (device or host half)"""
    N = 1 << n
    rng = np.random.default_rng(seed)
    w = two_adic_generator(n)
    ninv = pow(N, P - 2, P)
    rows = sample_rows(n, rng)
    ev = eval_columns(n, rng)
    names = list(ev)
    coef = run_intt([ev[k] for k in names], n, device)
    rev = brev_idx(n)
    assert (coef < np.uint64(P)).all(), "non-canonical coefficient"
    # inverse: value for value (random column) and closed forms (slot p holds N c[bitrev p])
    for i, k in enumerate(names):
        if k in ("random", "impulse0"):
            assert np.array_equal(coef[i], idft_unscaled(oracle, ev[k])[rev]), f"2^{n} inverse, {k} column"
    for p in rows:
        j = int(rev[p])
        want = {"zero": 0, "p-1": (-N) % P if j == 0 else 0, "impulse0": int(ev["impulse0"][0]),
                "impulseN-1": (P - 2) * pow(w, j, P) % P, "const": N * 0x0123456789ABCDEF % P if j == 0 else 0,
                "x": N % P if j == 1 % N else 0, "x^(N-1)": N % P if j == N - 1 else 0}
        for k, v in want.items():
            if N == 1 and k in ("x", "x^(N-1)", "impulseN-1"):
                continue
            assert int(coef[names.index(k)][p]) == v, f"2^{n} inverse, {k} column, slot {p}"
    # forward: the pipeline columns plus coefficient columns set directly
    src = {"random": coef[names.index("random")], "const": coef[names.index("const")], "x": coef[names.index("x")],
           "x^(N-1)": coef[names.index("x^(N-1)")], "zero": np.zeros(N, dtype=np.uint64),
           "all p-1": np.full(N, P - 1, dtype=np.uint64), "slot0": np.zeros(N, dtype=np.uint64),
           "slotN-1": np.zeros(N, dtype=np.uint64)}
    src["slot0"][0] = 12345
    src["slotN-1"][N - 1] = P - 3
    snames = list(src)
    for bases in base_sets(n):
        out = run_fwd([src[k] for k in snames], n, bases, device)
        assert (out < np.uint64(P)).all(), f"2^{n} forward: non-canonical evaluation"
        for bi, g in enumerate(bases):
            full = ["random"] if n > 12 else snames
            for k in full:
                assert np.array_equal(out[snames.index(k), bi], coset_eval(oracle, src[k], g)), f"2^{n} forward, {k}, base {bi}"
            for r in rows:
                x = g * pow(w, r, P) % P
                geo = N % P if x == 1 else (pow(x, N, P) - 1) * pow(x - 1, P - 2, P) % P
                want = {"const": 0x0123456789ABCDEF, "x": x, "x^(N-1)": pow(x, N - 1, P), "zero": 0,
                        "all p-1": (-geo * ninv) % P, "slot0": 12345 * ninv % P,
                        "slotN-1": (P - 3) * pow(x, N - 1, P) * ninv % P}
                for k, v in want.items():
                    assert int(out[snames.index(k), bi, r]) == v, f"2^{n} forward, {k}, base {bi} ({g:#x}), row {r}"
    return coef


def ntt_id(n):
    n1, n2 = split(n)
    return f"n={n}-single" if n1 == 0 else f"n={n}-split{n1}x{n2}" + ("-fixed" if n >= 16 else "-runtime")


def test_references_self_check(oracle):
    """npmul against Python integers; the numpy transform against the oracle's O(N^2) sum and its fast DFT"""
    rng = np.random.default_rng(9)
    a = np.concatenate([np.array(EDGES, dtype=np.uint64), rng.integers(0, 1 << 64, 4000, dtype=np.uint64, endpoint=False)])
    b = np.roll(a, 7)
    assert [int(x) for x in npmul(a, b)] == [int(x) * int(y) % P for x, y in zip(a, b)]
    assert [int(x) for x in npadd(canon(a), canon(b))] == [(int(x) + int(y)) % P for x, y in zip(canon(a), canon(b))]
    assert [int(x) for x in np_powers(5, 5000)] == [pow(5, i, P) for i in range(5000)]
    for n in range(1, 11):
        col = canon(rng.integers(0, 1 << 64, 1 << n, dtype=np.uint64, endpoint=False))
        naive = np.zeros_like(col)
        oracle.orc_naive_dft(ob.ptr(col), n, ob.ptr(naive))
        assert np.array_equal(np_dft(col, two_adic_generator(n)), naive), f"numpy DFT 2^{n}"
        assert np.array_equal(orc_dft(oracle, col), naive), f"oracle DFT 2^{n}"


@pytest.mark.parametrize("n", range(1, 15), ids=ntt_id)
def test_ntt_host_half(oracle, n):
    """the block functions of the NTT kernels on the host (run-time schedules) against the same references"""
    check_ntt(n, oracle, device=False, seed=100 + n)


@pytest.mark.gpu
@pytest.mark.parametrize("n", range(1, 23), ids=ntt_id)
def test_ntt_device(oracle, n):
    """mk::launch_intt and mk::launch_fwd_ntt at every size: single pass up to 2^11, run-time two-pass 2^12 .. 2^15 and
    the seven fixed-size splits 2^16 .. 2^22"""
    check_ntt(n, oracle, device=True, seed=200 + n)


# ---------------------------------------------------------------------------------------------------------------------
# The public LDE path and one proof with the (8, 9) split
# ---------------------------------------------------------------------------------------------------------------------
def rand_felts(shape, seed):
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(canon(rng.integers(0, 1 << 64, shape, dtype=np.uint64, endpoint=False)))


# (log_n, width, log_blowup): widths end the column-group loop of lde_matrix on a partial group where the group size
# allows (groups of 5 columns at 2^16, 2 at 2^17, 1 above)
LDE_CASES = [(16, 7, 3), (17, 3, 3), (18, 2, 3), (19, 2, 3), (20, 2, 3), (21, 2, 3), (22, 2, 3),
             (16, 7, 1), (17, 3, 1), (16, 7, 4), (17, 3, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("log_n,width,lb", LDE_CASES, ids=[f"2^{a}-w{b}-blowup{1 << c}" for a, b, c in LDE_CASES])
def test_coset_lde_public_path(oracle, log_n, width, lb):
    pkg = pkgload.load_pkg()
    B, W = pkg.binding, pkg.workload
    params = W.miden_pcs_params() if lb == 3 else B.PcsParams(lb, 2, 1, 1, 2, 6, 3)
    m = rand_felts((1 << log_n, width), 300 + log_n)
    m[:, 0] = m[::-1, 0]
    m[0, -1] = P - 1
    shift = lde_shift(log_n + lb)
    got = np.zeros(((1 << log_n) << lb, width), dtype=np.uint64)
    s = B.Session(params, 0)
    try:
        rc = B.lib().mdn_coset_lde_batch(s.handle, C.byref(B.Matrix(B.ptr(m), log_n, width)), lb, shift, B.ptr(got.reshape(-1)))
        assert rc == 0, B.lib().mdn_last_error(s.handle)
    finally:
        s.close()
    exp = np.zeros_like(got)
    oracle.orc_coset_lde_batch(C.byref(ob.Matrix(ob.ptr(m), log_n, width)), lb, shift, ob.ptr(exp.reshape(-1)))
    bad = np.nonzero((got != exp).any(axis=1))[0]
    assert len(bad) == 0, f"2^{log_n} LDE differs in {len(bad)} rows, first bit-reversed row {bad[0]}"


@pytest.mark.gpu
def test_proof_with_the_8_9_split():
    """heights 2^17 and 2^16 with the Miden parameters: the 2^17 trace LDE and the quotient LDE on its non-trace bases
    inside the real proof path, compared stage by stage with the oracle prover"""
    from test_gpu_parity import _compare_proofs
    pkg = pkgload.load_pkg()
    B, W = pkg.binding, pkg.workload
    params = W.miden_pcs_params()
    s = B.Session(params, 0)
    B.lib().mdn_set_debug(s.handle, 1)
    try:
        _compare_proofs(s, params, W.Workload([17, 16], widths=(12, 9), aux_widths=(1, 2)))
    finally:
        s.close()
