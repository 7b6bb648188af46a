"""The two references of tests/test_lookup_registers.py against each other, without a GPU: the C++ lowering of version-2
lookup programs (orc_logup_aux_registers, tests/oracle_lookup_registers, every row evaluated once in row order) builds
the same aux traces and finals as the Python-integer restatement of the chiplets' loops -- for the MUL-like and
STORE-like AIRs at several heights, with width-20 messages and with the deliberately wrong role-3 update, and for one
AIR with 1 to 4 registers that read each other, one of them also reading a preprocessed column -- and refuses programs
that are not version 2."""
import numpy as np
import pytest

import test_lookup_registers as T

P = T.P
RND = [0x0123456789ABCDEF % P, 0x1111111122222222 % P, 0x5555555566666666 % P, 0x2718281828459045 % P]


def rows_array(rows):
    return np.array([[w for e in row for w in e] for row in rows], dtype=np.uint64)


@pytest.mark.parametrize("log_mul, log_store, width, wrong", [(3, 3, 3, False), (8, 6, 3, False), (6, 9, 3, True), (5, 5, 20, False)])
def test_cpp_lowering_equals_the_python_builder_on_the_chiplets(log_mul, log_store, width, wrong):
    case = T.Case(log_mul, log_store, width=width, wrong_role3=wrong)
    for inst, (prog, trace, per, prep) in enumerate(case.oracle_airs()):
        aux, fin = T.oracle_aux(prog, trace, prep, per, RND)
        rows, want = case.aux_rows(inst, RND)
        assert fin == want
        assert np.array_equal(aux, rows_array(rows))


@pytest.mark.parametrize("k, log_n, prep", [(1, 5, False), (2, 7, True), (3, 6, False), (4, 8, False), (4, 3, True)])
def test_cpp_lowering_equals_the_python_builder_with_k_registers(k, log_n, prep):
    case = T.KCase(k, log_n, prep=prep)
    aux, fin = T.oracle_aux(case.lookup(), case.trace, case.prep, T.PER4, RND)
    rows, want = case.aux_rows(0, RND)
    assert fin == want == (0, 0)                       # the column closes within the AIR
    assert np.array_equal(aux, rows_array(rows))
    assert any(int(x) for x in aux[1:, 2:].reshape(-1)), "the registers must move"


def test_cpp_lowering_refuses_other_versions():
    case = T.KCase(2, 4)
    with pytest.raises(RuntimeError, match="bad header"):
        T.oracle_aux(case.lookup(registers=False), case.trace, None, T.PER4, RND)
    bad = case.lookup().copy()
    bad[5] = 3                                         # three registers announced, two updates given
    with pytest.raises(RuntimeError, match="bad length"):
        T.oracle_aux(bad, case.trace, None, T.PER4, RND)
