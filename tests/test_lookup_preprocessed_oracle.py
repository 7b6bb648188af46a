"""The two references of tests/test_lookup_preprocessed.py against each other, without a GPU: the C++ lowering of lookup
programs that read preprocessed columns (orc_logup_aux_prep, tests/oracle_lookup_prep) builds the same aux traces and
finals as the Python-integer builder that reads the preprocessed table directly -- for the LUT (op 15 at offsets 0 and
1, the wrap row N - 1 active) and for the requester, at mixed heights and with width-18 messages -- and refuses op 15
where the AIR has no such preprocessed column."""
import numpy as np
import pytest

import test_lookup_preprocessed as T

P = T.P
RND = [0x0123456789ABCDEF % P, 0x1111111122222222 % P, 0x5555555566666666 % P, 0x2718281828459045 % P]


@pytest.mark.parametrize("log_lut, log_req, width", [(6, 8, 3), (8, 6, 3), (6, 7, 18), (5, None, 3), (4, None, 18)])
def test_cpp_lowering_equals_the_python_builder(log_lut, log_req, width):
    case = T.Case(log_lut, log_req, width=width)
    aux, fin = T.oracle_aux(case.lut_lookup(), case.lut, log_lut, 2, case.prep, case.per, RND)
    rows, want = case.aux_rows(T.LUT, RND)
    assert fin == want
    assert np.array_equal(aux, np.array([[*acc, *f1] for acc, f1 in rows], dtype=np.uint64))
    n = 1 << log_lut
    assert tuple(aux[n - 1, 2:4]) != (0, 0), "the wrap row's bus-1 fraction must be non-zero"
    if log_req is not None:
        aux, fin = T.oracle_aux(case.req_lookup(), case.req, log_req, 7, None, None, RND)
        rows, want = case.aux_rows(T.REQ, RND)
        assert fin == want
        assert np.array_equal(aux, np.array([[*acc, *f1] for acc, f1 in rows], dtype=np.uint64))


def test_cpp_lowering_reads_the_next_row_with_the_wrap():
    """The wrap row reads row 0: rotate the table's column c by one row, and the wrap row's fraction follows the new
    row 0 as the Python builder has it (and differs from the unrotated table's)."""
    case = T.Case(5, None)
    before = T.oracle_aux(case.lut_lookup(), case.lut, 5, 2, case.prep, case.per, RND)[0][31, 2:4].copy()
    case.prep[:, 2] = np.roll(case.prep[:, 2], -1)
    aux, fin = T.oracle_aux(case.lut_lookup(), case.lut, 5, 2, case.prep, case.per, RND)
    rows, want = case.aux_rows(T.LUT, RND)
    assert fin == want and tuple(int(x) for x in aux[31, 2:4]) == rows[31][1]
    assert tuple(aux[31, 2:4]) != tuple(before)


def test_cpp_lowering_refuses_op15_out_of_range():
    case = T.Case(5, None)
    with pytest.raises(RuntimeError, match="preprocessed column out of range"):
        T.oracle_aux(case.lut_lookup(), case.lut, 5, 2, case.prep[:, :2], case.per, RND)
    with pytest.raises(RuntimeError, match="preprocessed column out of range"):
        T.oracle_aux(case.lut_lookup(), case.lut, 5, 2, None, case.per, RND)
