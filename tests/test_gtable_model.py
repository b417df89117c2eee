"""CPU: the plain model of the fixed-base comb table (tests/gtable_model.py) that tests/test_gpu_gtable.py holds the device
table to, checked against an independent double-and-add, against the engine's own recoding of the single-entry scalars,
and against the host build of the table (tests/host_emul)."""
import ctypes
import random

import numpy as np
import pytest

from tests import adversarial
from tests import group_schedule as S
from tests import gtable_model as M


@pytest.fixture(scope="module")
def table():
    return M.build()


def _boundary_entries():
    """every row's d = 1, 2, 0x7FFF, 0x8000, and row 15's 0xFFFF and 0x10000"""
    out = [M.entry(r, d) for r in range(M.ROWS) for d in (1, 2, 0x7FFF, 0x8000)]
    return out + [M.entry(15, 0xFFFF), M.entry(15, 0x10000)]


def test_layout():
    assert M.ENTRIES == 557056 and M.entry(15, 0x10000) == M.ENTRIES - 1
    for e in (0, 1, M.ROW - 1, M.ROW, 15 * M.ROW - 1, 15 * M.ROW, 16 * M.ROW, M.ENTRIES - 1):
        assert M.entry(*M.row_d(e)) == e


def test_entries_against_double_and_add(table):
    """the boundary entries of every row and a seeded sample of 2,000 against adversarial.mul (double and add, one
    inversion per addition)"""
    rnd = random.Random(4242)
    es = _boundary_entries() + rnd.sample(range(M.ENTRIES), 2000)
    # d * B_row with B_row = 2^(16 row) * G, both by double and add: 17 doublings per entry instead of up to 256
    rows = [adversarial.mul(1 << (16 * r), adversarial.G) for r in range(M.ROWS)]
    assert rows[0] == adversarial.G and rows == M.bases()
    for e in es:
        row, d = M.row_d(e)
        assert M.point(table, e) == adversarial.mul(d, rows[row]), (e, row, d)
    # the scalars that select them: scalar_for(e) * G is the entry itself, except for the carry entry, whose scalar also
    # reads entry(14, 1) negated
    for e in _boundary_entries():
        want = adversarial.mul(M.scalar_for(e), adversarial.G)
        got = M.point(table, e)
        if e == M.ENTRIES - 1:
            b14 = M.point(table, M.entry(14, 1))
            got = adversarial.add(got, (b14[0], (-b14[1]) % M.P))
        assert got == want, e


def test_single_entry_scalars_recode_to_one_digit():
    """prepare_u1 (the model of sc_prepare_u1, itself checked on the device) of scalar_for(e) has exactly the digits
    digits_for(e): one non-zero digit at the entry's row with the entry's d, or (-1 at row 14, 65536 at row 15) for the
    carry entry"""
    for e in range(M.ENTRIES):
        k = M.scalar_for(e)
        assert 0 < k < M.N
        gd = S.prepare_u1(k)
        want = M.digits_for(e)
        assert {i: v for i, v in enumerate(gd) if v} == want, (e, M.row_d(e))
    assert M.digits_for(M.ENTRIES - 1) == {14: -1, 15: 65536}


def test_host_build_table_matches_model(table, emul):
    """the host build of the table (emul_gtable_build: incremental Jacobian additions, one inversion per row) equals the
    model at a stride-97 sample and at every row's first and last entries"""
    emul.emul_gtable_build()
    es = sorted(set(range(0, M.ENTRIES, 97)) | {M.entry(r, d) for r in range(M.ROWS) for d in (1, M.row_size(r))})
    xy = (ctypes.c_uint32 * 16)()
    for e in es:
        emul.emul_gtable_get(e, xy)
        assert np.array_equal(np.frombuffer(xy, dtype=np.uint32), table[e]), (e, M.row_d(e))
