"""The stored factor, bit for bit, on the matrices of tests/factor_digest.py: the shape matrices of tests/ldl_shapes.py
(every front shape the factor kernels dispatch on, and one regularised pivot in each kind of front, wide F and D
fronts included), and the C4 block-angular QP at 1/25 of its size, whose level 0 holds thousands of wide fronts.

tests/golden/ldl/factor_digests.json was written on an H100 by the build whose level-0 kernel factored the pivot block
column by column with one thread per pivot and per-pivot counter atomics, and whose pivot-block inverses were a
separate pass over the finished panels.  Every entry of L (inverted pivot blocks included), D and 1/D, and the
regularisation and inertia counts, must be what that build stored: the faster kernels do the same operations in the
same order per entry.  scripts/make_factor_digests.py regenerates the file."""
import json
import os

import pytest

import factor_digest

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ldl", "factor_digests.json")
with open(GOLDEN) as _fp:
    WANT = json.load(_fp)


@pytest.mark.parametrize("name", sorted(WANT))
def test_factor_is_bitwise_the_golden_one(name):
    want = WANT[name]
    s = factor_digest.solver(factor_digest.case(name))
    got = factor_digest.digest(s)
    assert got == want
    # a second refactor of the same values stores the same bits
    assert factor_digest.digest(s) == want
    s.close()


def test_golden_covers_every_case():
    assert sorted(WANT) == sorted(c.name for c in factor_digest.cases())
