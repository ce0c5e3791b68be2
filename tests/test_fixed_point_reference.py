"""CPU self-test of the exact fixed-point histogram reference (helpers.fixed_point_hist) that the bit-exact GPU tests
compare with: every cell of it lies within the fixed point's rounding, count * 2^-(k+1), of the oracle's fp64 histogram,
and the integer arithmetic holds at the 16-bit limits the kernel is designed around."""
import numpy as np
import pytest

from helpers import cell_counts, cell_sums, fixed_point_hist, fixed_point_rows, pow2_exponent


@pytest.fixture(scope="module")
def orc():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


class _Lay:
    """Identity layout (one feature per column) in the attribute form oracle_py.make_layout reads."""

    def __init__(self, bins):
        n, c = bins.shape
        self.bins, self.num_data, self.num_columns, self.num_features = bins, n, c, c
        z = np.zeros(c, np.int32)
        self.feat_column, self.feat_lo, self.feat_num_bin = np.arange(c, dtype=np.int32), np.ones(c, np.int32), np.full(c, 256, np.int32)
        self.feat_mfb, self.feat_default_bin, self.feat_missing, self.feat_real_index = z, z, z, np.arange(c, dtype=np.int32)


def test_pow2_exponent():
    assert pow2_exponent(0.0) == 0
    assert pow2_exponent(1.0) == 29                          # 1 * 2^29 < 2^30, 2^30 is not
    assert pow2_exponent(np.nextafter(np.float32(1), np.float32(0))) == 30
    assert pow2_exponent(3.0) == 28
    for b in (1e-30, 0.37, 5.0, 123456.0, 3e30):
        k = pow2_exponent(b)
        assert b * 2.0 ** k < 2 ** 30 <= b * 2.0 ** (k + 1)


def test_fixed_point_rows_round_half_even():
    q = fixed_point_rows(np.array([0.5, 1.5, 2.5, -0.5, -1.5, -2.5], np.float32), 0)
    np.testing.assert_array_equal(q, [0, 2, 2, 0, -2, -2])


def test_cell_sums_at_the_16_bit_limits():
    """|q| just below 2^30 in 65 504 rows of one cell: the hi / lo halves and their recombination stay exact."""
    n = 65504 * 3 + 7
    bins = np.zeros((n, 2), np.uint8)
    bins[:, 1] = 255
    top = 2 ** 30 - 64
    for q in (np.full(n, top), np.full(n, -top), np.where(np.arange(n) % 2 == 0, top, -top + 1)):
        s = cell_sums(bins, None, q)
        assert s[0, 0] == s[1, 255] == int(q.sum())
        assert (s[:, 1:255] == 0).all()
    rows = np.arange(0, n, 3)
    assert cell_counts(bins, rows)[0, 0] == len(rows)


@pytest.mark.parametrize("n,c,subset,const_hess", [(5000, 7, False, False), (3001, 33, True, False),
                                                    (4000, 5, False, True), (1, 3, False, False)])
def test_fixed_point_hist_within_rounding_of_oracle(orc, n, c, subset, const_hess):
    rng = np.random.default_rng(n + c)
    bins = rng.integers(0, 256, (n, c), dtype=np.uint8)
    bins[: n // 2, 0] = 3                                     # one crowded cell
    g = (rng.normal(size=n) * 3).astype(np.float32)
    h = np.full(n, 0.7, np.float32) if const_hess else (rng.random(n) + 0.05).astype(np.float32)
    rows = np.sort(rng.choice(n, n // 3, replace=False)).astype(np.int32) if subset else None
    sums, vals, (kg, kh) = fixed_point_hist(bins, rows, g, h, const_hess=const_hess)
    want = orc.construct_histogram(_Lay(bins), rows, g, h)
    cnt = cell_counts(bins, rows)
    assert (np.abs(vals[..., 0] - want[..., 0]) <= cnt * 2.0 ** -(kg + 1)).all()
    assert (np.abs(vals[..., 1] - want[..., 1]) <= cnt * 2.0 ** -(kh + 1)).all()
    assert np.array_equal(vals[..., 1] == 0, cnt == 0)
    # the integers are what the values say, and the scale came from ALL rows, not the subset
    assert kg == pow2_exponent(np.abs(g).max())
    np.testing.assert_array_equal(np.ldexp(vals[..., 0], kg), sums[..., 0].astype(np.float64))
