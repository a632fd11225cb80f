"""The novelty oracle (oracle/novelty_oracle.py) without a GPU: its distances are scipy's cKDTree's, and its order is
the contract's (ties to the lower row, NaN rows after every number, k > A takes every row, A = 1).  Its fp32 fmaf is
correctly rounded, and its blend at w = 1 is the centered rank bit for bit."""
import numpy as np
import pytest

from oracle import nes_oracle as orc
from oracle import novelty_oracle as no

spatial = pytest.importorskip('scipy.spatial')


@pytest.mark.parametrize('n,A,d,k', [(7, 50, 3, 10), (20, 300, 24, 5), (3, 40, 32, 32), (5, 1, 3, 10), (4, 6, 2, 10)])
def test_distances_are_the_kd_tree_s(n, A, d, k):
    rs = np.random.RandomState(n * A + d)
    q = rs.randn(n, d).astype(np.float32)
    a = rs.randn(A, d).astype(np.float32)
    dist, _ = spatial.cKDTree(a.astype(np.float64)).query(q.astype(np.float64), k=min(k, A))
    dist = np.asarray(dist, dtype=np.float64).reshape(n, -1)
    want = np.array([sum(float(x) for x in row) / row.size for row in dist])
    np.testing.assert_allclose(no.novelty(q, a, k), want, rtol=1e-12)
    # the fp32 restatement is within a few ulps of it (d fp32 roundings of the squares and sums, one of the sqrt)
    np.testing.assert_allclose(no.novelty_fp32(q, a, k), want, rtol=(d + 4) * 2.0 ** -24)


def test_ties_go_to_the_lower_row_and_nan_rows_come_last():
    a = np.array([[2, 0], [0, 1], [np.nan, 0], [1, 0], [0, 2], [0, -1]], dtype=np.float32)
    q = np.zeros((1, 2), dtype=np.float32)
    d2 = no.sq_distances_fp32(q, a)[0]
    assert np.argsort(d2, kind='stable').tolist() == [1, 3, 5, 0, 4, 2]
    assert no.novelty_fp32(q, a, 3)[0] == np.float32(1.0)
    assert no.novelty_fp32(q, a, 5)[0] == np.float32((1 + 1 + 1 + 2 + 2) / 5)
    assert np.isnan(no.novelty_fp32(q, a, 6)[0])                 # the NaN row is the sixth
    assert np.isnan(no.novelty_fp32(np.full((1, 2), np.nan, np.float32), a, 1)[0])


def test_k_past_the_archive_takes_every_row():
    a = np.array([[3, 4], [0, 0]], dtype=np.float32)
    q = np.zeros((1, 2), dtype=np.float32)
    assert no.novelty_fp32(q, a, 10)[0] == np.float32(2.5)
    assert no.novelty_fp32(q, a[:1], 32)[0] == np.float32(5.0)      # A = 1


def test_fmaf32_is_correctly_rounded():
    rs = np.random.RandomState(3)
    a, b, c = (rs.randn(20000).astype(np.float32) for _ in range(3))
    from fractions import Fraction
    got = no.fmaf32(a, b, c)
    for i in range(0, 20000, 97):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))                    # within one ulp; pick the nearer of its neighbours
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda x: (abs(Fraction(float(x)) - exact), int(np.float32(x).view(np.uint32)) & 1))
        assert got[i] == best, i


def test_blend_at_w_1_is_the_centered_rank_and_at_w_0_the_novelty_rank():
    rs = np.random.RandomState(0)
    f, nov = rs.randn(65).astype(np.float32), rs.rand(65).astype(np.float32)
    s_f = orc.fitness_shift(f).astype(np.float32)
    assert no.blend(f, nov, 1.0).tobytes() == s_f.tobytes()
    assert no.blend(f, nov, 0.0).tobytes() == orc.fitness_shift(nov).astype(np.float32).tobytes()


def test_the_nsra_schedule():
    w, stall = 1.0, 0
    w, stall = no.adapt(w, stall, True)
    assert (w, stall) == (1.0, 0)
    for i in range(9):
        w, stall = no.adapt(w, stall, False)
    assert (w, stall) == (1.0, 9)
    w, stall = no.adapt(w, stall, False)
    assert (w, stall) == (0.95, 0)
    w, stall = no.adapt(w, stall, True)
    assert (w, stall) == (1.0, 0)
    w = 0.02
    for i in range(10):
        w, stall = no.adapt(w, stall, False)
    assert w == 0.0


def test_the_integer_oracle_is_the_fp32_one():
    rs = np.random.RandomState(7)
    for n, A, d, k in ((9, 40, 3, 10), (5, 7, 32, 32), (4, 1, 1, 3), (6, 300, 24, 1)):
        q = rs.randint(-8, 9, size=(n, d)).astype(np.float32)
        a = rs.randint(-8, 9, size=(A, d)).astype(np.float32)
        a[rs.rand(A) < 0.1, 0] = np.nan
        q[0, -1] = np.nan
        np.testing.assert_array_equal(no.novelty_integer(q, a, k, chunk=4), no.novelty_fp32(q, a, k))
