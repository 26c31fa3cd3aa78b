"""The cases of test_compression_gpu.py::test_twobit_residual_over_steps without a GPU: the oracle
alone shows that they can tell summation orders apart. Where the threshold is 0.1 or 1/3 and at
least 4 sources are summed, a decode that folded the sources in reverse, or pairwise, would give
other bits than the reference's left fold (ElementwiseSum, comm.h:552-596) at every step; with
threshold 0.25 every partial sum is exact and no order can be told from another."""
import numpy as np
import pytest

from test_compression_gpu import ORDER_NSRC, ORDER_THRESHOLDS, order_trajectory, store_threshold


def pairwise(vals):
    if len(vals) == 1:
        return vals[0]
    h = len(vals) // 2
    return (pairwise(vals[:h]) + pairwise(vals[h:])).astype(np.float32)


def folds(o, deq):
    """left fold (the store's order), reversed left fold and pairwise tree of one step's sources,
    all keys of the call end to end"""
    cat = [np.concatenate([deq[k][i] for k in range(len(deq))]) for i in range(len(deq[0]))]
    return o.reduce(cat, 'device'), o.reduce(cat[::-1], 'device'), pairwise(cat)


def differs(a, b):
    return int(np.count_nonzero(a.view(np.uint32) != b.view(np.uint32)))


@pytest.mark.parametrize("t", ORDER_THRESHOLDS, ids=["t0.25", "t0.1", "t1_3"])
@pytest.mark.parametrize("nsrc", [n for n in ORDER_NSRC if n >= 4])
def test_order_cases_are_order_sensitive(oracle, t, nsrc):
    for step, (_, deq) in enumerate(order_trajectory(oracle, t, nsrc)):
        left, rev, tree = folds(oracle, deq)
        if t == 0.25:
            assert differs(left, rev) == 0 and differs(left, tree) == 0, step
        else:
            assert differs(left, rev) > 0 and differs(left, tree) > 0, step


def test_exact_threshold_cases_cannot_tell_orders(oracle):
    """t = 0.25 at every source count: the decoded values are multiples of a power of two small
    enough that every partial sum is exact"""
    for nsrc in ORDER_NSRC:
        for step, (_, deq) in enumerate(order_trajectory(oracle, 0.25, nsrc)):
            left, rev, tree = folds(oracle, deq)
            assert differs(left, rev) == 0 and differs(left, tree) == 0, (nsrc, step)


def test_store_threshold_is_dmlc_stof():
    """the store parses its threshold with dmlc::stof, which is not a correctly rounded parse: the
    threshold test_twobit_edge_values uses in exponent form lands one float above np.float32(t)"""
    for t in (0.25, 0.5, 0.1, 1 / 3):
        assert store_threshold(t) == float(np.float32(t))
    t = 1.2345e-05
    assert store_threshold(t) == float(np.nextafter(np.float32(t), np.float32(1)))


def test_oracle_edge_semantics(oracle):
    """what test_twobit_edge_values relies on the oracle's C code for: a value exactly on +-t
    fires, one ulp inside does not until the next step carries it over, NaN never fires and stays
    in the residual, +-inf fire at every step and stay infinite"""
    f = np.float32
    thr = store_threshold(1 / 3)
    g = np.array([thr, -thr, np.nextafter(f(thr), f(0)), np.nan, np.inf, -np.inf], f)
    res = np.zeros(g.size, f)
    t = float(f(thr))
    for want in ([t, -t, 0.0, 0.0, t, -t], [t, -t, t, 0.0, t, -t]):
        deq = oracle.dequantize_2bit(oracle.quantize_2bit(g, res, thr), g.size, thr)
        assert deq.tolist() == want
        assert np.isnan(res[3]) and res[4] == np.inf and res[5] == -np.inf
