"""The NDArray arithmetic, fill and cast operators without a GPU: the numpy restatements of
oracle/golden_ndarray_ops.py against the reference's own code (oracle/_ref/libmxref_ndarith.so) on
every case, on all 65,536 float16 bit patterns, and on the scalar and value parses; and
tests/golden/ndarray_ops.npz against both."""
import math

import numpy as np
import pytest

import golden_ndarray_ops as G

live = pytest.mark.skipif(G.ref() is None, reason="needs oracle/_ref/libmxref_ndarith.so")
KINDS = ('array', 'scalar', 'full', 'cast')


@pytest.fixture(scope="module")
def fixture():
    d = np.load(G.os.path.join(G.GOLD, "ndarray_ops.npz"))
    return {str(n): (s, h) for n, s, h in zip(d['names'], d['sha256'], d['head'])}


def test_fixture_lists_every_case(fixture):
    names = [case[0] for _, case in G.all_cases()]
    assert len(set(names)) == len(names)
    assert sorted(names) == sorted(fixture)


@pytest.mark.parametrize("kind", KINDS)
def test_restatement_equals_fixture(fixture, kind):
    for k, case in G.all_cases():
        if k != kind:
            continue
        out = G.restate(kind, case)
        dt = G.out_dtype(kind, case)
        sha, head = fixture[case[0]]
        assert np.array_equal(G.head_bytes(out, dt), head), case[0]
        assert np.array_equal(G.sha256(out, dt), sha), case[0]


@live
@pytest.mark.parametrize("kind", KINDS)
def test_library_equals_restatement_and_fixture(fixture, kind):
    n = 0
    for k, case in G.all_cases():
        if k != kind:
            continue
        got = G.live(kind, case)
        if got is None:           # bfloat16: the reference has none
            continue
        dt = G.out_dtype(kind, case)
        assert G.same(got, G.restate(kind, case), dt), case[0]
        assert np.array_equal(G.sha256(got, dt), fixture[case[0]][0]), case[0]
        n += 1
    assert n > 0


# ------------------------------------------------------------------------- every float16 value
ALL_HALVES = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)
PARTNERS = [0.1, 1.0, -3.5, 65504.0, 6e-8, -0.0, math.inf, math.nan]


@live
def test_every_float16_through_sqrt_add_mul_and_scalars():
    r = G.ref()
    h = ALL_HALVES
    assert G.same(r.sqrt(h, 'float16'), G.sqrt(h, 'float16'), 'float16')
    for p in PARTNERS:
        b = np.full(h.shape, p, np.float16)
        for op in ('plus', 'minus', 'mul'):
            assert G.same(r.binary(op, h, b, 'float16'), G.binary(op, h, b, 'float16'), 'float16'), (op, p)
            assert G.same(r.binary(op, b, h, 'float16'), G.binary(op, b, h, 'float16'), 'float16'), (op, p)
    for s in ('0.1', '-2.5', '1e-08', '65519.0', '1.00048828125', '1.2345e-05'):
        for op in ('plus', 'mul'):
            assert G.same(r.binary_scalar(op, h, s, 'float16'),
                          G.binary_scalar(op, h, s, 'float16'), 'float16'), (op, s)


def test_half_scalar_is_rounded_to_half_before_the_add():
    """h + 0.1 adds half(0.1), not float(0.1): the two differ on many halves"""
    h = ALL_HALVES[np.isfinite(ALL_HALVES)]
    want = G.binary_scalar('plus', h, '0.1', 'float16')
    unrounded = (h.astype(np.float32) + np.float32(0.1)).astype(np.float16)
    assert (want.view(np.uint16) != unrounded.view(np.uint16)).sum() > 10000


@live
def test_every_float16_cast_to_every_dtype_and_back():
    r = G.ref()
    h = ALL_HALVES
    for dst in ('float32', 'float64'):
        wide = r.cast(h, 'float16', dst)
        assert G.same(wide, G.cast(h, 'float16', dst), dst)
        assert G.same(r.cast(wide, dst, 'float16'), h, 'float16')
    for dst in ('int32', 'int64'):
        fin = h[np.isfinite(h)]
        assert G.same(r.cast(fin, 'float16', dst), G.cast(fin, 'float16', dst), dst)
    # the float32 and float64 values half-way between neighbouring halves: ties go to even
    fin = np.sort(h[np.isfinite(h) & (h >= 0)].astype(np.float64))
    mids = np.concatenate([(fin[:-1] + fin[1:]) / 2, [65520.0, 65519.996]])
    mids = np.concatenate([mids, -mids])
    for src in ('float32', 'float64'):
        x = mids.astype(G.STORE[src])
        assert G.same(r.cast(x, src, 'float16'), G.cast(x, src, 'float16'), 'float16'), src
    ints = np.arange(-70000, 70000, dtype=np.int64)
    for src in ('int32', 'int64'):
        x = ints.astype(G.STORE[src])
        assert G.same(r.cast(x, src, 'float16'), G.cast(x, src, 'float16'), 'float16'), src


# ------------------------------------------------------------------------------------- parses
@live
def test_scalar_is_parsed_by_stod_not_dmlc_stof():
    """the *_scalar operators parse with std::stod and round once; dmlc::stof differs on the
    fixture's differing strings"""
    r = G.ref()
    d = np.load(G.os.path.join(G.GOLD, 'scalar_parse.npz'))
    stof = {repr(float(v)): p for v, p in zip(d['values'], d['parsed'])}
    diff = G._differing_parses()
    assert len(diff) > 100
    one = np.ones(1, np.float32)
    for s in diff:
        got = r.binary_scalar('mul', one, s, 'float32')[0]
        assert got.view(np.uint32) == np.float32(float(s)).view(np.uint32), s
        assert got.view(np.uint32) != np.float32(stof[s]).view(np.uint32), s
    got = r.binary_scalar('mul', one, '1.2345e-05', 'float32')[0]
    assert got.view(np.uint32) == np.float32(1.2345e-05).view(np.uint32)


@live
def test_integer_scalar_is_truncated_first():
    r = G.ref()
    three = np.array([3, -3], np.int32)
    assert r.binary_scalar('mul', three, '2.5', 'int32').tolist() == [6, -6]
    assert r.binary_scalar('plus', three, '-0.9', 'int32').tolist() == [3, -3]
    assert G.binary_scalar('mul', three, '2.5', 'int32').tolist() == [6, -6]


@live
@pytest.mark.parametrize("value", G.FULL_VALUES + [1 / 3, 1e-300, 123456.789, 2.0 ** 70, -7.25e-5])
def test_full_value_parse(value):
    """_full's value goes through dmlc::stod (not always correctly rounded), restated by dmlc_stod"""
    parsed, _ = G.ref().full(value, 1, 'float64')
    want = G.dmlc_stod(repr(float(value)))
    assert parsed == want or (math.isnan(parsed) and math.isnan(want))


@live
def test_examples():
    r = G.ref()
    a = np.array([2 ** 40 + 1], np.int64)
    assert r.binary('plus', a, np.zeros(1, np.int64), 'int64')[0] == 2 ** 40 + 1
    assert r.binary_scalar('plus', np.array([0.1]), '0', 'float64')[0] == 0.1
    assert r.sqrt(np.array([16785408], np.int32), 'int32')[0] == 4096
    assert r.cast(np.array([2 ** 53 - 1], np.int64), 'int64', 'int64')[0] == 2 ** 53 - 1
    assert r.full(2 ** 24 + 1, 1, 'int64')[1][0] == 2 ** 24 + 1
    assert r.full(-0.0, 1, 'float32')[1].view(np.uint32)[0] == 0        # Fill's val == 0 branch
