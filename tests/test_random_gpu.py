"""_random_normal and mx.random.seed on the GPU, bit for bit against the reference's own GPU sampler
(oracle/_ref/libmxref_random_gpu.so, built by oracle/random_gpu.mk; oracle/golden_random.py keeps
the reference's 4 generator copies per GPU, its round robin and its seeds in host memory):

- every dtype at N = 1, 63, 64, 65, 64*32768 - 1, 64*32768, 64*32768 + 1, 10 M and 64 M;
- loc / scale from tiny to huge, negative loc; each parsed once to float as the operator does;
- an unaligned out slice and runs that are not a whole number of 16-B vectors;
- nine calls in a row with odd N (the round robin twice, each state's cached Box-Muller value
  carried over), and the state arrays of all 4 copies after them;
- seed(s) and seed(s, ctx=gpu(0)) each start their stream again; different seeds differ;
- every refusal leaves the next call's output as if it had not happened;
- a short statistical check (mean, variance, KS at 10^6 samples), for readers, not for parity."""
import ctypes
import math

import numpy as np
import pytest

import golden_random as GR
import kvoracle as K

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(GR.ref() is None, reason="needs oracle/_ref/libmxref_random_gpu.so")]
DTYPES = ['float16', 'bfloat16', 'float32', 'float64']
BITS = {'float16': np.uint16, 'bfloat16': np.uint16, 'float32': np.uint32, 'float64': np.uint64}
SIZES = [1, 63, 64, 65, 64 * 32768 - 1, 64 * 32768, 64 * 32768 + 1, 10_000_000, 64 << 20]


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def f32(x):
    """the float32 the operator parses from str(x) (dmlc::stof)"""
    return float(K.dmlc_stof(str(x)))


def bits(nd, dtype):
    x = nd.asnumpy()
    if dtype == 'bfloat16':
        return (x.view(np.uint32) >> 16).astype(np.uint16).ravel()
    return x.view(BITS[dtype]).ravel()


def want_bits(x, dtype):
    return np.ascontiguousarray(x).view(BITS[dtype]).ravel()


def check(got, want, what):
    if np.array_equal(got, want):
        return
    bad = np.nonzero(got != want)[0] if got.shape == want.shape else []
    pytest.fail('%s: %d of %d elements differ, first at %s' % (what, len(bad), want.size, bad[:6]))


def start(mx, seed):
    mx.random.seed(seed)
    return GR.RefGenerators(0, seed)


def lib_states(mx, copy):
    buf = np.zeros(GR.NUM_STATES * GR.STATE_BYTES, np.uint8)
    mx.base.check_call(mx.base._LIB.B200KVRandomStates(0, copy, buf.ctypes.data_as(ctypes.c_void_p),
                                                        ctypes.c_size_t(buf.size)))
    return buf


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_and_size(mx, dtype, n):
    ref = start(mx, 7)
    out = mx.random.normal(0, 1, shape=(n,), dtype=dtype, ctx=mx.gpu(0))
    check(bits(out, dtype), want_bits(ref.normal(n, 0.0, 1.0, dtype), dtype), '%s n=%d' % (dtype, n))


PARAMS = [(0, 1), (-3.5, 0.25), (2.0, 1e-30), (-1e-3, 2e-38), (0.1, 1e30), (-1e30, 3e38), (1e4, 7.0)]


@pytest.mark.parametrize("loc,scale", PARAMS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_loc_scale(mx, dtype, loc, scale):
    ref = start(mx, 123)
    n = 100_003
    out = mx.random.normal(loc, scale, shape=(n,), dtype=dtype, ctx=mx.gpu(0))
    want = ref.normal(n, f32(loc), f32(scale), dtype)
    check(bits(out, dtype), want_bits(want, dtype), '%s loc=%r scale=%r' % (dtype, loc, scale))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [4097, 100, 64 * 32768 + 5])
def test_unaligned_out_slice(mx, dtype, n):
    """out = a[1:] of a fresh array: element 0 stays, the rest is the stream (scalar store path)"""
    ref = start(mx, 99)
    a = mx.random.normal(0, 1, shape=(n + 1,), dtype=dtype, ctx=mx.gpu(0))
    first = bits(a, dtype)[0]
    ref.normal(n + 1, 0.0, 1.0, dtype)
    mx.random.normal(-1.0, 2.0, dtype=dtype, out=a[1:])
    got = bits(a, dtype)
    assert got[0] == first
    check(got[1:], want_bits(ref.normal(n, -1.0, 2.0, dtype), dtype), 'slice %s n=%d' % (dtype, n))


def test_nine_calls_and_states(mx):
    """odd N leaves a cached Box-Muller value in states that draw an odd count; nine calls take
    copies 1, 2, 3, 0, 1, 2, 3, 0, 1; every copy's 32768 states equal the reference's afterwards"""
    ref = start(mx, 2024)
    for k in range(9):
        dtype = DTYPES[k % 4]
        n = 64 * 32768 + 2 * k + 1 if k % 3 == 0 else 999 + 64 * k
        out = mx.random.normal(0.5, 1.5, shape=(n,), dtype=dtype, ctx=mx.gpu(0))
        check(bits(out, dtype), want_bits(ref.normal(n, 0.5, 1.5, dtype), dtype), 'call %d' % k)
    for c in range(GR.COPIES):
        assert np.array_equal(lib_states(mx, c), ref.copies[c]), 'copy %d states differ' % c


def test_seed_all_restarts_the_stream(mx):
    def draws():
        return [bits(mx.random.normal(0, 1, shape=(5000 + i,), ctx=mx.gpu(0)), 'float32') for i in range(5)]
    mx.random.seed(31)
    a = draws()
    mx.random.seed(31)
    b = draws()
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    mx.random.seed(32)
    c = draws()
    assert not any(np.array_equal(x, y) for x, y in zip(a, c))


def test_seed_ctx_restarts_the_stream(mx):
    mx.random.seed(5, ctx=mx.gpu(0))
    ref = GR.RefGenerators(0, 0)
    ref.seed_ctx(5)
    a = [mx.random.normal(0, 1, shape=(777,), ctx=mx.gpu(0)) for _ in range(5)]
    for i, x in enumerate(a):
        check(bits(x, 'float32'), want_bits(ref.normal(777, 0.0, 1.0, 'float32'), 'float32'), 'ctx call %d' % i)
    mx.random.seed(5, ctx=mx.gpu(0))
    b = mx.random.normal(0, 1, shape=(777,), ctx=mx.gpu(0))
    assert np.array_equal(bits(b, 'float32'), bits(a[0], 'float32'))
    # the per-device seed has no device term, which is 0 on gpu(0): seed(5) draws the same there,
    # and seed(6) on this device does not
    mx.random.seed(5)
    c = mx.random.normal(0, 1, shape=(777,), ctx=mx.gpu(0))
    assert np.array_equal(bits(c, 'float32'), bits(a[0], 'float32'))
    mx.random.seed(6, ctx=mx.gpu(0))
    d = mx.random.normal(0, 1, shape=(777,), ctx=mx.gpu(0))
    assert not np.array_equal(bits(d, 'float32'), bits(a[0], 'float32'))


def test_refusals_leave_the_stream_and_out(mx):
    ref = start(mx, 77)
    o = mx.nd.array(np.arange(10, dtype=np.float32), mx.gpu(0))
    before = o.asnumpy().copy()
    rsp = mx.nd.sparse.zeros('row_sparse', (10, 3), mx.gpu(0))
    calls = [
        (lambda: mx.random.normal(0, 0, shape=(10,), ctx=mx.gpu(0)), 'scale parameter in gaussian has to be positive'),
        (lambda: mx.random.normal(0, -1, out=o), 'scale parameter in gaussian has to be positive'),
        (lambda: mx.random.normal(0, float('nan'), out=o), 'scale parameter in gaussian has to be positive'),
        (lambda: mx.random.normal(0, 1, shape=(10,), ctx=mx.cpu(0)), 'GPU only'),
        (lambda: mx.random.normal(0, 1, shape=(10,), ctx=mx.gpu(0), foo=1), "Cannot find argument 'foo'"),
        (lambda: mx.random.normal(0, 1, shape=(11,), out=o), 'wrong shape'),
        (lambda: mx.random.normal(0, 1, dtype='float16', out=o), 'differs from dtype'),
        (lambda: mx.random.normal(0, 1, shape=(10,), dtype='int32', ctx=mx.gpu(0)), 'Invalid Input'),
        (lambda: mx.random.normal(0, 1, out=rsp), 'dense'),
    ]
    for call, match in calls:
        with pytest.raises(mx.MXNetError, match=match):
            call()
    assert np.array_equal(o.asnumpy(), before)
    got = mx.random.normal(0, 1, out=o)
    check(bits(got, 'float32'), want_bits(ref.normal(10, 0.0, 1.0, 'float32'), 'float32'), 'after refusals')


def test_statistics(mx):
    from scipy import stats
    mx.random.seed(1)
    x = mx.random.normal(3.0, 2.0, shape=(1_000_000,), ctx=mx.gpu(0)).asnumpy().astype(np.float64)
    assert abs(x.mean() - 3.0) < 0.01
    assert abs(x.var() / 4.0 - 1.0) < 0.01
    assert stats.kstest((x - 3.0) / 2.0, 'norm').pvalue > 1e-4
    assert math.isfinite(x.sum())
