"""_random_uniform, _random_exponential, _random_gamma, _random_randint and the _like forms on the
GPU, bit for bit against the reference's own GPU samplers (oracle/_ref/libmxref_sample_gpu.so and
libmxref_random_gpu.so, built by oracle/sample_gpu.mk and oracle/random_gpu.mk;
oracle/golden_sample.py keeps the reference's 4 generator copies per GPU, its round robin and its
seeds in host memory, and draws every sampler from them in turn):

- every operator at every dtype at N = 1, 63, 64, 65, 64*32768 - 1, 64*32768, 64*32768 + 1 and
  10 M, float32 also at 64 M;
- parameter edges: an empty or huge uniform range, tiny and huge lam, gamma's alpha < 1 branch and
  heavy rejection, randint ranges of 1, 2, 2^31 and past 2^33, negative low, and int32 wrapping;
- twelve calls that interleave all five distributions with odd N share one stream, and the state
  arrays of all 4 copies equal the reference's after them; seed(s) and seed(s, ctx) restart it;
- an unaligned out slice takes the scalar store path and leaves element 0 alone;
- the _like forms take data's shape and dtype, and out may be data;
- every refusal leaves out and the next draw as if it had not happened;
- mean, variance and KS at 10^6 samples per distribution, for readers, not for parity."""
import ctypes
import math

import numpy as np
import pytest

import golden_random as GR
import golden_sample as GS
import kvoracle as K

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not GS.available(),
                                 reason="needs oracle/_ref/libmxref_random_gpu.so and libmxref_sample_gpu.so")]
FLOATS = ['float16', 'bfloat16', 'float32', 'float64']
BITS = {'float16': np.uint16, 'bfloat16': np.uint16, 'float32': np.uint32, 'float64': np.uint64,
        'int32': np.uint32, 'int64': np.uint64}
SIZES = [1, 63, 64, 65, 64 * 32768 - 1, 64 * 32768, 64 * 32768 + 1, 10_000_000]


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
    return GS.SampleGenerators(0, seed)


def lib_states(mx, copy):
    buf = np.zeros(GR.NUM_STATES * GR.STATE_BYTES, np.uint8)
    mx.base.check_call(mx.base._LIB.B200KVRandomStates(0, copy, buf.ctypes.data_as(ctypes.c_void_p),
                                                        ctypes.c_size_t(buf.size)))
    return buf


# (distribution, python call, reference call) with the parameters of each size / dtype case
def _uniform(mx, ref, n, dtype, **kw):
    return (mx.random.uniform(-1.5, 2.5, shape=(n,), dtype=dtype, ctx=mx.gpu(0), **kw),
            ref.uniform(n, -1.5, 2.5, dtype))


def _exponential(mx, ref, n, dtype, **kw):
    return (mx.random.exponential(0.25, shape=(n,), dtype=dtype, ctx=mx.gpu(0), **kw),
            ref.exponential(n, f32(1.0 / 0.25), dtype))


def _gamma(mx, ref, n, dtype, **kw):
    return (mx.random.gamma(0.7, 2.0, shape=(n,), dtype=dtype, ctx=mx.gpu(0), **kw),
            ref.gamma(n, f32(0.7), 2.0, dtype))


def _randint(mx, ref, n, dtype, **kw):
    return (mx.random.randint(-7, 1 << 34, shape=(n,), dtype=dtype, ctx=mx.gpu(0), **kw),
            ref.randint(n, -7, 1 << 34, dtype))


DRAWS = {'uniform': _uniform, 'exponential': _exponential, 'gamma': _gamma, 'randint': _randint}
CASES = [(d, t) for d in ('uniform', 'exponential', 'gamma') for t in FLOATS] + \
        [('randint', 'int32'), ('randint', 'int64')]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("dist,dtype", CASES)
def test_every_dtype_and_size(mx, dist, dtype, n):
    ref = start(mx, 7)
    got, want = DRAWS[dist](mx, ref, n, dtype)
    check(bits(got, dtype), want_bits(want, dtype), '%s %s n=%d' % (dist, dtype, n))


@pytest.mark.parametrize("dist", ['uniform', 'exponential', 'gamma', 'randint'])
def test_float32_64m(mx, dist):
    ref = start(mx, 8)
    dtype = 'int32' if dist == 'randint' else 'float32'
    got, want = DRAWS[dist](mx, ref, 64 << 20, dtype)
    check(bits(got, dtype), want_bits(want, dtype), '%s 64M' % dist)


def test_randint_defaults_to_int32(mx):
    ref = start(mx, 3)
    got = mx.random.randint(0, 10, shape=(1000,), ctx=mx.gpu(0))
    assert got.dtype == np.int32
    check(bits(got, 'int32'), want_bits(ref.randint(1000, 0, 10, 'int32'), 'int32'), 'default dtype')


UNIFORM = [(0.0, 0.0), (3.25, 3.25), (-5.0, -1e-3), (-3e38, 3e38), (1e-30, 2e-30), (-1e4, 1e30)]


@pytest.mark.parametrize("low,high", UNIFORM)
@pytest.mark.parametrize("dtype", FLOATS)
def test_uniform_edges(mx, dtype, low, high):
    ref = start(mx, 21)
    n = 100_003
    got = mx.random.uniform(low, high, shape=(n,), dtype=dtype, ctx=mx.gpu(0))
    check(bits(got, dtype), want_bits(ref.uniform(n, f32(low), f32(high), dtype), dtype),
          'uniform %s [%r, %r)' % (dtype, low, high))


@pytest.mark.parametrize("scale", [1e-30, 1e-3, 1.0, 1e3, 1e30])
@pytest.mark.parametrize("dtype", FLOATS)
def test_exponential_edges(mx, dtype, scale):
    ref = start(mx, 22)
    n = 100_003
    got = mx.random.exponential(scale, shape=(n,), dtype=dtype, ctx=mx.gpu(0))
    check(bits(got, dtype), want_bits(ref.exponential(n, f32(1.0 / scale), dtype), dtype),
          'exponential %s scale=%r' % (dtype, scale))


@pytest.mark.parametrize("alpha", [1e-3, 0.5, 1.0, 1.5, 9.0, 1e4])
@pytest.mark.parametrize("beta", [1e-3, 1.0, 7.5])
@pytest.mark.parametrize("dtype", FLOATS)
def test_gamma_edges(mx, dtype, alpha, beta):
    ref = start(mx, 23)
    n = 65_537
    got = mx.random.gamma(alpha, beta, shape=(n,), dtype=dtype, ctx=mx.gpu(0))
    check(bits(got, dtype), want_bits(ref.gamma(n, f32(alpha), f32(beta), dtype), dtype),
          'gamma %s alpha=%r beta=%r' % (dtype, alpha, beta))


RANGES = [(0, 1), (-9, -8), (0, 2), (-1, 1), (0, 1 << 31), (-(1 << 31), 0), (0, 1 << 32),
          (5, (1 << 33) + 12345), (-(1 << 40), 1 << 40), (-(1 << 62), (1 << 62) - 1),
          (1 << 31, (1 << 31) + 3), ((1 << 40) - 3, (1 << 40) + 100)]


@pytest.mark.parametrize("low,high", RANGES)
@pytest.mark.parametrize("dtype", ['int32', 'int64'])
def test_randint_edges(mx, dtype, low, high):
    """ranges of 1 and 2, 2^31 and 2^32, past 2^33 (every value is rand_int64() itself), negative
    low; int32 outputs of values outside int32 wrap as the reference's OType(x) does"""
    ref = start(mx, 24)
    n = 100_003
    got = mx.random.randint(low, high, shape=(n,), dtype=dtype, ctx=mx.gpu(0))
    want = ref.randint(n, low, high, dtype)
    check(bits(got, dtype), want_bits(want, dtype), 'randint %s [%d, %d)' % (dtype, low, high))
    if dtype == 'int64':
        x = got.asnumpy()
        assert x.min() >= low and x.max() < high


def test_twelve_mixed_calls_and_states(mx):
    """odd N leaves a cached Box-Muller value in states that draw an odd count of normals; the next
    uniform, randint or gamma draw on the same copy continues the same Philox stream. Twelve calls
    take copies 1, 2, 3, 0 three times; every copy's states equal the reference's afterwards."""
    ref = start(mx, 2025)
    gpu = mx.gpu(0)
    calls = [
        ('normal', 'float32', lambda n: mx.random.normal(0.5, 1.5, shape=(n,), ctx=gpu),
         lambda n: ref.normal(n, 0.5, 1.5, 'float32')),
        ('uniform', 'float64', lambda n: mx.random.uniform(-1, 1, shape=(n,), dtype='float64', ctx=gpu),
         lambda n: ref.uniform(n, -1.0, 1.0, 'float64')),
        ('randint', 'int64', lambda n: mx.random.randint(-3, 1 << 35, shape=(n,), dtype='int64', ctx=gpu),
         lambda n: ref.randint(n, -3, 1 << 35, 'int64')),
        ('gamma', 'float16', lambda n: mx.random.gamma(0.3, 2, shape=(n,), dtype='float16', ctx=gpu),
         lambda n: ref.gamma(n, f32(0.3), 2.0, 'float16')),
        ('exponential', 'bfloat16', lambda n: mx.random.exponential(3, shape=(n,), dtype='bfloat16', ctx=gpu),
         lambda n: ref.exponential(n, f32(1.0 / 3), 'bfloat16')),
        ('normal', 'float64', lambda n: mx.random.normal(0, 1, shape=(n,), dtype='float64', ctx=gpu),
         lambda n: ref.normal(n, 0.0, 1.0, 'float64')),
    ]
    for k in range(12):
        name, dtype, mine, theirs = calls[k % len(calls)]
        n = 64 * 32768 + 2 * k + 1 if k % 4 == 0 else 1001 + 66 * k
        check(bits(mine(n), dtype), want_bits(theirs(n), dtype), 'call %d (%s)' % (k, name))
    for c in range(GR.COPIES):
        assert np.array_equal(lib_states(mx, c), ref.copies[c]), 'copy %d states differ' % c


def _mixed(mx, ctx):
    return [bits(mx.random.uniform(shape=(999,), ctx=ctx), 'float32'),
            bits(mx.random.normal(shape=(1001,), ctx=ctx), 'float32'),
            bits(mx.random.gamma(0.5, shape=(777,), ctx=ctx), 'float32'),
            bits(mx.random.randint(0, 100, shape=(555,), ctx=ctx), 'int32'),
            bits(mx.random.exponential(shape=(333,), ctx=ctx), 'float32')]


def test_seed_restarts_the_mixed_sequence(mx):
    gpu = mx.gpu(0)
    mx.random.seed(41)
    a = _mixed(mx, gpu)
    mx.random.seed(41)
    b = _mixed(mx, gpu)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    mx.random.seed(41, ctx=gpu)
    ref = GS.SampleGenerators(0, 0)
    ref.seed_ctx(41)
    c = _mixed(mx, gpu)
    want = [ref.uniform(999, 0.0, 1.0, 'float32'), ref.normal(1001, 0.0, 1.0, 'float32'),
            ref.gamma(777, 0.5, 1.0, 'float32'), ref.randint(555, 0, 100, 'int32'),
            ref.exponential(333, 1.0, 'float32')]
    for i, (x, w) in enumerate(zip(c, want)):
        dt = 'int32' if i == 3 else 'float32'
        check(x, want_bits(w, dt), 'seed ctx call %d' % i)
    # the per-device seed has no device term, which is 0 on gpu(0)
    assert all(np.array_equal(x, y) for x, y in zip(a, c))


@pytest.mark.parametrize("dist,dtype", [('uniform', 'float16'), ('exponential', 'float32'),
                                        ('gamma', 'float64'), ('gamma', 'bfloat16'),
                                        ('randint', 'int32'), ('randint', 'int64')])
@pytest.mark.parametrize("n", [4097, 100, 64 * 32768 + 5])
def test_unaligned_out_slice(mx, dist, dtype, n):
    """out = a[1:]: element 0 stays, the rest is the stream (scalar store path)"""
    ref = start(mx, 99)
    a, _ = DRAWS[dist](mx, ref, n + 1, dtype)
    first = bits(a, dtype)[0]
    calls = {'uniform': (lambda o: mx.random.uniform(-1.5, 2.5, out=o), lambda: ref.uniform(n, -1.5, 2.5, dtype)),
             'exponential': (lambda o: mx.random.exponential(0.25, out=o),
                             lambda: ref.exponential(n, f32(1.0 / 0.25), dtype)),
             'gamma': (lambda o: mx.random.gamma(0.7, 2.0, out=o), lambda: ref.gamma(n, f32(0.7), 2.0, dtype)),
             'randint': (lambda o: mx.random.randint(-7, 1 << 34, out=o),
                         lambda: ref.randint(n, -7, 1 << 34, dtype))}
    mine, theirs = calls[dist]
    mine(a[1:])
    got = bits(a, dtype)
    assert got[0] == first
    check(got[1:], want_bits(theirs(), dtype), 'slice %s %s n=%d' % (dist, dtype, n))


LIKE = [('uniform_like', {'low': -2, 'high': 5}, lambda r, n, t: r.uniform(n, -2.0, 5.0, t)),
        ('normal_like', {'loc': 1, 'scale': 3}, lambda r, n, t: r.normal(n, 1.0, 3.0, t)),
        ('exponential_like', {'lam': 4}, lambda r, n, t: r.exponential(n, 4.0, t)),
        ('gamma_like', {'alpha': 0.4, 'beta': 2}, lambda r, n, t: r.gamma(n, f32(0.4), 2.0, t))]


@pytest.mark.parametrize("name,params,theirs", LIKE, ids=[x[0] for x in LIKE])
@pytest.mark.parametrize("dtype", FLOATS)
def test_like_forms(mx, name, params, theirs, dtype):
    """shape and dtype from data, data unchanged; then out = data draws into data itself"""
    ref = start(mx, 55)
    data = mx.nd.zeros((37, 129), mx.gpu(0), dtype=dtype)
    data[:] = 3
    before = bits(data, dtype).copy()
    fn = getattr(mx.nd.random, name)
    got = fn(data, **params)
    assert got.shape == (37, 129) and got.dtype == data.dtype
    n = 37 * 129
    check(bits(got, dtype), want_bits(theirs(ref, n, dtype), dtype), name)
    assert np.array_equal(bits(data, dtype), before)
    fn(data, out=data, **params)
    check(bits(data, dtype), want_bits(theirs(ref, n, dtype), dtype), name + ' out=data')


def test_refusals_leave_the_stream_and_out(mx):
    ref = start(mx, 77)
    gpu = mx.gpu(0)
    o = mx.nd.array(np.arange(10, dtype=np.float32), gpu)
    oi = mx.nd.array(np.arange(10, dtype=np.int32), gpu, dtype='int32')
    before, before_i = o.asnumpy().copy(), oi.asnumpy().copy()
    rsp = mx.nd.sparse.zeros('row_sparse', (10, 3), gpu)
    calls = [
        (lambda: mx.random.uniform(2, 1, out=o), 'low must be less or equal to high'),
        (lambda: mx.random.uniform(0, float('nan'), out=o), 'low must be less or equal to high'),
        (lambda: mx.random.exponential(-2, out=o), 'lambda parameter in exponential'),
        (lambda: mx.random.exponential(float('nan'), out=o), 'lambda parameter in exponential'),
        (lambda: mx.random.gamma(0, 1, out=o), 'alpha parameter in gamma'),
        (lambda: mx.random.gamma(1, 0, out=o), 'beta parameter in gamma'),
        (lambda: mx.random.gamma(float('nan'), 1, out=o), 'alpha parameter in gamma'),
        (lambda: mx.random.randint(4, 3, out=oi), 'low must be less or equal to high'),
        (lambda: mx.random.randint(4, 4, out=oi), 'high must be greater than low'),
        (lambda: mx.random.randint(0, 4, out=o), 'int32 and int64 outputs only'),
        (lambda: mx.random.uniform(0, 1, out=oi), 'float16, bfloat16, float32 and float64 outputs only'),
        (lambda: mx.random.uniform(0, 1, dtype='float64', out=o), 'differs from dtype'),
        (lambda: mx.random.randint(0, 4, dtype='int64', out=oi), 'differs from dtype'),
        (lambda: mx.random.gamma(1, 1, shape=(11,), out=o), 'wrong shape'),
        (lambda: mx.random.uniform(0, 1, shape=(10,), ctx=mx.cpu(0)), 'GPU only'),
        (lambda: mx.random.exponential(1, shape=(10,), ctx=gpu, foo=1), "Cannot find argument 'foo'"),
        (lambda: mx.random.uniform(0, 1, out=rsp), 'dense'),
        (lambda: mx.nd.random.uniform_like(rsp), 'dense'),
        (lambda: mx.nd.random.gamma_like(o, out=mx.nd.zeros((11,), gpu)), 'wrong shape'),
        (lambda: mx.nd.random.normal_like(o, out=mx.nd.zeros((10,), gpu, dtype='float16')), 'differs'),
        (lambda: mx.nd.random.exponential_like(oi), 'float16, bfloat16, float32 and float64 outputs only'),
        (lambda: mx.nd.random.normal_like(o, scale=0), 'scale parameter in gaussian'),
        (lambda: mx.nd.random.uniform_like(o, shape=(2,)), "Cannot find argument 'shape'"),
        (lambda: mx.nd.random.uniform_like(mx.nd.zeros((10,), mx.cpu(0))), 'GPU only'),
    ]
    for call, match in calls:
        with pytest.raises(mx.MXNetError, match=match):
            call()
    assert np.array_equal(o.asnumpy(), before) and np.array_equal(oi.asnumpy(), before_i)
    got = mx.random.uniform(0, 1, out=o)
    check(bits(got, 'float32'), want_bits(ref.uniform(10, 0.0, 1.0, 'float32'), 'float32'), 'after refusals')
    for c in range(GR.COPIES):
        assert np.array_equal(lib_states(mx, c), ref.copies[c]), 'copy %d states differ' % c


def test_statistics(mx):
    from scipy import stats
    mx.random.seed(1)
    n = 1_000_000
    gpu = mx.gpu(0)

    def sample(fn):
        x = fn().asnumpy().astype(np.float64)
        assert math.isfinite(x.sum())
        return x
    x = sample(lambda: mx.random.uniform(-2, 3, shape=(n,), ctx=gpu))
    assert x.min() >= -2 and x.max() < 3
    assert abs(x.mean() - 0.5) < 0.01 and abs(x.var() / (25 / 12) - 1) < 0.01
    assert stats.kstest(x, 'uniform', args=(-2, 5)).pvalue > 1e-4
    x = sample(lambda: mx.random.exponential(2.0, shape=(n,), ctx=gpu))
    assert abs(x.mean() / 2 - 1) < 0.01 and abs(x.var() / 4 - 1) < 0.02
    assert stats.kstest(x, 'expon', args=(0, 2.0)).pvalue > 1e-4
    for alpha, beta in ((0.5, 2.0), (1.0, 1.0), (9.0, 0.5)):
        x = sample(lambda: mx.random.gamma(alpha, beta, shape=(n,), ctx=gpu))
        assert abs(x.mean() / (alpha * beta) - 1) < 0.01
        assert abs(x.var() / (alpha * beta * beta) - 1) < 0.02
        assert stats.kstest(x, 'gamma', args=(alpha, 0, beta)).pvalue > 1e-4
    x = sample(lambda: mx.random.randint(-3, 7, shape=(n,), ctx=gpu))
    counts = np.bincount((x + 3).astype(np.int64), minlength=10)
    assert len(counts) == 10 and stats.chisquare(counts).pvalue > 1e-4
