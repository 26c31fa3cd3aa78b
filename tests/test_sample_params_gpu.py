"""_sample_uniform, _sample_normal, _sample_gamma and _sample_exponential (NDArray parameters) on the
GPU, bit for bit against the reference's own multi-sample samplers
(oracle/_ref/libmxref_sample_params_gpu.so, built by oracle/sample_params_gpu.mk;
oracle/golden_sample_params.py draws them from the same 4 generator copies as the scalar samplers):

- every distribution x parameter dtype x output dtype, at nParm = 1, nBatch = 1, and nBatch 3, 7
  and 129, with N on both sides of 64 and of 64 * 32768; all 4 copies' states afterwards;
- unaligned parameter and out slices, and out equal to a parameter array;
- gamma at alpha 0 and -0.5, which end in the reference;
- a mixed scalar / array sequence across the round robin, and a reseed;
- gamma parameters whose draw cannot end (NaN, +-inf, -1) give NaN there, and every other thread's
  elements of that call are the reference's (they are never passed to the reference);
- _rdiv_scalar against the reference's functor, and exponential(scale=NDArray);
- refusals that need arrays leave out and the stream alone."""
import ctypes

import numpy as np
import pytest

import golden_random as GR
import golden_sample_params as GP
import kvoracle as K

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not GP.available(),
                                 reason="needs oracle/_ref/libmxref_sample_params_gpu.so and the sampler oracles")]
DTYPES = ['float16', 'float32', 'float64']
BITS = {'float16': np.uint16, 'float32': np.uint32, 'float64': np.uint64}
# (nParm, shape): N = nParm * prod(shape)
LAYOUTS = [(1, (63,)), (1, (65,)), (65, ()), (21, (3,)), (10, (7,)), (3, (129,)), (64, (1,)),
           (64 * 32768 - 1, ()), (299593, (7,)), (16257, (129,)), (1, (64 * 32768 + 1,))]


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def bits(x, dtype):
    x = x.asnumpy() if hasattr(x, 'asnumpy') else np.ascontiguousarray(x)
    return x.view(BITS[dtype]).ravel()


def check(got, want, what):
    if np.array_equal(got, want):
        return
    bad = np.nonzero(got != want)[0] if got.shape == want.shape else []
    pytest.fail('%s: %d of %d elements differ, first at %s' % (what, len(bad), want.size, bad[:6]))


def start(mx, seed):
    mx.random.seed(seed)
    return GP.ParamGenerators(0, seed)


def lib_states(mx, copy):
    buf = np.zeros(GR.NUM_STATES * GR.STATE_BYTES, np.uint8)
    mx.base.check_call(mx.base._LIB.B200KVRandomStates(0, copy, buf.ctypes.data_as(ctypes.c_void_p),
                                                        ctypes.c_size_t(buf.size)))
    return buf


def check_states(mx, ref, skip=()):
    for c in range(GR.COPIES):
        if c not in skip:
            assert np.array_equal(lib_states(mx, c), ref.copies[c]), 'copy %d states differ' % c


def params(dist, nparm, ptype, seed):
    """parameter arrays of one distribution: uniform (low, high), normal (mu, sigma), gamma (alpha
    mixing < 1 and >= 1, beta), exponential (lam, None)"""
    rng = np.random.default_rng(seed)
    if dist == 'uniform':
        lo = rng.uniform(-2, 1, nparm)
        return lo.astype(ptype), (lo + rng.uniform(0, 3, nparm)).astype(ptype)
    if dist == 'normal':
        return rng.uniform(-1, 1, nparm).astype(ptype), rng.uniform(0.1, 2, nparm).astype(ptype)
    if dist == 'gamma':
        return rng.uniform(0.2, 3, nparm).astype(ptype), rng.uniform(0.5, 2, nparm).astype(ptype)
    return rng.uniform(0.2, 5, nparm).astype(ptype), None


def draw(mx, dist, a, b, shape, otype=None, out=None):
    fn = getattr(mx.nd, 'sample_' + dist)
    kw = {'shape': shape}
    if otype is not None:
        kw['dtype'] = otype
    args = [a] if b is None else [a, b]
    return fn(*args, out=out, **kw)


@pytest.mark.parametrize("dist", ['uniform', 'normal', 'gamma', 'exponential'])
@pytest.mark.parametrize("ptype", DTYPES)
@pytest.mark.parametrize("otype", DTYPES)
def test_every_dtype_and_layout(mx, dist, ptype, otype):
    ref = start(mx, 1234)
    gpu = mx.gpu(0)
    for k, (nparm, shape) in enumerate(LAYOUTS):
        a, b = params(dist, nparm, ptype, k)
        na = mx.nd.array(a, gpu, dtype=ptype)
        nb = None if b is None else mx.nd.array(b, gpu, dtype=ptype)
        got = draw(mx, dist, na, nb, shape, otype)
        assert got.shape == (nparm,) + shape and got.dtype == np.dtype(otype)
        n = nparm * int(np.prod(shape))
        check(bits(got, otype), bits(ref.multisample(dist, a, b, n, otype), otype),
              '%s %s->%s nparm=%d shape=%s' % (dist, ptype, otype, nparm, shape))
    check_states(mx, ref)


@pytest.mark.parametrize("dist,ptype,otype", [('uniform', 'float16', 'float32'), ('normal', 'float32', 'float16'),
                                              ('gamma', 'float64', 'float32'), ('exponential', 'float32', 'float64')])
@pytest.mark.parametrize("nparm,shape", [(4099, ()), (37, (129,)), (64 * 32768 + 3, ())])
def test_unaligned_slices(mx, dist, ptype, otype, nparm, shape):
    """parameters a[1:] and out o[1:]: o[0] stays, the rest is the stream"""
    ref = start(mx, 8)
    gpu = mx.gpu(0)
    a, b = params(dist, nparm + 1, ptype, 3)
    na = mx.nd.array(a, gpu, dtype=ptype)[1:]
    nb = None if b is None else mx.nd.array(b, gpu, dtype=ptype)[1:]
    o = mx.nd.zeros((nparm + 1,) + shape, gpu, dtype=otype)
    o[:] = 5
    draw(mx, dist, na, nb, shape, out=o[1:])
    got = bits(o, otype)
    per = int(np.prod(shape))
    assert np.all(got[:per] == bits(np.full(per, 5, otype), otype))
    want = ref.multisample(dist, a[1:], None if b is None else b[1:], nparm * per, otype)
    check(got[per:], bits(want, otype), 'slice %s' % dist)
    check_states(mx, ref)


@pytest.mark.parametrize("dist", ['uniform', 'normal', 'gamma', 'exponential'])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nparm", [100, 4097, 64 * 32768 + 1])
def test_out_is_a_parameter(mx, dist, dtype, nparm):
    ref = start(mx, 31)
    gpu = mx.gpu(0)
    a, b = params(dist, nparm, dtype, 5)
    na = mx.nd.array(a, gpu, dtype=dtype)
    nb = None if b is None else mx.nd.array(b, gpu, dtype=dtype)
    target = nb if nb is not None else na
    draw(mx, dist, na, nb, (), out=target)
    check(bits(target, dtype), bits(ref.multisample(dist, a, b, nparm, dtype), dtype), 'out=param %s' % dist)


@pytest.mark.parametrize("ptype", DTYPES)
@pytest.mark.parametrize("otype", DTYPES)
def test_gamma_alpha_zero_and_negative_half(mx, ptype, otype):
    ref = start(mx, 5)
    gpu = mx.gpu(0)
    a = np.array([0.0, -0.5, 0.5, -0.0, 2.0], ptype)
    b = np.array([1.0, 2.0, 1.0, 3.0, 0.5], ptype)
    got = mx.nd.sample_gamma(mx.nd.array(a, gpu, dtype=ptype), mx.nd.array(b, gpu, dtype=ptype),
                             shape=(50,), dtype=otype)
    check(bits(got, otype), bits(ref.multisample('gamma', a, b, 250, otype), otype), 'gamma alpha 0 / -0.5')
    check_states(mx, ref)


def test_mixed_scalar_and_array_sequence_and_reseed(mx):
    ref = start(mx, 2026)
    gpu = mx.gpu(0)
    f32 = lambda x: float(K.dmlc_stof(str(x)))  # noqa: E731
    mu, sg = params('normal', 333, 'float32', 1)
    al, be = params('gamma', 129, 'float64', 2)
    lo, hi = params('uniform', 64, 'float16', 3)
    nmu, nsg = mx.nd.array(mu, gpu), mx.nd.array(sg, gpu)
    nal, nbe = mx.nd.array(al, gpu, dtype='float64'), mx.nd.array(be, gpu, dtype='float64')
    nlo, nhi = mx.nd.array(lo, gpu, dtype='float16'), mx.nd.array(hi, gpu, dtype='float16')
    calls = [
        ('float32', lambda: mx.random.normal(0.5, 1.5, shape=(1001,), ctx=gpu),
         lambda: ref.normal(1001, 0.5, 1.5, 'float32')),
        ('float32', lambda: mx.random.normal(nmu, nsg, shape=(3,)),
         lambda: ref.multisample('normal', mu, sg, 999, 'float32')),
        ('float64', lambda: mx.random.gamma(nal, nbe, shape=(7,), dtype='float64'),
         lambda: ref.multisample('gamma', al, be, 903, 'float64')),
        ('float32', lambda: mx.random.uniform(-1, 1, shape=(64 * 32768 + 1,), ctx=gpu),
         lambda: ref.uniform(64 * 32768 + 1, -1.0, 1.0, 'float32')),
        ('float16', lambda: mx.random.uniform(nlo, nhi, shape=(65,), dtype='float16'),
         lambda: ref.multisample('uniform', lo, hi, 64 * 65, 'float16')),
        ('float32', lambda: mx.random.gamma(0.3, 2, shape=(777,), ctx=gpu),
         lambda: ref.gamma(777, f32(0.3), 2.0, 'float32')),
        ('float32', lambda: mx.random.randn(5, loc=nmu, scale=nsg),
         lambda: ref.multisample('normal', mu, sg, 333 * 5, 'float32')),
    ]
    for k in range(len(calls)):
        dtype, mine, theirs = calls[k]
        check(bits(mine(), dtype), bits(theirs(), dtype), 'call %d' % k)
    check_states(mx, ref)
    mx.random.seed(77)
    ref.seed_all(77)
    for k in (1, 0, 2, 4):
        dtype, mine, theirs = calls[k]
        check(bits(mine(), dtype), bits(theirs(), dtype), 'after reseed, call %d' % k)
    check_states(mx, ref)


@pytest.mark.parametrize("ptype", DTYPES)
@pytest.mark.parametrize("otype", DTYPES)
def test_gamma_that_cannot_end_is_nan(mx, ptype, otype):
    """N = 200: 4 threads of 50 elements. Thread 1 meets alphas NaN, +inf, -inf and -1 at elements
    60, 70, 80 and 90: those are NaN, and its run differs from the reference's from element 60 on
    (the reference never returns there). Threads 0, 2 and 3, and elements 50..59, are the
    reference's, computed with those four alphas replaced by 1.5."""
    ref = start(mx, 6)
    gpu = mx.gpu(0)
    a, b = params('gamma', 200, ptype, 9)
    bad = {60: np.nan, 70: np.inf, 80: -np.inf, 90: -1.0}
    for i, v in bad.items():
        a[i] = v
    got = bits(mx.nd.sample_gamma(mx.nd.array(a, gpu, dtype=ptype), mx.nd.array(b, gpu, dtype=ptype),
                                  dtype=otype), otype)
    safe = a.copy()
    for i in bad:
        safe[i] = 1.5
    want = bits(ref.multisample('gamma', safe, b, 200, otype), otype)
    keep = np.r_[0:60, 100:200]
    check(got[keep], want[keep], 'other threads')
    vals = got.view(np.dtype(otype))
    assert all(np.isnan(vals[i]) for i in bad), vals[list(bad)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("scalar", ['1.0', '2.5', '-3', '0.1'])
def test_rdiv_scalar(mx, dtype, scalar):
    rng = np.random.default_rng(4)
    x = np.concatenate([rng.uniform(-4, 4, 4099), [0.0, -0.0, np.inf, -np.inf, 1e-30]]).astype(dtype)
    parsed, want = GP.rdiv_scalar(x, scalar)
    gpu = mx.gpu(0)
    got = mx.nd.array(x, gpu, dtype=dtype).__rtruediv__(float(scalar))
    assert float(scalar) == parsed
    check(bits(got, dtype), bits(want, dtype), '_rdiv_scalar %s %s' % (dtype, scalar))
    got = mx.random._invoke('_rdiv_scalar', [mx.nd.array(x, gpu, dtype=dtype)], scalar=scalar)
    check(bits(got, dtype), bits(want, dtype), '_rdiv_scalar(scalar=%s)' % scalar)


def test_exponential_scale_array(mx):
    ref = start(mx, 12)
    gpu = mx.gpu(0)
    scale = np.random.default_rng(0).uniform(0.1, 4, 300).astype(np.float32)
    got = mx.random.exponential(mx.nd.array(scale, gpu), shape=(9,))
    _, lam = GP.rdiv_scalar(scale, '1.0')
    check(bits(got, 'float32'), bits(ref.multisample('exponential', lam, None, 2700, 'float32'), 'float32'),
          'exponential(scale=NDArray)')


def test_refusals_leave_the_stream_and_out(mx):
    ref = start(mx, 77)
    gpu = mx.gpu(0)
    a = mx.nd.array(np.ones(10, np.float32), gpu)
    b = mx.nd.array(np.full(10, 2, np.float32), gpu)
    big = mx.nd.array(np.arange(20, dtype=np.float32), gpu)
    o = mx.nd.array(np.arange(10, dtype=np.float32), gpu)
    before, before_big = o.asnumpy().copy(), big.asnumpy().copy()
    rsp = mx.nd.sparse.zeros('row_sparse', (10, 3), gpu)
    d = mx.nd.array(np.ones(10, np.float64), gpu, dtype='float64')
    i32 = mx.nd.array(np.ones(10, np.int32), gpu, dtype='int32')
    bf = mx.nd.zeros((10,), gpu, dtype='bfloat16')
    cpu = mx.nd.zeros((10,), mx.cpu(0))
    pinned = mx.nd.zeros((10,), mx.cpu_pinned(0))
    calls = [
        (lambda: mx.nd.sample_uniform(a, out=o), r'takes 2 inputs \(1 given\)'),
        (lambda: mx.random._invoke('_sample_exponential', [a, b]), r'takes 1 input \(2 given\)'),
        (lambda: mx.nd.sample_uniform(a, big), 'shape differs'),
        (lambda: mx.nd.sample_uniform(a, d), 'dtype float64 differs'),
        (lambda: mx.nd.sample_normal(i32, i32), 'integer and bfloat16 parameters are not supported'),
        (lambda: mx.nd.sample_normal(bf, bf), 'integer and bfloat16 parameters are not supported'),
        (lambda: mx.nd.sample_exponential(mx.nd.zeros((0,), gpu)), 'must not be empty'),
        (lambda: mx.nd.sample_uniform(a, b, out=mx.nd.zeros((11,), gpu)), 'wrong shape'),
        (lambda: mx.nd.sample_uniform(a, b, shape=(2,), out=o), 'wrong shape'),
        (lambda: mx.nd.sample_uniform(a, b, dtype='float64', out=o), 'Inferred output type does not match'),
        (lambda: mx.nd.sample_uniform(a, b, out=mx.nd.zeros((10,), gpu, dtype='int32')), 'Output type must be'),
        (lambda: mx.nd.sample_gamma(a, b, out=rsp), 'dense'),
        (lambda: mx.nd.sample_gamma(rsp, rsp), 'dense'),
        (lambda: mx.nd.sample_gamma(cpu, cpu), 'GPU only'),
        (lambda: mx.nd.sample_gamma(pinned, pinned), 'GPU only'),
        (lambda: mx.nd.sample_gamma(a, b, out=cpu), "parameters' GPU"),
        (lambda: mx.nd.sample_normal(big[0:10], b, out=big[5:15]), 'overlaps parameter 0'),
        (lambda: mx.nd.sample_normal(a, big[5:15], out=big[0:10]), 'overlaps parameter 1'),
        (lambda: mx.nd.sample_exponential(a, shape=(0,)), 'shape parameter must be non-zero'),
        (lambda: mx.nd.sample_exponential(a, foo=1), "Cannot find argument 'foo'"),
        (lambda: mx.random.gamma(float('inf'), 1, out=o), 'alpha must be finite'),
        (lambda: mx.nd.random.gamma_like(o, alpha=float('inf')), 'alpha must be finite'),
        (lambda: mx.nd.random.gamma_like(o, alpha=float('inf'), out=o), 'alpha must be finite'),
    ]
    for call, match in calls:
        with pytest.raises(mx.MXNetError, match=match):
            call()
    assert np.array_equal(o.asnumpy(), before) and np.array_equal(big.asnumpy(), before_big)
    got = mx.nd.sample_uniform(a, b, out=o)
    want = ref.multisample('uniform', np.ones(10, np.float32), np.full(10, 2, np.float32), 10, 'float32')
    check(bits(got, 'float32'), bits(want, 'float32'), 'after refusals')
    check_states(mx, ref)


def test_statistics(mx):
    """for readers, not for parity: per-parameter means at 10^5 samples"""
    gpu = mx.gpu(0)
    mx.random.seed(3)
    mu = mx.nd.array(np.array([-2, 0, 3], np.float32), gpu)
    sg = mx.nd.array(np.array([0.5, 1, 2], np.float32), gpu)
    x = mx.nd.sample_normal(mu, sg, shape=(100000,)).asnumpy()
    assert np.allclose(x.mean(axis=1), [-2, 0, 3], atol=0.03)
    assert np.allclose(x.std(axis=1), [0.5, 1, 2], rtol=0.02)
    al = mx.nd.array(np.array([0.5, 4], np.float32), gpu)
    be = mx.nd.array(np.array([2, 0.5], np.float32), gpu)
    g = mx.nd.sample_gamma(al, be, shape=(100000,)).asnumpy()
    assert np.allclose(g.mean(axis=1), [1.0, 2.0], rtol=0.03)
