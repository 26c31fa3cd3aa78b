"""The uniform, exponential, gamma and randint samplers and the _like forms without a GPU: the oracle
recipe builds and exports the reference's samplers, the eight operators are registered as the rows
of sample_ops.cc, every sample_kernel instantiation compiles for sm_90a with no spills and no stack
frame, the Python functions map their arguments as the reference's ndarray/random.py does, and
refusals come before any generator exists."""
import ctypes
import os
import re
import subprocess

import pytest

import golden_sample as GS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "anand_mxnet_b200", "csrc")
OPS = [("_random_uniform", "RandomSample"), ("_random_exponential", "RandomSample"),
       ("_random_gamma", "RandomSample"), ("_random_randint", "RandomSample"),
       ("_random_uniform_like", "RandomSampleLike"), ("_random_normal_like", "RandomSampleLike"),
       ("_random_exponential_like", "RandomSampleLike"), ("_random_gamma_like", "RandomSampleLike")]


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


@pytest.mark.skipif(not os.path.isfile("/root/reference/src/common/random_generator.cu"),
                    reason="needs the reference's sources")
def test_recipe_builds_and_exports_the_samplers():
    GS.build()
    lib = ctypes.CDLL(GS.LIB)
    for name in ("uniform", "exponential", "gamma", "randint", "time"):
        assert hasattr(lib, "mxref_sample_" + name), name


def test_operators_registered(mx):
    for name, _ in OPS:
        h = ctypes.c_void_p()
        assert mx.base._LIB.NNGetOpHandle(name.encode(), ctypes.byref(h)) == 0 and h.value, name
    with open(os.path.join(CSRC, "sample_ops.cc")) as f:
        rows = re.findall(r'\{"([^"]+)",\s*(\w+),', f.read())
    assert rows == OPS
    for name in ("uniform", "normal", "randn", "exponential", "gamma", "randint"):
        assert getattr(mx.nd.random, name) is getattr(mx.random, name)
    for name in ("uniform_like", "normal_like", "exponential_like", "gamma_like"):
        assert callable(getattr(mx.nd.random, name))
    with pytest.raises(AttributeError):
        mx.nd.random.poisson


def test_ptxas_no_spills(tmp_path):
    """sample_kernel: uniform, exponential and gamma at four dtypes, randint at int32 and int64"""
    from anand_mxnet_b200 import build as B
    src = os.path.join(B.CSRC, "random_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.flags_for("random_kernels.cu") +
                       ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "r.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    blocks = re.split(r"Compiling entry function ", r.stderr)[1:]
    found = [(b.split("'")[1],) + re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, "
                                            r"(\d+) bytes spill loads", b).groups()
             for b in blocks if re.match(r"'\w*sample_kernel", b)]
    assert len(found) == 14, r.stderr[-4000:]
    assert all(f == s == l == '0' for _, f, s, l in found), found


def _captured(mx, monkeypatch):
    calls = []

    def fake(op, inputs, out=None, **kwargs):
        calls.append((op, len(inputs), out, kwargs))
    monkeypatch.setattr(mx.random, "_invoke", fake)
    return calls


def test_python_argument_mapping(mx, monkeypatch):
    calls = _captured(mx, monkeypatch)
    ctx = mx.gpu(0)
    mx.random.exponential(4, shape=(3,), ctx=ctx)
    mx.random.exponential(scale=0.5, shape=2, ctx=ctx, dtype='float16')
    mx.random.randint(-5, 7, shape=(2, 2), ctx=ctx)
    mx.random.uniform(ctx=ctx)
    mx.random.gamma(2, 3, shape=(4,), ctx=ctx, dtype='bfloat16')
    mx.random.randn(2, 3, loc=1, ctx=ctx)
    got = [(op, kw) for op, _, _, kw in calls]
    assert got[0] == ('_random_exponential', {'lam': 0.25, 'shape': (3,), 'ctx': ctx})
    assert got[1] == ('_random_exponential', {'lam': 2.0, 'shape': (2,), 'dtype': 'float16', 'ctx': ctx})
    # no dtype: the operator's default, int32
    assert got[2] == ('_random_randint', {'low': -5, 'high': 7, 'shape': (2, 2), 'ctx': ctx})
    assert got[3] == ('_random_uniform', {'low': 0, 'high': 1, 'shape': (1,), 'ctx': ctx})
    assert got[4] == ('_random_gamma', {'alpha': 2, 'beta': 3, 'shape': (4,), 'dtype': 'bfloat16', 'ctx': ctx})
    assert got[5][0] == '_random_normal'


def test_like_argument_mapping(mx, monkeypatch):
    calls = _captured(mx, monkeypatch)
    data = object()
    mx.nd.random.uniform_like(data, 1, 2)
    mx.nd.random.normal_like(data, scale=3)
    mx.nd.random.exponential_like(data, lam=5)
    mx.nd.random.gamma_like(data, alpha=0.5, out=data)
    assert [(op, n, kw) for op, n, _, kw in calls] == [
        ('_random_uniform_like', 1, {'low': 1, 'high': 2}),
        ('_random_normal_like', 1, {'loc': 0, 'scale': 3}),
        ('_random_exponential_like', 1, {'lam': 5}),
        ('_random_gamma_like', 1, {'alpha': 0.5, 'beta': 1})]
    assert calls[3][2] is data


def test_refused_without_gpu_work(mx):
    """each refusal comes before any generator or device is touched: on a machine without a GPU
    they all raise their own message rather than the missing device's"""
    gpu, cpu = mx.gpu(0), mx.cpu(0)
    calls = [
        (lambda: mx.random.uniform(0, 1, shape=(4,), ctx=cpu), 'GPU only'),
        (lambda: mx.random.exponential(1, shape=(4,), ctx=cpu), 'GPU only'),
        (lambda: mx.random.gamma(1, 1, shape=(4,), ctx=cpu), 'GPU only'),
        (lambda: mx.random.randint(0, 5, shape=(4,), ctx=cpu), 'GPU only'),
        (lambda: mx.random.uniform(2, 1, shape=(4,), ctx=gpu), 'low must be less or equal to high'),
        (lambda: mx.random.uniform(0, float('nan'), shape=(4,), ctx=gpu), 'low must be less or equal to high'),
        (lambda: mx.random.randint(5, 4, shape=(4,), ctx=gpu), 'low must be less or equal to high'),
        (lambda: mx.random.randint(5, 5, shape=(4,), ctx=gpu), 'high must be greater than low'),
        (lambda: mx.random.randint(-2 ** 63, 2 ** 63 - 1, shape=(4,), ctx=gpu), 'fit in int64'),
        (lambda: mx.random.exponential(-1, shape=(4,), ctx=gpu), 'lambda parameter in exponential'),
        (lambda: mx.random.gamma(0, 1, shape=(4,), ctx=gpu), 'alpha parameter in gamma'),
        (lambda: mx.random.gamma(1, -2, shape=(4,), ctx=gpu), 'beta parameter in gamma'),
        (lambda: mx.random.gamma(1, float('nan'), shape=(4,), ctx=gpu), 'beta parameter in gamma'),
        (lambda: mx.random.uniform(0, 1, shape=(4,), dtype='int32', ctx=gpu), 'Invalid Input'),
        (lambda: mx.random.randint(0, 5, shape=(4,), dtype='float32', ctx=gpu),
         r"valid values are: \{'None', 'int32', 'int64'\}"),
        (lambda: mx.random.uniform(0, 1, shape=(4,), ctx=gpu, foo=1), "Cannot find argument 'foo'"),
        (lambda: mx.random.randint(0, 5, shape=(4,), ctx=gpu, loc=1), "Cannot find argument 'loc'"),
        (lambda: mx.random.uniform(0, 1, ctx=gpu, out=None, shape=()), 'shape is required'),
    ]
    for call, match in calls:
        with pytest.raises(mx.MXNetError, match=match):
            call()
    with pytest.raises(mx.MXNetError, match="Required parameter high"):
        mx.random._invoke('_random_randint', [], low=0, shape=(2,), ctx=gpu)
    with pytest.raises(ValueError, match="NDArray parameters"):
        mx.random.gamma(mx.nd.NDArray.__new__(mx.nd.NDArray), 1)
