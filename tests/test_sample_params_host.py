"""Sampling with NDArray parameters without a GPU: the oracle recipe builds and exports the
reference's multi-sample samplers and _rdiv_scalar, the operators are registered as the rows of
sample_param_ops.cc, every param_draw_kernel instantiation compiles for sm_90a with no spills and no
stack frame, the Python functions map NDArray parameters as the reference's _random_helper does, and
the refusals that need no array come before any generator exists."""
import ctypes
import os
import re
import subprocess

import pytest

import golden_sample_params as GP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "anand_mxnet_b200", "csrc")
OPS = [("_sample_uniform", "MultiSample"), ("sample_uniform", "MultiSample"),
       ("_sample_normal", "MultiSample"), ("sample_normal", "MultiSample"),
       ("_sample_gamma", "MultiSample"), ("sample_gamma", "MultiSample"),
       ("_sample_exponential", "MultiSample"), ("sample_exponential", "MultiSample"),
       ("_rdiv_scalar", "RDivScalar")]


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


@pytest.mark.skipif(not os.path.isfile("/root/reference/src/common/random_generator.cu"),
                    reason="needs the reference's sources")
def test_recipe_builds_and_exports_the_samplers():
    GP.build()
    lib = ctypes.CDLL(GP.LIB)
    for name in ("mxref_multisample", "mxref_multisample_time"):
        assert hasattr(lib, name), name
    assert hasattr(ctypes.CDLL(GP.RDIV_LIB), "mxref_ar_rdiv_scalar")


@pytest.mark.skipif(not os.path.isfile("/root/reference/src/operator/tensor/matrix_op-inl.h"),
                    reason="needs the reference's sources")
def test_rdiv_oracle_on_the_cpu():
    import numpy as np
    GP.build()
    parsed, out = GP.rdiv_scalar(np.array([2, 4, -0.0], np.float32), "1.0")
    assert parsed == 1.0
    assert out.tolist() == [0.5, 0.25, float('-inf')]


def test_operators_registered(mx):
    for name, _ in OPS:
        h = ctypes.c_void_p()
        assert mx.base._LIB.NNGetOpHandle(name.encode(), ctypes.byref(h)) == 0 and h.value, name
    with open(os.path.join(CSRC, "sample_param_ops.cc")) as f:
        rows = re.findall(r'\{"([^"]+)",\s*(\w+),', f.read())
    assert rows == OPS
    for name in ("uniform", "normal", "gamma", "exponential"):
        assert callable(getattr(mx.nd, "sample_" + name))
    assert mx.nd.NDArray.__rdiv__ is mx.nd.NDArray.__rtruediv__


def test_ptxas_no_spills(tmp_path):
    """param_draw_kernel: 4 distributions x 3 parameter dtypes x 3 output dtypes"""
    from anand_mxnet_b200 import build as B
    src = os.path.join(B.CSRC, "random_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.flags_for("random_kernels.cu") +
                       ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "r.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    blocks = re.split(r"Compiling entry function ", r.stderr)[1:]
    found = [(b.split("'")[1],) + re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, "
                                            r"(\d+) bytes spill loads", b).groups()
             for b in blocks if re.match(r"'\w*param_draw_kernel", b)]
    assert len(found) == 36, r.stderr[-4000:]
    assert all(f == s == l == '0' for _, f, s, l in found), found


def _captured(mx, monkeypatch):
    """every _invoke of random.py and ndarray.py recorded; _rdiv_scalar answers with an NDArray"""
    calls = []
    fake_nd = mx.nd.NDArray.__new__(mx.nd.NDArray)

    def fake(op, inputs, out=None, **kwargs):
        calls.append((op, list(inputs), out, kwargs))
        return fake_nd if op == '_rdiv_scalar' else None
    monkeypatch.setattr(mx.random, "_invoke", fake)
    monkeypatch.setattr(mx.ndarray, "_invoke", fake)
    return calls, fake_nd


def _nd(mx):
    return mx.nd.NDArray.__new__(mx.nd.NDArray)


def test_python_argument_mapping(mx, monkeypatch):
    calls, lam = _captured(mx, monkeypatch)
    a, b, o = _nd(mx), _nd(mx), _nd(mx)
    mx.random.uniform(a, b)
    mx.random.normal(a, b, shape=(2, 3), dtype='float16', ctx=mx.gpu(0), out=o)
    mx.random.randn(4, loc=a, scale=b)
    mx.random.gamma(a, b, shape=5, dtype='float64')
    mx.random.exponential(a, shape=(7,))
    mx.nd.random.uniform(low=a, high=b, out=o)
    mx.random.normal(1, 2, shape=(3,), ctx=mx.gpu(0))
    assert [c[0] for c in calls] == ['_sample_uniform', '_sample_normal', '_sample_normal', '_sample_gamma',
                                     '_rdiv_scalar', '_sample_exponential', '_sample_uniform', '_random_normal']
    # shape and dtype only when given; ctx is not passed
    assert calls[0][1:] == ([a, b], None, {})
    assert calls[1][1:] == ([a, b], o, {'shape': (2, 3), 'dtype': 'float16'})
    assert calls[2][1:] == ([a, b], None, {'shape': (4,)})
    assert calls[3][1:] == ([a, b], None, {'shape': (5,), 'dtype': 'float64'})
    # exponential(scale=NDArray): lam = 1.0 / scale through NDArray.__rtruediv__
    assert calls[4][1:] == ([a], None, {'scalar': 1.0})
    assert calls[5][1:] == ([lam], None, {'shape': (7,)})
    assert calls[6][1:] == ([a, b], o, {})
    assert calls[7][3]['loc'] == 1 and calls[7][3]['scale'] == 2


def test_mixed_and_randint_arrays_refused(mx, monkeypatch):
    calls, _ = _captured(mx, monkeypatch)
    a = _nd(mx)
    for call in (lambda: mx.random.uniform(a, 1), lambda: mx.random.uniform(0, a),
                 lambda: mx.random.normal(a, 1), lambda: mx.random.randn(2, scale=a),
                 lambda: mx.random.gamma(1, a), lambda: mx.random.randint(a, a),
                 lambda: mx.random.randint(0, a)):
        with pytest.raises(ValueError, match="NDArray parameters"):
            call()
    assert calls == []


def test_refused_without_gpu_work(mx):
    """each refusal comes before any generator or device is touched: on a machine without a GPU they
    all raise their own message rather than the missing device's"""
    gpu = mx.gpu(0)
    inv = mx.random._invoke
    calls = [
        (lambda: mx.random.gamma(float('inf'), 1, shape=(4,), ctx=gpu), 'alpha must be finite'),
        (lambda: mx.random.gamma(float('-inf'), 1, shape=(4,), ctx=gpu), 'alpha parameter in gamma'),
        (lambda: inv('_sample_uniform', []), r'takes 2 inputs \(0 given\)'),
        (lambda: inv('_sample_exponential', []), r'takes 1 input \(0 given\)'),
        (lambda: inv('sample_gamma', [], shape=(2, 0)), 'shape parameter must be non-zero'),
        (lambda: inv('_sample_normal', [], dtype='bfloat16'), "Invalid Input: 'bfloat16'"),
        (lambda: inv('_sample_normal', [], dtype='int32'), 'Invalid Input'),
        (lambda: inv('_sample_uniform', [], ctx=gpu), "Cannot find argument 'ctx'"),
        (lambda: inv('_sample_exponential', [], lam=1), "Cannot find argument 'lam'"),
    ]
    for call, match in calls:
        with pytest.raises(mx.MXNetError, match=match):
            call()
