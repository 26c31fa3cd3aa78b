"""clip_global_norm / multi_scale without a GPU: the operator names resolve and are listed in the C
header, the numpy restatements (oracle/golden_clip_global_norm.py) equal
tests/golden/clip_global_norm.npz and the reference's own functors live, the scalar strings parse as
std::stod-then-float (not as a direct float parse, and not as dmlc::stof), the Python wrappers
marshal one operator call and keep the reference's warning / return-type contract, the unscale mirror
makes one bulk call and raises the reference's TypeErrors, and the three kernels compile for sm_90a
without spills."""
import ctypes
import os
import re
import subprocess
import warnings
from fractions import Fraction

import numpy as np
import pytest

import golden_clip_global_norm as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
live = pytest.mark.skipif(G.ref() is None, reason="needs oracle/_ref/libmxref_clip.so")


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_operators_are_registered_and_documented():
    import anand_mxnet_b200 as mx
    header = open(os.path.join(ROOT, "include", "b200kv_c_api.h")).read()
    for name in ('_b200kv_clip_global_norm', '_b200kv_multi_scale'):
        h = ctypes.c_void_p()
        assert mx.base._LIB.NNGetOpHandle(name.encode(), ctypes.byref(h)) == 0 and h.value
        assert name in header
    assert callable(mx.gluon.utils.clip_global_norm) and callable(mx.nd.contrib.multi_scale)


# ------------------------------------------------------------------ restatement vs fixture / live
def test_scale_restatement_matches_golden(golden):
    g = golden("clip_global_norm")
    cases = G.scale_cases()
    assert eq(g['scale_norm'], np.array([n for n, _ in cases], F).view(np.uint32))
    assert list(g['scale_max_norm']) == [m for _, m in cases]
    got = np.array([G.scale_of(n, m) for n, m in cases], F)
    assert eq(got.view(np.uint32), g['scale_out'])
    # every branch is present: not clipped, clipped, denormal, zero, nan
    out = g['scale_out'].view(F)
    assert (out == 1).any() and ((out > 0) & (out < 1)).any() and (out == 0).any() and np.isnan(out).any()
    assert ((out > 0) & (out < 1.1754944e-38)).any()


@live
def test_scale_restatement_matches_live_reference():
    for n, m in G.scale_cases():
        assert eq(G.ref().scale(n, m), G.scale_of(n, m)), (n, m)


@pytest.mark.parametrize("name", sorted(G.SETS))
def test_set_restatement_matches_golden(golden, name):
    case, g = G.SETS[name], golden("clip_global_norm")
    xs = G.inputs(case, name)
    norm = G.norm_of(xs)
    assert eq(np.array([norm], F).view(np.uint32), g[name + '_norm']) or (
        np.isnan(norm) and np.isnan(g[name + '_norm'].view(F)[0]))
    for i, x in enumerate(xs):
        assert eq(G.restate(norm, case['max_norm'], x).view(np.uint32), g['%s_out%d' % (name, i)]), (name, i)


@live
@pytest.mark.parametrize("name", sorted(G.SETS))
def test_set_restatement_matches_live_reference(name):
    case, r = G.SETS[name], G.ref()
    xs = G.inputs(case, name)
    with np.errstate(all='ignore'):
        norm = r.sqrt(r.sum_sq(xs))
    assert eq(norm, G.norm_of(xs)) or (np.isnan(norm) and np.isnan(G.norm_of(xs)))
    if np.isfinite(norm):      # where the norm is inf / nan the library leaves the arrays alone
        s = r.scale(norm, case['max_norm'])
        for x in xs:
            assert eq(r.mul(x, s), G.restate(norm, case['max_norm'], x))


@pytest.mark.parametrize("name", sorted(G.SCALE_SETS))
def test_multi_scale_restatement_matches_golden_and_live(golden, name):
    case, g = G.SCALE_SETS[name], golden("clip_global_norm")
    for i, x in enumerate(G.scale_inputs(case, name)):
        want = G.multi_scale(x, case['scalar'])
        assert eq(want.view(np.uint32), g['mscale_%s_out%d' % (name, i)]), (name, i)
        if G.ref() is not None:
            assert eq(G.ref().mul_scalar(x, case['scalar']), want)


def test_fixture_holds_nothing_else(golden):
    want = {'scale_norm', 'scale_max_norm', 'scale_out'}
    for name, case in G.SETS.items():
        want |= {name + '_norm'} | {'%s_out%d' % (name, i) for i in range(len(case['sizes']))}
    for name, case in G.SCALE_SETS.items():
        want |= {'mscale_%s_out%d' % (name, i) for i in range(len(case['sizes']))}
    assert set(golden("clip_global_norm").files) == want


def test_scalar_parse_is_stod_then_one_rounding():
    tie = '1.0000000596046447753906250000000001'     # above 1 + 2^-24 by less than a double resolves
    assert G.parse_scalar(tie) == F(1.0)
    assert Fraction(tie) > 1 + Fraction(1, 2 ** 24)   # so the float32 nearest to the decimal is 1 + 2^-23
    assert G.parse_scalar('16777217') == F(16777216.0)
    assert G.parse_scalar('1e39') == F(np.inf) and G.parse_scalar('7e-46') == F(0.0)
    assert G.parse_scalar('1e-45').view(np.uint32) == 1
    # str(float) of the Python front-end round-trips the double, so 1 / 65536 arrives exactly
    assert G.parse_scalar(str(1.0 / 65536)) == F(2.0 ** -16)
    if G.ref() is not None:
        one = np.ones(1, F)
        for s in G.SCALARS:
            assert eq(G.ref().mul_scalar(one, s), np.array([G.parse_scalar(s)], F)), s
        with pytest.raises(RuntimeError):
            G.ref().mul_scalar(one, 'abc')


# ---------------------------------------------------------------------- the Python wrappers
class Stub(object):
    """stands for an NDArray: counts every host wait"""
    waits = 0

    def __init__(self, value):
        self.value = value

    def asscalar(self):
        Stub.waits += 1
        return self.value

    def asnumpy(self):
        Stub.waits += 1
        return np.array([self.value], F)

    def wait_to_read(self):
        Stub.waits += 1


@pytest.fixture
def invoked(monkeypatch):
    import anand_mxnet_b200 as mx
    calls = []

    def fake(op, inputs, out=None, **kwargs):
        calls.append((op, list(inputs), out, kwargs))
        return fake.result
    fake.result = Stub(F(5.0))
    Stub.waits = 0
    monkeypatch.setattr(mx.nd, '_invoke', fake)
    return mx, calls, fake


def test_clip_global_norm_wrapper(invoked):
    mx, calls, fake = invoked
    arrays = [Stub(0), Stub(1), Stub(2)]
    got = mx.gluon.utils.clip_global_norm(arrays, 0.25, check_isfinite=False)
    assert got is fake.result and Stub.waits == 0
    assert calls == [('_b200kv_clip_global_norm', arrays, None, dict(num_arrays=3, max_norm=0.25))]
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        got = mx.gluon.utils.clip_global_norm(arrays, 0.25)
    assert type(got) is float and got == 5.0 and Stub.waits == 1 and len(calls) == 2 and not w
    for bad in (np.nan, np.inf):
        fake.result = Stub(F(bad))
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            got = mx.gluon.utils.clip_global_norm(arrays, 1)
        assert len(w) == 1 and w[0].category is UserWarning and w[0].filename == __file__
        assert str(w[0].message) == 'nan or inf is detected. Clipping results will be undefined.'
        assert type(got) is float and not np.isfinite(got)
    with pytest.raises(AssertionError):
        mx.gluon.utils.clip_global_norm([], 1.0)


def test_multi_scale_wrapper_and_unscale_mirror(invoked):
    mx, calls, fake = invoked
    from compat import mxnet_amp_unscale as U
    from compat import mxnet_optimizer as M
    a, b, c = Stub(0), Stub(1), Stub(2)
    assert mx.nd.contrib.multi_scale(a, b, scalar=0.5) is None
    assert calls == [('_b200kv_multi_scale', [a, b], None, dict(num_arrays=2, scalar=0.5))]
    del calls[:]

    class P(object):
        def __init__(self, grad):
            self._grad = grad

    class Trainer(object):
        _params = [P([a]), P(None), P([b]), P([c])]
        _scale = 1.0 / 65536
    t = Trainer()
    U.unscale(t)
    assert calls == [('_b200kv_multi_scale', [a, b, c], None, dict(num_arrays=3, scalar=1.0 / 65536))]
    assert t._scale == 1. and Stub.waits == 0
    with pytest.raises(TypeError, match="AMP is currently only compatible with Gluon Trainer"):
        U.unscale(M.SGD(learning_rate=0.1))
    with pytest.raises(TypeError, match="optimizer_or_trainer should be a Gluon Trainer or an optimizer, instead is"):
        U.unscale(3)


def test_ptxas_no_spills(tmp_path):
    """clip_norm_partial_kernel, clip_norm_fold_kernel, clip_norm_scale_kernel"""
    from anand_mxnet_b200 import build as B
    src = os.path.join(B.CSRC, "multi_tensor_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "m.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    blocks = re.split(r"Compiling entry function ", r.stderr)[1:]   # one per kernel
    found = [(b.split("'")[1],) + re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", b).groups()
             for b in blocks if re.match(r"'\w*clip_norm_(partial|fold|scale)_kernel", b)]
    assert len(found) == 3, r.stderr[-4000:]
    assert all(s == '0' and l == '0' for _, s, l in found), found
