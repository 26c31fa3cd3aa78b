"""reset_arrays / zeros_like without a GPU: the operator names and Python wrappers resolve, the
tests/compat zero_grad mirror issues the same operator calls as the reference's own
ParameterDict.zero_grad (its source text, run over recording stand-ins), and reset_arrays_kernel
compiles for sm_90a without spills."""
import ast
import ctypes
import os
import re
import subprocess
from collections import OrderedDict, defaultdict

import numpy as np
import pytest

import ref_python as RP

REF_PARAMETER_PY = os.path.join(RP.REF_PY, "gluon", "parameter.py")
live_src = pytest.mark.skipif(not os.path.isfile(REF_PARAMETER_PY), reason="needs the reference's parameter.py")


def test_operators_are_registered():
    import anand_mxnet_b200 as mx
    for name in (b'reset_arrays', b'zeros_like', b'_sparse_zeros_like'):
        h = ctypes.c_void_p()
        assert mx.base._LIB.NNGetOpHandle(name, ctypes.byref(h)) == 0 and h.value, name
    assert callable(mx.nd.reset_arrays) and callable(mx.nd.zeros_like) and callable(mx.nd.sparse.zeros_like)


# ------------------------------------------------------------------ the tests/compat mirror
class Grad(object):
    def __init__(self, name, stype, ctx):
        self.name, self.stype, self.ctx = name, stype, ctx


class Param(object):
    def __init__(self, grad_req, grads):
        self.grad_req, self._grad = grad_req, grads

    def list_grad(self):
        return list(self._grad)


class Recorder(object):
    """the two operators zero_grad calls, logging (operator, arrays in order, parameters)"""

    def __init__(self):
        self.log = []

    def zeros_like(self, data, out=None):
        self.log.append(('zeros_like', [data.name], {'out': None if out is None else out.name}))

    def reset_arrays(self, *arrays, **kwargs):
        self.log.append(('reset_arrays', [a.name for a in arrays], dict(kwargs)))


def reference_zero_grad():
    """ParameterDict.zero_grad of the reference, compiled from its source text (nothing imported)"""
    tree = ast.parse(open(REF_PARAMETER_PY).read())
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == 'ParameterDict']
    assert len(cls) == 1
    fn = [f for f in cls[0].body if isinstance(f, ast.FunctionDef) and f.name == 'zero_grad']
    assert len(fn) == 1
    fn[0].decorator_list = []
    rec = Recorder()
    ns = {'defaultdict': defaultdict, 'ndarray': rec, 'is_np_array': lambda: False}
    exec(compile(ast.Module(body=fn, type_ignores=[]), REF_PARAMETER_PY, "exec"), ns)
    return ns['zero_grad'], rec


def case_params(seed):
    """parameters over two contexts: dense and row_sparse gradients, grad_req 'null', 'add' and
    'write', and initialised parameters with no gradient"""
    rng = np.random.default_rng(seed)
    ctxs = [('gpu', 0), ('gpu', 1)] if rng.random() < 0.8 else [('gpu', 0)]
    params = OrderedDict()
    for i in range(int(rng.integers(0, 40))):
        req = str(rng.choice(['write', 'add', 'add', 'null']))
        kind = rng.random()
        if kind < 0.15:
            grads = None
        else:
            stype = 'row_sparse' if kind < 0.4 else 'default'
            grads = [Grad('p%d_%s%d' % (i, c[0], c[1]), stype, c) for c in ctxs]
        params['p%d' % i] = Param(req, grads)
    return params


@live_src
@pytest.mark.parametrize("seed", range(25))
def test_zero_grad_mirror_vs_reference(seed, monkeypatch):
    from compat import mxnet_gluon_parameter as P
    ref, ref_rec = reference_zero_grad()
    params = case_params(seed)
    ref(params)
    mine = Recorder()
    monkeypatch.setattr(P, 'ndarray', mine)
    P.zero_grad(params)
    assert mine.log == ref_rec.log
    # what the calls carry: num_arrays is the count, zeros_like writes its own input
    for op, names, kw in ref_rec.log:
        if op == 'reset_arrays':
            assert kw == {'num_arrays': len(names)}
        else:
            assert kw == {'out': names[0]}


@live_src
def test_zero_grad_mirror_vs_reference_fixed_mix(monkeypatch):
    """the interleaving spelled out once: row_sparse gradients are zeroed as they are met, then one
    reset_arrays per context in the order the contexts were first seen"""
    from compat import mxnet_gluon_parameter as P
    c0, c1 = ('gpu', 0), ('gpu', 1)
    params = OrderedDict([
        ('a', Param('write', [Grad('a0', 'default', c0), Grad('a1', 'default', c1)])),
        ('e', Param('add', [Grad('e0', 'row_sparse', c0), Grad('e1', 'row_sparse', c1)])),
        ('n', Param('null', [Grad('n0', 'default', c0), Grad('n1', 'default', c1)])),
        ('u', Param('add', None)),
        ('b', Param('add', [Grad('b0', 'default', c0), Grad('b1', 'default', c1)])),
    ])
    want = [('zeros_like', ['e0'], {'out': 'e0'}), ('zeros_like', ['e1'], {'out': 'e1'}),
            ('reset_arrays', ['a0', 'b0'], {'num_arrays': 2}), ('reset_arrays', ['a1', 'b1'], {'num_arrays': 2})]
    ref, ref_rec = reference_zero_grad()
    ref(params)
    assert ref_rec.log == want
    mine = Recorder()
    monkeypatch.setattr(P, 'ndarray', mine)
    P.zero_grad(params)
    assert mine.log == want
    for empty in (OrderedDict(), OrderedDict([('n', params['n']), ('u', params['u'])])):
        mine.log[:] = []
        P.zero_grad(empty)
        assert mine.log == []


def test_ptxas_no_spills(tmp_path):
    from anand_mxnet_b200 import build as B
    src = os.path.join(B.CSRC, "multi_tensor_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "m.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    blocks = re.split(r"Compiling entry function ", r.stderr)[1:]   # one per kernel
    found = [re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", b).groups()
             for b in blocks if re.match(r"'\w*reset_arrays_kernel", b)]
    assert found == [('0', '0')], r.stderr[-4000:]
