"""TEST INFRASTRUCTURE ONLY -- the reference's own Adamax, Nadam and AdaDelta optimizer classes
(python/mxnet/optimizer/optimizer.py:1768-1825, 1904-2029, loaded unmodified by oracle/ref_python.py)
running over the reference's own arithmetic. Their `update` composes NDArray arithmetic, so the
stand-in NDArray here lowers every operator as the reference's ndarray.py does (`_ufunc_helper`,
`__iadd__` / `__isub__` / `__imul__` / `__itruediv__`) and runs it in oracle/_ref/libmxref_arith.so
(golden_arith_ops.ref(): the compiled functors, the _*_scalar parsers and ClipParam):

    nd + nd, nd += nd    broadcast_add        nd + s     _plus_scalar
    nd - nd, nd -= nd    broadcast_sub        nd - s     _minus_scalar
    nd * nd, nd *= nd    broadcast_mul        nd * s, s * nd, nd *= s    _mul_scalar
    nd / nd, nd /= nd    broadcast_div        nd / s, nd /= s            _div_scalar
    maximum(nd, nd)      broadcast_maximum    abs(nd)    abs      sqrt(nd)    sqrt
    clip(nd, lo, hi)     clip(a_min=str(lo), a_max=str(hi))

`x[:]` is a view of x's buffer, and an in-place operator writes that buffer, so `x[:] op= y` updates x.
fp32 -> fp16 `cast` is oracle/ref_python_update.py's (half_t's round to nearest even).

Writes tests/golden/updater_trajectories_arith.npz, the weights after each of 4 steps and, for
AdaDelta (whose `grad *= rescale_grad` writes the caller's gradient), the gradient after each step:

    make -f oracle/arith_ops.mk && python oracle/ref_python_arith.py
"""
import contextlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import golden_arith_ops as GA  # noqa: E402
import ref_python as RP  # noqa: E402
import ref_python_update as RPU  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
CLASSES = ('Adamax', 'Nadam', 'AdaDelta')


def available():
    return RP.available() and GA.ref() is not None


def _dt(a):
    return np.dtype(a.dtype).name


def _scalar(s):
    """a Python scalar as the generated front-end formats it: str(float(s))"""
    return str(float(s))


class NDArray(RP.NDArray):
    """RP.NDArray whose arithmetic is the reference's operators"""

    def _new(self, a):
        return NDArray(np.ascontiguousarray(a).reshape(self.a.shape), self.context)

    def _put(self, a):
        self.a[...] = a.reshape(self.a.shape)
        return self

    def __getitem__(self, key):
        return NDArray(self.a[key], self.context)

    def astype(self, dtype, copy=True):
        return NDArray(self.a.astype(np.dtype(dtype)), self.context)

    def copy(self):
        return NDArray(self.a.copy(), self.context)

    def _apply(self, other, op, scalar_op):
        r, dt = GA.ref(), _dt(self.a)
        if isinstance(other, RP.NDArray):
            assert other.a.shape == self.a.shape and other.a.dtype == self.a.dtype
            RP.LOG.append((op, {}))
            return r.array_op(op, self.a, other.a, dt)
        RP.LOG.append((scalar_op, {'scalar': _scalar(other)}))
        if scalar_op == '_div_scalar':
            return r.div_scalar(self.a, _scalar(other), dt)[1]
        return r.binary_scalar({'_plus_scalar': 'plus', '_minus_scalar': 'minus',
                                '_mul_scalar': 'mul'}[scalar_op], self.a, _scalar(other), dt)

    def __add__(self, other):
        return self._new(self._apply(other, 'broadcast_add', '_plus_scalar'))

    __radd__ = __add__

    def __sub__(self, other):
        return self._new(self._apply(other, 'broadcast_sub', '_minus_scalar'))

    def __mul__(self, other):
        return self._new(self._apply(other, 'broadcast_mul', '_mul_scalar'))

    __rmul__ = __mul__

    def __truediv__(self, other):
        return self._new(self._apply(other, 'broadcast_div', '_div_scalar'))

    def __iadd__(self, other):
        return self._put(self._apply(other, 'broadcast_add', '_plus_scalar'))

    def __isub__(self, other):
        return self._put(self._apply(other, 'broadcast_sub', '_minus_scalar'))

    def __imul__(self, other):
        return self._put(self._apply(other, 'broadcast_mul', '_mul_scalar'))

    def __itruediv__(self, other):
        return self._put(self._apply(other, 'broadcast_div', '_div_scalar'))


def zeros(shape, ctx=None, dtype=None, stype=None, **_):
    assert stype in (None, 'default')
    return NDArray(np.zeros(shape, np.float32 if dtype is None else np.dtype(dtype)), ctx)


def clip(data, a_min, a_max, out=None):
    RP.LOG.append(('clip', {'a_min': str(a_min), 'a_max': str(a_max)}))
    res = GA.ref().clip(data.a, str(a_min), str(a_max), _dt(data.a))[1]
    return data._new(res) if out is None else out._put(res)


def maximum(lhs, rhs):
    return lhs._new(lhs._apply(rhs, 'broadcast_maximum', None))


def absolute(data, out=None):
    RP.LOG.append(('abs', {}))
    res = GA.ref().abs(data.a, _dt(data.a))
    return data._new(res) if out is None else out._put(res)


def sqrt(data, out=None):
    RP.LOG.append(('sqrt', {}))
    res = GA.ref().sqrt(data.a, _dt(data.a))
    return data._new(res) if out is None else out._put(res)


def op_table():
    """the names the reference's optimizer module imports for these optimizers"""
    return dict(NDArray=NDArray, zeros=zeros, clip=clip, maximum=maximum, NDabs=absolute, abs=absolute,
                sqrt=sqrt, cast=RPU.cast)


@contextlib.contextmanager
def reference_python_arith():
    """with reference_python_arith() as (opt, sched): ref_python.reference_python() with the
    stand-in NDArray's arithmetic and the operator functions above bound in the optimizer module"""
    assert available(), "needs /root/reference, oracle/_ref/libmxref.so and libmxref_arith.so"
    with RP.reference_python() as (opt, sched):
        nd = sys.modules['mxnet.ndarray']
        for k, f in op_table().items():
            setattr(nd, k, f)
            setattr(opt, k, f)          # optimizer.py bound them at import (from ..ndarray import ...)
        yield opt, sched


def trajectory_cases():
    """4 steps per case through one updater, keys in order (Nadam's m_schedule is optimizer-wide
    and advances once per key update). Gradients are kept as two halves per key (the store's two
    pushed values); g/2 + g/2 == g exactly, so the merged gradient is `grads` in either order."""
    rng = np.random.default_rng(0xB200 + 11)
    shapes = [(4, 4), (40, 25), (1027,), (3,)]

    def plan(dtype=np.float32):
        w0 = [rng.uniform(-1, 1, s).astype(np.float32).astype(dtype) for s in shapes]
        grads = []
        for _ in range(4):
            gs = []
            for s in shapes:
                g = rng.uniform(-1, 1, s).astype(dtype)
                g[np.abs(g) < 2.0 ** -12] = dtype(0.5)          # halves stay exact in float16
                assert np.array_equal(g, (g / dtype(2)) * dtype(2))
                gs.append(g)
            grads.append(gs)
        return dict(shapes=shapes, w0=w0, grads=grads, dtype=np.dtype(dtype).name)
    c = {}
    c['adamax'] = dict(plan(), opt=('Adamax', dict(wd=1e-4, rescale_grad=0.5)))
    c['adamax_clip'] = dict(plan(), opt=('Adamax', dict(learning_rate=0.01, clip_gradient=0.5)))
    c['adamax_mp_fp16'] = dict(plan(np.float16), opt=('Adamax', dict(wd=1e-4, rescale_grad=1 / 64,
                                                                     multi_precision=True)))
    c['nadam'] = dict(plan(), opt=('Nadam', dict(wd=1e-4, rescale_grad=0.5)))
    c['nadam_clip'] = dict(plan(), opt=('Nadam', dict(learning_rate=0.01, clip_gradient=0.5)))
    c['nadam_clip0'] = dict(plan(), opt=('Nadam', dict(clip_gradient=0.0, wd=1e-3)))
    c['nadam_mp_fp16'] = dict(plan(np.float16), opt=('Nadam', dict(learning_rate=0.01, rescale_grad=1 / 64,
                                                                   multi_precision=True)))
    c['adadelta'] = dict(plan(), opt=('AdaDelta', dict(wd=1e-4, rescale_grad=0.5)))
    c['adadelta_clip'] = dict(plan(), opt=('AdaDelta', dict(rho=0.95, epsilon=1e-6, clip_gradient=0.3)))
    c['adadelta_clip0'] = dict(plan(), opt=('AdaDelta', dict(clip_gradient=0, wd=1e-3, rescale_grad=2.0)))
    c['adadelta_mp_fp16'] = dict(plan(np.float16), opt=('AdaDelta', dict(wd=1e-4, rescale_grad=1 / 64,
                                                                         multi_precision=True)))
    return c


def run_trajectory(opt_mod, case, ndarray=NDArray):
    """(weights, gradients) after every step: [step][key], through opt_mod's own Updater"""
    name, kw = case['opt']
    upd = opt_mod.get_updater(getattr(opt_mod, name)(**kw))
    ws = [ndarray(w.copy()) for w in case['w0']]
    w_out, g_out = [], []
    for gs in case['grads']:
        gnd = [ndarray(g.copy()) for g in gs]
        for k, g in enumerate(gnd):
            upd(k, g, ws[k])
        w_out.append([w.a.copy() for w in ws])
        g_out.append([g.a.copy() for g in gnd])
    return w_out, g_out


def gen_trajectories():
    d = {}
    with reference_python_arith() as (opt, _):
        for name, case in trajectory_cases().items():
            ws, gs = run_trajectory(opt, case)
            for step in range(len(ws)):
                for k, w in enumerate(ws[step]):
                    assert not np.any(np.isnan(w)), (name, step, k)
                    d["%s_step%d_w%d" % (name, step, k)] = w
                    if case['opt'][0] == 'AdaDelta':
                        d["%s_step%d_g%d" % (name, step, k)] = gs[step][k]
    np.savez_compressed(os.path.join(GOLD, "updater_trajectories_arith.npz"), **d)
    return d


if __name__ == "__main__":
    GA.build()
    print("wrote", len(gen_trajectories()), "arrays")
