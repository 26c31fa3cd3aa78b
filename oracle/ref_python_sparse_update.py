"""TEST INFRASTRUCTURE ONLY -- the reference's own Ftrl and AdaGrad optimizer classes
(python/mxnet/optimizer/optimizer.py, loaded unmodified by oracle/ref_python.py) training row_sparse
tables over the reference's own row_sparse kernels (golden_sparse_update_ops.ref(), i.e.
oracle/_ref/libmxref_sparse_update.so). The stand-in `mxnet.ndarray` of oracle/ref_python.py gains
a row_sparse array (`RspNDArray`), `zeros(..., stype='row_sparse')`, `ftrl_update` for row_sparse
operands and `sparse.adagrad_update`.

Writes tests/golden/updater_trajectories_sparse.npz (the reference's Python cannot travel to the GPU
machine; the fixture does): per case, key and step, the table and the optimizer states after the step.

    make -f oracle/sparse_update_ops.mk && python oracle/ref_python_sparse_update.py
"""
import contextlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import golden_sparse_update_ops as GS  # noqa: E402
import ref_python as RP  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
F = np.float32


def available():
    return RP.available() and GS.ref() is not None


class RspNDArray(RP.NDArray):
    """numpy-backed stand-in for a RowSparseNDArray: ascending ids + their rows"""
    stype = 'row_sparse'

    def __init__(self, shape, idx, vals, ctx=None):
        self._shape = tuple(shape)
        self.idx = np.asarray(idx, np.int64)
        self.vals = np.ascontiguousarray(vals, F).reshape((len(self.idx),) + self._shape[1:])
        self.context = ctx or RP.Context()

    shape = property(lambda self: self._shape)
    dtype = property(lambda self: np.float32)
    size = property(lambda self: int(np.prod(self._shape)))

    def asnumpy(self):
        d = np.zeros(self._shape, F)
        d[self.idx] = self.vals
        return d

    def copy(self):
        return RspNDArray(self._shape, self.idx.copy(), self.vals.copy(), self.context)

    def __getstate__(self):
        return {'shape': self._shape, 'idx': self.idx, 'vals': self.vals}

    def __setstate__(self, st):
        self.__init__(st['shape'], st['idx'], st['vals'])


def zeros(shape, ctx=None, dtype=None, stype=None, **kw):
    if stype == 'row_sparse':
        return RspNDArray(shape, np.zeros(0, np.int64), np.zeros((0,) + tuple(shape[1:]), F), ctx)
    return RP.zeros(shape, ctx, dtype, stype, **kw)


def call(fn, name, ins, out, params):
    """one operator call on stand-in arrays through fn (GS.ref() or GS.restate), in place"""
    w, g = ins[0], ins[1]
    rows = w.shape[0]
    row_len = int(np.prod(w.shape[1:]))
    stypes, nnr, bufs = [], [], []
    for i, a in enumerate(ins):
        rsp = isinstance(a, RspNDArray)
        stypes.append(1 if rsp else 0)
        if i == 1:
            nnr.append(len(a.idx))
            bufs.append(a.vals.reshape(len(a.idx), row_len))
        elif rsp:       # a table: all rows (ids 0..rows-1) or none
            assert len(a.idx) in (0, rows) and (len(a.idx) == 0 or np.array_equal(a.idx, np.arange(rows)))
            nnr.append(len(a.idx))
            full = np.zeros((rows, row_len), F)
            full[:len(a.idx)] = a.vals.reshape(len(a.idx), row_len)
            bufs.append(full)
        else:
            nnr.append(0)
            bufs.append(a.a.reshape(rows, row_len))
    fn(name, stypes, nnr, bufs, g.idx, rows, row_len, out is w, **params)
    for i, a in enumerate(ins):
        if i != 1 and isinstance(a, RspNDArray):
            a.idx = np.arange(nnr[i], dtype=np.int64)
            a.vals = bufs[i][:nnr[i]].reshape((nnr[i],) + a.shape[1:]).copy()
    return out


def _op(name, fn=None):
    def op(*args, **kwargs):
        out = kwargs.pop('out')
        kwargs.pop('name', None)
        RP.LOG.append((name, {k: str(v) for k, v in kwargs.items()}))
        return call(fn or GS.ref(), name, list(args), out, kwargs)
    op.__name__ = name
    return op


def op_table(fn=None):
    """the names the reference's Ftrl / AdaGrad (and the tests/compat mirror) use; fn: the kernel
    behind the operators (default: the reference's own, GS.ref())"""
    sparse = types.SimpleNamespace(adagrad_update=_op('_sparse_adagrad_update', fn),
                                   ftrl_update=_op('_sparse_ftrl_update', fn))
    return {'zeros': zeros, 'ftrl_update': _op('ftrl_update', fn), 'sparse': sparse}


@contextlib.contextmanager
def reference_python_sparse_update():
    """with reference_python_sparse_update() as (opt, sched): ref_python.reference_python() with the
    row_sparse stand-ins bound in the reference's optimizer module"""
    assert available(), "needs /root/reference, oracle/_ref/libmxref.so and libmxref_sparse_update.so"
    with RP.reference_python() as (opt, sched):
        nd = sys.modules['mxnet.ndarray']
        for k, f in op_table().items():
            if k == 'sparse':
                nd.sparse.adagrad_update = f.adagrad_update
                nd.sparse.ftrl_update = f.ftrl_update
                f = nd.sparse
            setattr(nd, k, f)
            setattr(opt, k, f)          # optimizer.py bound them at import (from ..ndarray import ...)
        yield opt, sched


SHAPES = [(40, 8), (23, 5), (9, 512), (17,)]


def trajectory_cases():
    """4 steps per case; every step updates a different seeded row set of each key (always the
    first and last rows, never the rows listed in COLD). Gradients are kept as two halves per key
    (the store's two pushed values over the same rows); g/2 + g/2 == g exactly."""
    rng = np.random.default_rng(0xB200 + 11)

    def plan():
        w0 = [rng.uniform(-1, 1, s).astype(F) for s in SHAPES]
        for w in w0:
            w[w == 0] = F(0.5)                           # every row stays stored by tostype
        grads = []
        for _ in range(4):
            gs = []
            for s in SHAPES:
                rows = s[0]
                hot = np.arange(rows)[np.arange(rows) % 4 != 2]          # rows 2, 6, 10, ... stay cold
                pick = rng.choice(hot[1:-1], size=max(1, len(hot) // 2), replace=False)
                ids = np.unique(np.concatenate([[0, rows - 1] if (rows - 1) % 4 != 2 else [0], pick]))
                g = rng.uniform(-1, 1, (len(ids),) + s[1:]).astype(F)
                g[np.abs(g) < 2.0 ** -12] = F(0.5)
                assert np.array_equal(g, (g / F(2)) * F(2))
                gs.append((ids.astype(np.int64), g))
            grads.append(gs)
        return dict(shapes=SHAPES, w0=w0, grads=grads)
    c = {}
    c['ftrl'] = dict(plan(), opt=('Ftrl', dict(learning_rate=0.1, lamda1=0.01, beta=1, wd=1e-4)))
    c['ftrl_clip'] = dict(plan(), opt=('Ftrl', dict(learning_rate=0.05, lamda1=0.02, beta=0.5,
                                                    clip_gradient=0.5)))
    c['adagrad'] = dict(plan(), opt=('AdaGrad', dict(learning_rate=0.05)))
    c['adagrad_rescale'] = dict(plan(), opt=('AdaGrad', dict(learning_rate=0.1, eps=1e-6,
                                                             rescale_grad=1 / 8, clip_gradient=2.0)))
    return c


def cold_rows(shape):
    return np.arange(shape[0])[np.arange(shape[0]) % 4 == 2]


def run_trajectory(opt_mod, case, make_rsp=RspNDArray):
    """(tables, states) after every step: [step][key], through opt_mod's own Updater"""
    name, kw = case['opt']
    upd = opt_mod.get_updater(getattr(opt_mod, name)(**kw))
    ws = [make_rsp(w.shape, np.arange(w.shape[0]), w.copy()) for w in case['w0']]
    out = []
    for gs in case['grads']:
        for k, (ids, g) in enumerate(gs):
            upd(k, make_rsp(ws[k].shape, ids, g.copy()), ws[k])
        states = []
        for k in range(len(ws)):
            s = upd.states[k]
            states.append([x.asnumpy() for x in (s if isinstance(s, (tuple, list)) else [s])])
        out.append(([w.asnumpy() for w in ws], states))
    return out


def gen_trajectories():
    d = {}
    with reference_python_sparse_update() as (opt, _):
        for name, case in trajectory_cases().items():
            for step, (ws, sts) in enumerate(run_trajectory(opt, case)):
                for k, (w, st) in enumerate(zip(ws, sts)):
                    assert not np.any(np.isnan(w)), (name, step, k)
                    d["%s_step%d_w%d" % (name, step, k)] = w
                    for i, s in enumerate(st):
                        d["%s_step%d_w%d_s%d" % (name, step, k, i)] = s
    np.savez_compressed(os.path.join(GOLD, "updater_trajectories_sparse.npz"), **d)


if __name__ == "__main__":
    GS.build()
    gen_trajectories()
