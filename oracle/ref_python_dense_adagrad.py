"""TEST INFRASTRUCTURE ONLY -- the reference's own AdaGrad (python/mxnet/optimizer/optimizer.py:
1632-1688) and GroupAdaGrad (optimizer/contrib.py:30-100) classes, loaded unmodified by
oracle/ref_python.py, training dense weights with dense gradients over the reference's own operators.
Their dense branches compose NDArray arithmetic; the stand-in NDArray of oracle/ref_python_arith.py
runs it in oracle/_ref/libmxref_arith.so, and this module adds what those two branches need beyond
it, from oracle/_ref/libmxref_dense_adagrad.so (golden_dense_adagrad.ref()):

    square(nd)                          square
    mean(nd, axis=..., keepdims=...)    mean, with the keywords the caller gave, str()-formatted
    nd op nd, rhs of shape lhs.shape[:-1] + (1,)
                                        broadcast_add / _sub / _mul / _div / _maximum, row broadcast

Writes tests/golden/updater_trajectories_dense_adagrad.npz: per case, step and key the weight
(`<case>_step<s>_w<k>`) and the history (`<case>_step<s>_w<k>_s0`) after the step:

    make -f oracle/arith_ops.mk -f oracle/dense_adagrad.mk && python oracle/ref_python_dense_adagrad.py
"""
import contextlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import golden_dense_adagrad as GD  # noqa: E402
import ref_python as RP  # noqa: E402
import ref_python_arith as RPA  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
CLASSES = ('AdaGrad', 'GroupAdaGrad')


def available():
    return RPA.available() and GD.ref() is not None


class NDArray(RPA.NDArray):
    """RPA.NDArray with the row broadcast of the binary operators"""

    def _new(self, a):
        return NDArray(np.ascontiguousarray(a).reshape(self.a.shape), self.context)

    def __getitem__(self, key):
        return NDArray(self.a[key], self.context)

    def astype(self, dtype, copy=True):
        return NDArray(self.a.astype(np.dtype(dtype)), self.context)

    def copy(self):
        return NDArray(self.a.copy(), self.context)

    def _apply(self, other, op, scalar_op):
        if isinstance(other, RP.NDArray) and other.a.shape != self.a.shape:
            assert other.a.shape == self.a.shape[:-1] + (1,) and other.a.dtype == self.a.dtype
            RP.LOG.append((op, {}))
            return GD.ref().broadcast(op, self.a, other.a, RPA._dt(self.a))
        return super(NDArray, self)._apply(other, op, scalar_op)


def zeros(shape, ctx=None, dtype=None, stype=None, **_):
    assert stype in (None, 'default')
    return NDArray(np.zeros(shape, np.float32 if dtype is None else np.dtype(dtype)), ctx)


def square(data, out=None):
    RP.LOG.append(('square', {}))
    res = GD.ref().square(data.a, RPA._dt(data.a))
    return data._new(res) if out is None else out._put(res)


def mean(data, axis=None, keepdims=None, exclude=None, out=None):
    """the generated front-end passes only the keywords given, each as str()"""
    params = {k: str(v) for k, v in (('axis', axis), ('keepdims', keepdims), ('exclude', exclude))
              if v is not None}
    RP.LOG.append(('mean', params))
    res = GD.ref().mean(data.a, RPA._dt(data.a), **params)
    return NDArray(res, data.context) if out is None else out._put(res)


def op_table():
    """the names the reference's optimizer and contrib modules import for these optimizers"""
    t = RPA.op_table()
    t.update(NDArray=NDArray, zeros=zeros, square=square, mean=mean)
    return t


@contextlib.contextmanager
def reference_python_dense_adagrad():
    """with reference_python_dense_adagrad() as (opt, contrib): the reference's optimizer module
    and its optimizer/contrib.py over the stand-ins"""
    assert available(), "needs /root/reference and the oracle/_ref/ libraries"
    with RP.reference_python() as (opt, _):
        nd = sys.modules['mxnet.ndarray']
        for k, f in op_table().items():
            setattr(nd, k, f)
            setattr(opt, k, f)
        contrib = RP._load('mxnet.optimizer.contrib', os.path.join(RP.REF_PY, 'optimizer', 'contrib.py'))
        yield opt, contrib


def trajectory_cases():
    """4 steps per case through one updater, keys in order. Gradients are kept as two halves per
    key (the store's two pushed values); g/2 + g/2 == g exactly, so the merged gradient is `grads`
    in either order."""
    rng = np.random.default_rng(0xB200 + 13)
    dense_shapes = [(4, 4), (40, 25), (1027,), (3,), (2, 3, 4, 5)]
    group_shapes = [(40, 1), (17, 33), (6, 100), (3, 2)]

    def plan(shapes, dtype=np.float32):
        w0 = [rng.uniform(-1, 1, s).astype(np.float32).astype(dtype) for s in shapes]
        grads = []
        for _ in range(4):
            gs = []
            for s in shapes:
                # magnitudes 1e-2 to 1 side by side, so that a row's mean depends on its order
                g = (rng.uniform(-1, 1, s) * np.where(rng.random(s) < 0.5, 1.0, 1e-2)).astype(dtype)
                g[np.abs(g) < 2.0 ** -12] = dtype(0.5)          # halves stay exact in float16
                assert np.array_equal(g, (g / dtype(2)) * dtype(2))
                gs.append(g)
            grads.append(gs)
        return dict(shapes=shapes, w0=w0, grads=grads, dtype=np.dtype(dtype).name)
    c = {}
    c['adagrad'] = dict(plan(dense_shapes), opt=('AdaGrad', dict(wd=1e-4, rescale_grad=0.5)))
    c['adagrad_nowd'] = dict(plan(dense_shapes), opt=('AdaGrad', dict(learning_rate=0.1)))
    c['adagrad_clip'] = dict(plan(dense_shapes), opt=('AdaGrad', dict(learning_rate=0.05, clip_gradient=0.5,
                                                                     eps=1e-6)))
    c['adagrad_clip0'] = dict(plan(dense_shapes), opt=('AdaGrad', dict(clip_gradient=0, wd=1e-3,
                                                                      rescale_grad=2.0)))
    c['adagrad_mp_fp16'] = dict(plan(dense_shapes, np.float16),
                                opt=('AdaGrad', dict(wd=1e-4, rescale_grad=1 / 64, multi_precision=True)))
    c['group'] = dict(plan(group_shapes), opt=('GroupAdaGrad', dict(learning_rate=0.05)))
    c['group_clip'] = dict(plan(group_shapes), opt=('GroupAdaGrad', dict(learning_rate=0.1, eps=1e-6,
                                                                        clip_gradient=0.5)))
    c['group_rescale'] = dict(plan(group_shapes), opt=('GroupAdaGrad', dict(learning_rate=0.1,
                                                                           rescale_grad=1 / 8)))
    return c


def history(state):
    """the history array of a key's state (a multi-precision state is (weight32, history))"""
    return state[1] if isinstance(state, (tuple, list)) else state


def run_trajectory(opt_mod, cls, case, ndarray=NDArray):
    """(weights, histories) after every step: [step][key], through opt_mod's own Updater"""
    upd = opt_mod.get_updater(cls(**case['opt'][1]))
    ws = [ndarray(w.copy()) for w in case['w0']]
    w_out, h_out = [], []
    for gs in case['grads']:
        for k, g in enumerate(gs):
            upd(k, ndarray(g.copy()), ws[k])
        w_out.append([w.a.copy() for w in ws])
        h_out.append([history(upd.states[k]).a.copy() for k in range(len(ws))])
    return w_out, h_out


def classes(opt, contrib):
    return {'AdaGrad': opt.AdaGrad, 'GroupAdaGrad': contrib.GroupAdaGrad}


def gen_trajectories():
    d = {}
    with reference_python_dense_adagrad() as (opt, contrib):
        for name, case in trajectory_cases().items():
            ws, hs = run_trajectory(opt, classes(opt, contrib)[case['opt'][0]], case)
            for step in range(len(ws)):
                for k, (w, h) in enumerate(zip(ws[step], hs[step])):
                    assert not np.any(np.isnan(w)), (name, step, k)
                    d["%s_step%d_w%d" % (name, step, k)] = w
                    d["%s_step%d_w%d_s0" % (name, step, k)] = h
    np.savez_compressed(os.path.join(GOLD, "updater_trajectories_dense_adagrad.npz"), **d)
    return d


if __name__ == "__main__":
    GD.build()
    print("wrote", len(gen_trajectories()), "arrays")
