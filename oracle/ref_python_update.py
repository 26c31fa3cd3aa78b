"""TEST INFRASTRUCTURE ONLY -- the reference's own NAG / Signum / RMSProp / FTML / Ftrl optimizer
classes (python/mxnet/optimizer/optimizer.py, loaded unmodified by oracle/ref_python.py) running over
the reference's own operators: oracle/ref_python.py's stand-in `mxnet.ndarray` with the eight operators
those classes call forwarded to oracle/_ref/libmxref_update.so (golden_update_ops.ref(), the real
dmlc::Parameter parser + FCompute<cpu>), and fp32 -> fp16 `cast` as mshadow's half_t constructor
rounds it (nearest even), for the master-weight route of Optimizer.update_multi_precision.

Writes tests/golden/updater_trajectories_ext.npz (the reference's Python cannot travel to the GPU
machine; the fixture does):

    make -f oracle/update_ops.mk && python oracle/ref_python_update.py
"""
import contextlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import golden_update_ops as GU  # noqa: E402
import ref_python as RP  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")


def available():
    return RP.available() and GU.ref() is not None


def _update_op(name):
    def op(*args, **kwargs):
        out = kwargs.pop('out')
        kwargs.pop('name', None)
        ins = [a.a.reshape(-1) for a in RP._flat(args)]
        RP.LOG.append((name, {k: str(v) for k, v in kwargs.items()}))
        GU.ref().op_invoke(name, ins, [o.a.reshape(-1) for o in RP._flat([out])], **kwargs)
        return out
    op.__name__ = name
    return op


def cast(data, dtype, out=None):
    """Cast (src/operator/tensor/elemwise_unary_op.h): float32 -> float16 by half_t(float), round to
    nearest even -- numpy's conversion"""
    res = data.a.astype(np.dtype(dtype))
    if out is None:
        return RP.NDArray(res, data.context)
    out.a[...] = res
    return out


def op_table():
    """the names the reference's optimizer module imports for these optimizers"""
    t = {n: _update_op(n) for n in GU.OPS}
    t['cast'] = cast
    return t


@contextlib.contextmanager
def reference_python_update():
    """with reference_python_update() as (opt, sched): ref_python.reference_python() with the
    eight operators (and cast) bound in the reference's optimizer module"""
    assert available(), "needs /root/reference, oracle/_ref/libmxref.so and libmxref_update.so"
    with RP.reference_python() as (opt, sched):
        nd = sys.modules['mxnet.ndarray']
        for k, f in op_table().items():
            setattr(nd, k, f)
            setattr(opt, k, f)          # optimizer.py bound them at import (from ..ndarray import ...)
        yield opt, sched


def trajectory_cases():
    """4 steps of (key, merged gradient, stored weight) per key through the store's callback route,
    one case per optimizer branch. Gradients are kept as two halves per key (the store's two pushed
    values); g/2 + g/2 == g exactly, so the merged gradient is `grads` whatever the summation order."""
    rng = np.random.default_rng(0xB200 + 7)
    shapes = [(4, 4), (40, 25), (1027,), (3,), (2001,)]

    def plan(dtype=np.float32):
        w0 = [GU.F(rng.uniform(-1, 1, s)).astype(dtype) for s in shapes]
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
    c['nag_mom0'] = dict(plan(), opt=('NAG', dict(learning_rate=0.1, wd=1e-4, rescale_grad=1 / 256)))
    c['nag_mom'] = dict(plan(), opt=('NAG', dict(learning_rate=0.05, momentum=0.9, wd=1e-4, clip_gradient=0.5,
                                                 rescale_grad=0.5)))
    c['nag_mp_fp16'] = dict(plan(np.float16), opt=('NAG', dict(learning_rate=0.05, momentum=0.9, wd=1e-4,
                                                               rescale_grad=1 / 64, multi_precision=True)))
    c['signsgd'] = dict(plan(), opt=('Signum', dict(learning_rate=0.01, momentum=0.0, wd=1e-3)))
    c['signum'] = dict(plan(), opt=('Signum', dict(learning_rate=0.01, momentum=0.9, wd=1e-3, wd_lh=0.01,
                                                   clip_gradient=0.5)))
    c['rmsprop'] = dict(plan(), opt=('RMSProp', dict(learning_rate=0.001, gamma1=0.9, wd=1e-3,
                                                     clip_weights=0.5)))
    c['rmsprop_centered'] = dict(plan(), opt=('RMSProp', dict(learning_rate=0.001, gamma1=0.95, gamma2=0.9,
                                                              centered=True, clip_weights=0.5,
                                                              clip_gradient=0.5)))
    c['rmsprop_mp_fp16'] = dict(plan(np.float16), opt=('RMSProp', dict(learning_rate=0.001, wd=1e-4,
                                                                      multi_precision=True)))
    c['ftml'] = dict(plan(), opt=('FTML', dict(learning_rate=0.01, wd=1e-4, clip_gradient=0.5)))
    c['ftrl'] = dict(plan(), opt=('Ftrl', dict(learning_rate=0.1, lamda1=0.01, beta=1, wd=1e-4)))
    return c


def run_trajectory(opt_mod, case, ndarray=RP.NDArray):
    """weights after every step: [step][key], through opt_mod's own Updater"""
    name, kw = case['opt']
    upd = opt_mod.get_updater(getattr(opt_mod, name)(**kw))
    ws = [ndarray(w.copy()) for w in case['w0']]
    out = []
    for gs in case['grads']:
        for k, g in enumerate(gs):
            upd(k, ndarray(g.copy()), ws[k])
        out.append([w.a.copy() for w in ws])
    return out


def gen_trajectories():
    d = {}
    with reference_python_update() as (opt, _):
        for name, case in trajectory_cases().items():
            for step, ws in enumerate(run_trajectory(opt, case)):
                for k, w in enumerate(ws):
                    assert not np.any(np.isnan(w)), (name, step, k)
                    d["%s_step%d_w%d" % (name, step, k)] = w
    np.savez_compressed(os.path.join(GOLD, "updater_trajectories_ext.npz"), **d)


if __name__ == "__main__":
    GU.build()
    gen_trajectories()
