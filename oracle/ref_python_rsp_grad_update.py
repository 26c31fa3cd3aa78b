"""TEST INFRASTRUCTURE ONLY -- the reference's own NAG, Signum, RMSProp, FTML and Ftrl optimizer classes
(python/mxnet/optimizer/optimizer.py, loaded unmodified by oracle/ref_python.py) training DENSE tables
with row_sparse gradients (the `RspNDArray` of oracle/ref_python_sparse_update.py), which is what a
gluon Trainer hands them for Embedding(sparse_grad=True). Their operators have no FComputeEx for a
(dense weight, row_sparse gradient) pair, so the stand-ins densify the gradient at the operator
boundary (golden_rsp_grad_update_ops.densify, the reference's kFComputeFallback) and run the
reference's own dense operator (golden_update_ops.ref(), oracle/_ref/libmxref_update.so). NAG without
momentum calls sgd_update, whose (dense, row_sparse) form the reference does serve: the lazy update of
golden_sparse_sgd_adam.step over the reference's own kernels (oracle/_ref/libmxref.so).

Every operator call is logged with the storage types of its operands (`OPLOG`).

Writes tests/golden/updater_trajectories_rsp_grad.npz (the reference's Python cannot travel to the GPU
machine; the fixture does): per case, key and step, the table and the optimizer states after the step
(golden_rsp_grad_update_ops.put), and per case the operator log:

    make -f oracle/update_ops.mk && make -C oracle ref && python oracle/ref_python_rsp_grad_update.py
"""
import contextlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import golden_rsp_grad_update_ops as GR  # noqa: E402
import golden_sparse_sgd_adam as GSA  # noqa: E402
import golden_update_ops as GU  # noqa: E402
import kvoracle as K  # noqa: E402
import ref_python as RP  # noqa: E402
import ref_python_sparse_update as RSU  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
F = np.float32
OPLOG = []        # "operator(stype, stype, ...)" of every call, in order


def available():
    return RP.available() and GU.ref() is not None and K.ref() is not None


def _stypes(name, args):
    return "%s(%s)" % (name, ", ".join(a.stype for a in args))


def _fallback_op(name):
    """a dense-weight operator: a row_sparse gradient is densified first (kFComputeFallback)"""
    def op(*args, **kwargs):
        out = kwargs.pop('out')
        kwargs.pop('name', None)
        OPLOG.append(_stypes(name, args))
        RP.LOG.append((name, {k: str(v) for k, v in kwargs.items()}))
        assert all(not isinstance(a, RSU.RspNDArray) for i, a in enumerate(args) if i != 1)
        g = args[1]
        gd = GR.densify(g.shape, g.idx, g.vals) if isinstance(g, RSU.RspNDArray) else g.a
        ins = [args[0].a.reshape(-1), gd.reshape(-1)] + [a.a.reshape(-1) for a in args[2:]]
        GU.ref().op_invoke(name, ins, [out.a.reshape(-1)], **kwargs)
        return out
    op.__name__ = name
    return op


def sgd_update(weight, grad, out=None, **kwargs):
    """sgd_update on a dense weight: SGDUpdateEx's lazy (dense, row_sparse) form for a row_sparse
    gradient (lazy_update defaults to True), else the dense FCompute"""
    kwargs.pop('name', None)
    OPLOG.append(_stypes('sgd_update', [weight, grad]))
    if not isinstance(grad, RSU.RspNDArray):
        return RP.op_table()['sgd_update'](weight, grad, out=out, **kwargs)
    RP.LOG.append(('sgd_update', {k: str(v) for k, v in kwargs.items()}))
    assert out is weight
    rows = weight.shape[0]
    row_len = int(np.prod(weight.shape[1:]))
    GSA.step(K.ref(), 'sgd_update', [weight.a.reshape(rows, row_len)], [], None, grad.idx,
             grad.vals.reshape(len(grad.idx), row_len), kwargs)
    return out


def op_table():
    t = {n: _fallback_op(n) for n in GR.OPS}
    t['sgd_update'] = sgd_update
    return t


@contextlib.contextmanager
def reference_python_rsp_grad_update():
    """with reference_python_rsp_grad_update() as (opt, sched): ref_python.reference_python() with
    the stand-ins bound in the reference's optimizer module"""
    assert available(), "needs /root/reference, oracle/_ref/libmxref.so and libmxref_update.so"
    with RP.reference_python() as (opt, sched):
        nd = sys.modules['mxnet.ndarray']
        for k, f in op_table().items():
            setattr(nd, k, f)
            setattr(opt, k, f)          # optimizer.py bound them at import (from ..ndarray import ...)
        yield opt, sched


def trajectory_cases():
    """4 steps per case over the tables and row sets of ref_python_sparse_update.trajectory_cases
    (4 keys, first and last rows always in the gradient, two halves per key for the store's two
    pushed values); the tables are dense"""
    base = RSU.trajectory_cases()
    plans = [dict((k, base[n][k]) for k in ('shapes', 'w0', 'grads')) for n in sorted(base)]
    opts = {
        'nag_mom0': ('NAG', dict(learning_rate=0.1, wd=1e-4, rescale_grad=0.5)),
        'nag_mom': ('NAG', dict(learning_rate=0.05, momentum=0.9, wd=1e-4, clip_gradient=0.5)),
        'signsgd': ('Signum', dict(learning_rate=0.01, momentum=0.0, wd=1e-3)),
        'signum': ('Signum', dict(learning_rate=0.01, momentum=0.9, wd=1e-3, wd_lh=0.01, clip_gradient=0.5)),
        'rmsprop': ('RMSProp', dict(learning_rate=0.001, gamma1=0.9, wd=1e-3, clip_weights=0.5)),
        'rmsprop_centered': ('RMSProp', dict(learning_rate=0.001, gamma1=0.95, gamma2=0.9, centered=True,
                                             clip_weights=0.5, clip_gradient=0.5)),
        'ftml': ('FTML', dict(learning_rate=0.01, wd=1e-4, clip_gradient=0.5)),
        'ftrl': ('Ftrl', dict(learning_rate=0.1, lamda1=0.01, beta=1, wd=1e-4)),
    }
    return {name: dict(plans[i % len(plans)], opt=opt) for i, (name, opt) in enumerate(opts.items())}


# the operator each case's optimizer calls, and the storage types it receives
EXPECTED_CALL = {
    'nag_mom0': 'sgd_update(default, row_sparse)',
    'nag_mom': 'nag_mom_update(default, row_sparse, default)',
    'signsgd': 'signsgd_update(default, row_sparse)',
    'signum': 'signum_update(default, row_sparse, default)',
    'rmsprop': 'rmsprop_update(default, row_sparse, default)',
    'rmsprop_centered': 'rmspropalex_update(default, row_sparse, default, default, default)',
    'ftml': 'ftml_update(default, row_sparse, default, default, default)',
    'ftrl': 'ftrl_update(default, row_sparse, default, default)',
}


def states_of(s):
    """an Updater's state of one key as a list: NAG and Signum without momentum keep None"""
    return [] if s is None else list(s) if isinstance(s, (tuple, list)) else [s]


def run_trajectory(opt_mod, case, make_dense, make_rsp=RSU.RspNDArray):
    """(tables, states) after every step: [step][key], through opt_mod's own Updater"""
    name, kw = case['opt']
    upd = opt_mod.get_updater(getattr(opt_mod, name)(**kw))
    ws = [make_dense(w.copy()) for w in case['w0']]
    out = []
    for gs in case['grads']:
        for k, (ids, g) in enumerate(gs):
            upd(k, make_rsp(ws[k].shape, ids, g.copy()), ws[k])
        out.append(([w.asnumpy() for w in ws], [[x.asnumpy() for x in states_of(upd.states[k])]
                                                for k in range(len(ws))]))
    return out


def gen_trajectories():
    d = {}
    with reference_python_rsp_grad_update() as (opt, _):
        for name, case in trajectory_cases().items():
            del OPLOG[:]
            for step, (ws, sts) in enumerate(run_trajectory(opt, case, RP.NDArray)):
                for k, (w, st) in enumerate(zip(ws, sts)):
                    assert not np.any(np.isnan(w)), (name, step, k)
                    GR.put(d, "%s_step%d_w%d" % (name, step, k), w)
                    for i, s in enumerate(st):
                        GR.put(d, "%s_step%d_w%d_s%d" % (name, step, k, i), s)
            d["%s|log" % name] = np.array(OPLOG)
    np.savez_compressed(os.path.join(GOLD, "updater_trajectories_rsp_grad.npz"), **d)
    return d


if __name__ == "__main__":
    GU.build()
    print(len(gen_trajectories()), "arrays")
