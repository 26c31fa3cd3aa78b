"""TEST INFRASTRUCTURE ONLY -- the reference's own SGD, ccSGD and Adam optimizer classes
(python/mxnet/optimizer/optimizer.py, loaded unmodified by oracle/ref_python.py) training row_sparse
tables over the reference's own kernels (oracle/_ref/libmxref.so, through golden_sparse_sgd_adam.step).
The stand-in `mxnet.ndarray` of oracle/ref_python_sparse_update.py (row_sparse arrays and
`zeros(..., stype='row_sparse')`) gains sgd_update, sgd_mom_update and adam_update for a row_sparse
weight; calls on dense weights still go to the reference's FCompute<cpu>.

Writes tests/golden/updater_trajectories_sparse_sgd_adam.npz (the reference's Python cannot travel to
the GPU machine; the fixture does): per case, key and step, the table and the optimizer states after
the step, in full up to 1 024 elements and as a sha256 digest plus the first elements above that
(`put`; `matches` compares an array with an entry).

    make -C oracle ref && python oracle/ref_python_sparse_sgd_adam.py
"""
import contextlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import golden_sparse_sgd_adam as GSA  # noqa: E402
import golden_sparse_update_ops as GS  # noqa: E402
import golden_update_ops as GU  # noqa: E402
import kvoracle as K  # noqa: E402
import ref_python as RP  # noqa: E402
import ref_python_sparse_update as RSU  # noqa: E402
from ref_python_sparse_update import cold_rows  # noqa: E402,F401  (re-exported)

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
F = np.float32


def available():
    return RP.available() and K.ref() is not None


def _rsp_op(name, dense_op, b=None):
    """`name` on stand-in arrays: a row_sparse weight (every row) through golden_sparse_sgd_adam.step
    over backend b (default: the reference's kernels), any other weight through dense_op"""
    def op(*args, **kwargs):
        w = args[0]
        if not isinstance(w, RSU.RspNDArray):
            return dense_op(*args, **kwargs)
        out = kwargs.pop('out')
        kwargs.pop('name', None)
        RP.LOG.append((name, {k: str(v) for k, v in kwargs.items()}))
        assert out is w
        rows = w.shape[0]
        row_len = int(np.prod(w.shape[1:]))
        assert np.array_equal(w.idx, np.arange(rows)), "CheckAllRowsPresent"
        g, states = args[1], list(args[2:])
        sst = None if not states else GSA.RSP if isinstance(states[0], RSU.RspNDArray) else GSA.DNS
        tables, nnr = [w.vals.reshape(rows, row_len)], []
        for s in states:
            if sst == GSA.RSP:
                if len(s.idx) == 0:
                    s.vals = np.zeros((rows,) + s.shape[1:], F)
                nnr.append(len(s.idx))
                tables.append(s.vals.reshape(rows, row_len))
            else:
                tables.append(s.a.reshape(rows, row_len))
        GSA.step(b or K.ref(), name, tables, nnr, sst, g.idx, g.vals.reshape(len(g.idx), row_len), kwargs)
        for s, n in zip(states, nnr):
            s.idx = np.arange(n, dtype=np.int64)
        return out
    op.__name__ = name
    return op


def op_table(b=None):
    """the names the reference's SGD / ccSGD / Adam (and the tests/compat mirror) use, over
    ref_python.op_table(); b: the kernels behind the row_sparse-weight forms (default: the
    reference's own)"""
    dense = RP.op_table()
    t = {'zeros': RSU.zeros}
    for name in ('sgd_update', 'sgd_mom_update', 'adam_update'):
        t[name] = _rsp_op(name, dense[name], b)
    return t


@contextlib.contextmanager
def reference_python_sparse_sgd_adam():
    """with reference_python_sparse_sgd_adam() as (opt, sched): ref_python.reference_python() with
    the row_sparse stand-ins bound in the reference's optimizer module"""
    assert available(), "needs /root/reference and oracle/_ref/libmxref.so"
    with RP.reference_python() as (opt, sched):
        nd = sys.modules['mxnet.ndarray']
        for k, f in op_table().items():
            setattr(nd, k, f)
            setattr(opt, k, f)          # optimizer.py bound them at import (from ..ndarray import ...)
        yield opt, sched


def trajectory_cases():
    """4 steps per case over the tables and row sets of ref_python_sparse_update.trajectory_cases
    (cold rows never in a gradient; two halves per key for the store's two pushed values)"""
    base = RSU.trajectory_cases()
    plans = [dict((k, base[n][k]) for k in ('shapes', 'w0', 'grads')) for n in sorted(base)]
    opts = {
        'sgd_lazy': ('SGD', dict(learning_rate=0.1, wd=1e-4)),
        'sgd_std': ('SGD', dict(learning_rate=0.1, wd=1e-4, lazy_update=False)),
        'sgd_mom_lazy': ('SGD', dict(learning_rate=0.1, momentum=0.9, wd=1e-4, clip_gradient=0.5)),
        'sgd_mom_std': ('SGD', dict(learning_rate=0.1, momentum=0.9, wd=1e-4, rescale_grad=1 / 8,
                                    lazy_update=False)),
        'adam_lazy': ('Adam', dict(learning_rate=0.01, wd=1e-4)),
        'adam_std': ('Adam', dict(learning_rate=0.01, wd=1e-4, clip_gradient=0.5, lazy_update=False)),
        'ccsgd_lazy': ('ccSGD', dict(learning_rate=0.1, wd=1e-4, rescale_grad=0.5)),
        'ccsgd_mom_lazy': ('ccSGD', dict(learning_rate=0.1, momentum=0.9, wd=1e-4)),
        'ccsgd_mom_std': ('ccSGD', dict(learning_rate=0.1, momentum=0.9, lazy_update=False)),
    }
    return {name: dict(plans[i % len(plans)], opt=opt) for i, (name, opt) in enumerate(opts.items())}


def states_of(s):
    """an Updater's state of one key as a list: SGD without momentum keeps None"""
    return [] if s is None else list(s) if isinstance(s, (tuple, list)) else [s]


def run_trajectory(opt_mod, case, make_rsp=RSU.RspNDArray):
    """(tables, states) after every step: [step][key], through opt_mod's own Updater"""
    name, kw = case['opt']
    upd = opt_mod.get_updater(getattr(opt_mod, name)(**kw))
    ws = [make_rsp(w.shape, np.arange(w.shape[0]), w.copy()) for w in case['w0']]
    out = []
    for gs in case['grads']:
        for k, (ids, g) in enumerate(gs):
            upd(k, make_rsp(ws[k].shape, ids, g.copy()), ws[k])
        out.append(([w.asnumpy() for w in ws], [[x.asnumpy() for x in states_of(upd.states[k])]
                                                for k in range(len(ws))]))
    return out


def put(d, key, a):
    """fixture entry of one table or state: in full up to golden_sparse_update_ops.FULL_MAX elements,
    else its sha256 and first HEAD elements (golden_sparse_update_ops' layout)"""
    a = np.ascontiguousarray(a)
    if a.size <= GS.FULL_MAX:
        d[key] = a
    else:
        d[key + '|sha256'] = GU.digest(a)
        d[key + '|head'] = a.reshape(-1)[:GS.HEAD].copy()


def matches(gold, key, a):
    """a equals the fixture entry `key` bit for bit (in full, or by digest and head)"""
    want = {}
    put(want, key, a)
    return all(k in gold.files and np.array_equal(np.ascontiguousarray(v).view(np.uint8),
                                                  np.ascontiguousarray(gold[k]).view(np.uint8))
               for k, v in want.items())


def n_states(gold, name, step, k):
    """how many states the fixture holds for key k after `step`"""
    pre = "%s_step%d_w%d_s" % (name, step, k)
    return len({f.split('|')[0] for f in gold.files if f.startswith(pre)})


def gen_trajectories():
    d = {}
    with reference_python_sparse_sgd_adam() as (opt, _):
        for name, case in trajectory_cases().items():
            for step, (ws, sts) in enumerate(run_trajectory(opt, case)):
                for k, (w, st) in enumerate(zip(ws, sts)):
                    assert not np.any(np.isnan(w)), (name, step, k)
                    put(d, "%s_step%d_w%d" % (name, step, k), w)
                    for i, s in enumerate(st):
                        put(d, "%s_step%d_w%d_s%d" % (name, step, k, i), s)
    np.savez_compressed(os.path.join(GOLD, "updater_trajectories_sparse_sgd_adam.npz"), **d)
    return d


if __name__ == "__main__":
    print(len(gen_trajectories()), "arrays")
