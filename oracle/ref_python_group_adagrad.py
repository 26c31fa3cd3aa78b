"""TEST INFRASTRUCTURE ONLY -- the reference's own GroupAdaGrad optimizer class
(python/mxnet/optimizer/contrib.py, loaded unmodified beside optimizer.py by oracle/ref_python.py)
training tables over the reference's own _contrib_group_adagrad_update kernel
(golden_group_adagrad.ref(), i.e. oracle/_ref/libmxref_group_adagrad.so). The stand-in
`mxnet.ndarray` of oracle/ref_python_sparse_update.py gains `contrib.group_adagrad_update` and the
other names contrib.py imports (`mean`, unused by the row_sparse branch).

Writes tests/golden/updater_trajectories_group_adagrad.npz: per case, key and step, the table and
the history after the step. Cases `rsp_*` hold row_sparse tables (the store's updater callback);
cases `dns_*` hold dense tables with row_sparse gradients (a local updater, Gluon's
Embedding(sparse_grad=True) with update_on_kvstore=False).

    make -f oracle/group_adagrad.mk && python oracle/ref_python_group_adagrad.py
"""
import contextlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import golden_group_adagrad as GG  # noqa: E402
import ref_python as RP  # noqa: E402
import ref_python_sparse_update as RPS  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
F = np.float32


def available():
    return RPS.available() and GG.ref() is not None


def call(fn, ins, out, params):
    """one _contrib_group_adagrad_update on stand-in arrays through fn (GG.ref() or GG.restate)"""
    w, g, h = ins
    rows = w.shape[0]
    L = int(np.prod(w.shape[1:]))
    stypes, nnr, bufs = [], [], []
    for i, (a, width) in enumerate(zip(ins, (L, L, 1))):
        rsp = isinstance(a, RPS.RspNDArray)
        stypes.append(1 if rsp else 0)
        if i == 1:
            nnr.append(len(a.idx))
            bufs.append(np.ascontiguousarray(a.vals.reshape(len(a.idx), L)))
        elif rsp:       # a table: all rows (ids 0..rows-1) or none
            assert len(a.idx) in (0, rows) and (len(a.idx) == 0 or np.array_equal(a.idx, np.arange(rows)))
            nnr.append(len(a.idx))
            full = np.zeros((rows, width), F)
            full[:len(a.idx)] = a.vals.reshape(len(a.idx), width)
            bufs.append(full)
        else:
            nnr.append(0)
            bufs.append(a.a.reshape(rows, width))
    fn(GG.OP, stypes, nnr, bufs, g.idx, rows, L, out is w, **params)
    for i, a in enumerate(ins):
        if i != 1 and isinstance(a, RPS.RspNDArray):
            a.idx = np.arange(nnr[i], dtype=np.int64)
            a.vals = bufs[i][:nnr[i]].reshape((nnr[i],) + a.shape[1:]).copy()
    return out


def _group_adagrad_update(fn=None):
    def op(weight, grad, history, out=None, name=None, **kwargs):
        RP.LOG.append((GG.OP, {k: str(v) for k, v in kwargs.items()}))
        return call(fn or GG.ref(), [weight, grad, history], out, kwargs)
    op.__name__ = 'group_adagrad_update'
    return op


def op_table(fn=None):
    """the names the reference's GroupAdaGrad (and the tests/compat mirror) use; fn: the kernel behind
    the operator (default: the reference's own, GG.ref())"""
    return {'zeros': RPS.zeros,
            'contrib': types.SimpleNamespace(group_adagrad_update=_group_adagrad_update(fn))}


@contextlib.contextmanager
def reference_python_group_adagrad():
    """with reference_python_group_adagrad() as (opt, contrib, sched): the reference's optimizer,
    optimizer/contrib.py and lr_scheduler modules over the stand-ins"""
    assert available(), "needs /root/reference and the oracle/_ref/ libraries"
    with RPS.reference_python_sparse_update() as (opt, sched):
        nd = sys.modules['mxnet.ndarray']
        nd.contrib.group_adagrad_update = op_table()['contrib'].group_adagrad_update
        nd.mean = RP._unused('mean')   # the dense-gradient branch only
        contrib = RP._load('mxnet.optimizer.contrib', os.path.join(RP.REF_PY, 'optimizer', 'contrib.py'))
        yield opt, contrib, sched


class ListSched(object):
    """a learning-rate scheduler by table: the values FactorScheduler(step=2, factor=0.5,
    base_lr=0.1) gives for num_update 1..4 (test_mirror checks both against the reference)"""
    base_lr = 0.1
    LRS = [0.1, 0.1, 0.05, 0.05]

    def __call__(self, num_update):
        return self.LRS[min(num_update, len(self.LRS)) - 1]


SHAPES = [(40, 8), (23, 5), (9, 512), (17, 33)]


def trajectory_cases():
    """4 steps per case over RPS.trajectory_cases()'s row plans (rows in RPS.cold_rows never get a
    gradient); `sched` marks the case that runs with a learning-rate scheduler"""
    rng = np.random.default_rng(0xB200 + 12)

    def plan():
        w0 = [rng.uniform(-1, 1, s).astype(F) for s in SHAPES]
        for w in w0:
            w[w == 0] = F(0.5)
        grads = []
        for _ in range(4):
            gs = []
            for s in SHAPES:
                rows = s[0]
                hot = np.arange(rows)[np.arange(rows) % 4 != 2]
                pick = rng.choice(hot[1:-1], size=max(1, len(hot) // 2), replace=False)
                ids = np.unique(np.concatenate([[0, rows - 1] if (rows - 1) % 4 != 2 else [0], pick]))
                g = rng.uniform(-1, 1, (len(ids),) + s[1:]).astype(F)
                g[np.abs(g) < 2.0 ** -12] = F(0.5)
                assert np.array_equal(g, (g / F(2)) * F(2))
                gs.append((ids.astype(np.int64), g))
            grads.append(gs)
        return dict(shapes=SHAPES, w0=w0, grads=grads)
    c = {}
    for form in ('rsp', 'dns'):
        c[form] = dict(plan(), form=form, opt=dict(learning_rate=0.05))
        c[form + '_clip'] = dict(plan(), form=form, opt=dict(learning_rate=0.1, eps=1e-6, clip_gradient=0.5))
        c[form + '_rescale'] = dict(plan(), form=form, opt=dict(learning_rate=0.1, rescale_grad=1 / 8))
        c[form + '_sched'] = dict(plan(), form=form, opt=dict(), sched=True)
    return c


def run_trajectory(opt_mod, cls, case, sched, make_rsp=RPS.RspNDArray, make_dense=RP.NDArray):
    """(tables, histories) after every step: [step][key], through opt_mod's own Updater.
    sched: the scheduler object of a `sched` case"""
    kw = dict(case['opt'], lr_scheduler=sched) if case.get('sched') else case['opt']
    upd = opt_mod.get_updater(cls(**kw))
    if case['form'] == 'rsp':
        ws = [make_rsp(w.shape, np.arange(w.shape[0]), w.copy()) for w in case['w0']]
    else:
        ws = [make_dense(w.copy()) for w in case['w0']]
    out = []
    for gs in case['grads']:
        for k, (ids, g) in enumerate(gs):
            upd(k, make_rsp(ws[k].shape, ids, g.copy()), ws[k])
        out.append(([w.asnumpy() for w in ws], [upd.states[k].asnumpy() for k in range(len(ws))]))
    return out


def gen_trajectories():
    d = {}
    with reference_python_group_adagrad() as (opt, contrib, sched):
        for name, case in trajectory_cases().items():
            s = sched.FactorScheduler(step=2, factor=0.5, base_lr=0.1)
            for step, (ws, hs) in enumerate(run_trajectory(opt, contrib.GroupAdaGrad, case, s)):
                for k, (w, h) in enumerate(zip(ws, hs)):
                    assert not np.any(np.isnan(w)), (name, step, k)
                    d["%s_step%d_w%d" % (name, step, k)] = w
                    d["%s_step%d_w%d_s0" % (name, step, k)] = h
    np.savez_compressed(os.path.join(GOLD, "updater_trajectories_group_adagrad.npz"), **d)


if __name__ == "__main__":
    GG.build()
    gen_trajectories()
