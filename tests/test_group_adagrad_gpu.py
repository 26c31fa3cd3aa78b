"""_contrib_group_adagrad_update (GroupAdaGrad) on the GPU, bit for bit against the reference's own CPU
kernel: every case of tests/golden/group_adagrad.npz through mx.nd.contrib.group_adagrad_update (rows
outside the gradient untouched in the weight and the history, empty gradients, empty histories),
the refusals (operands untouched), and the reference GroupAdaGrad's trajectories
(tests/golden/updater_trajectories_group_adagrad.npz, written by oracle/ref_python_group_adagrad.py)
through the store's callback route, across a checkpoint, and through a local updater on dense
tables."""
import os
import pickle

import numpy as np
import pytest

import golden_group_adagrad as GG
from ref_python_group_adagrad import trajectory_cases, ListSched
from ref_python_sparse_update import cold_rows

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def rsp(mx, vals, ids, shape, dtype=np.float32):
    return mx.nd.sparse.row_sparse_array((vals.reshape((len(ids),) + tuple(shape[1:])), np.asarray(ids)),
                                         shape=shape, ctx=mx.gpu(0), dtype=dtype)


def table(mx, a, stype, empty=False):
    if stype == GG.DNS:
        return mx.nd.array(a, mx.gpu(0))
    if empty:
        return mx.nd.sparse.zeros('row_sparse', a.shape, mx.gpu(0))
    return rsp(mx, a, np.arange(a.shape[0]), a.shape)


def nnr(a):
    return a.indices.shape[0] if a.stype == 'row_sparse' else 0


@pytest.mark.parametrize("name", sorted(GG.CASES))
def test_group_adagrad_golden(mx, golden, name):
    case = GG.CASES[name]
    w0, h0, steps, h_nnr = GG.inputs(case)
    shape = case['shape']
    w = table(mx, w0.reshape(shape), case['wstype'])
    h = table(mx, h0, case['wstype'], h_nnr == 0)
    touched = np.zeros(shape[0], bool)
    for ids, g in steps:
        mx.nd.contrib.group_adagrad_update(w, rsp(mx, g, ids, shape), h, out=w, **case['params'])
        touched[ids] = True
    got = [w.asnumpy().reshape(shape[0], -1), h.asnumpy()]
    g = golden("group_adagrad")
    if case['wstype'] == GG.RSP:             # an empty history was zero-filled to every row
        assert eq(np.array([nnr(h)], np.int64), g['%s|nnr' % name])
    for tag, a in zip(['w', 's0'], got):
        if a.size <= GG.FULL_MAX:
            assert eq(a, g['%s|%s' % (name, tag)]), (name, tag)
        else:
            assert eq(a.reshape(-1)[:GG.HEAD], g['%s|%s|head' % (name, tag)]), (name, tag)
            assert eq(GG.GU.digest(a), g['%s|%s|sha256' % (name, tag)]), (name, tag)
    for a, before in zip(got, [w0, h0]):     # rows no gradient listed: bitwise as they were
        assert eq(a[~touched], before[~touched]), name


def _untouched(mx, call_, arrays):
    before = [(a.asnumpy().copy(), nnr(a)) for a in arrays]
    with pytest.raises(mx.base.MXNetError):
        call_()
    mx.nd.waitall()
    for a, (b, n) in zip(arrays, before):
        assert eq(a.asnumpy(), b) and nnr(a) == n


def test_group_adagrad_refusals(mx):
    rng = np.random.default_rng(5)
    rows, L = 12, 8
    shape = (rows, L)
    u = lambda *s: rng.uniform(-1, 1, s).astype(np.float32)  # noqa: E731
    f = mx.nd.contrib.group_adagrad_update
    g = rsp(mx, u(3, L), [0, 4, 11], shape)
    full = lambda: rsp(mx, u(rows, L), np.arange(rows), shape)  # noqa: E731
    hist = lambda: rsp(mx, u(rows, 1), np.arange(rows), (rows, 1))  # noqa: E731
    hempty = lambda: mx.nd.sparse.zeros('row_sparse', (rows, 1), mx.gpu(0))  # noqa: E731
    dense = lambda *s: mx.nd.array(u(*(s or shape)), mx.gpu(0))  # noqa: E731
    # a row_sparse weight that misses rows; a history that holds only some rows
    w, h = rsp(mx, u(rows - 1, L), np.arange(1, rows), shape), hempty()
    _untouched(mx, lambda: f(w, g, h, out=w, lr=0.1), [w, h])
    w, h = full(), rsp(mx, u(rows - 2, 1), np.arange(rows - 2), (rows, 1))
    _untouched(mx, lambda: f(w, g, h, out=w, lr=0.1), [w, h])
    # wd is not a GroupAdagradParam field, in either form
    w, h = full(), hist()
    _untouched(mx, lambda: f(w, g, h, out=w, lr=0.1, wd=0.0), [w, h])
    w, h = dense(), dense(rows, 1)
    _untouched(mx, lambda: f(w, g, h, out=w, lr=0.1, wd=0.01), [w, h])
    # a distinct out, and no out
    w, h, o = full(), hempty(), full()
    _untouched(mx, lambda: f(w, g, h, out=o, lr=0.1), [w, h, o])
    _untouched(mx, lambda: f(w, g, h, lr=0.1), [w, h])
    w, h, o = dense(), dense(rows, 1), dense()
    _untouched(mx, lambda: f(w, g, h, out=o, lr=0.1), [w, h, o])
    # all dense; mixed storage types
    w, h, gd = dense(), dense(rows, 1), dense()
    _untouched(mx, lambda: f(w, gd, h, out=w, lr=0.1), [w, h, gd])
    w, h = dense(), hempty()
    _untouched(mx, lambda: f(w, g, h, out=w, lr=0.1), [w, h])
    w, h = full(), dense(rows, 1)
    _untouched(mx, lambda: f(w, g, h, out=w, lr=0.1), [w, h])
    w, h = full(), hist()
    _untouched(mx, lambda: f(w, gd, h, out=w, lr=0.1), [w, h, gd])
    # float16
    w16 = mx.nd.array(u(rows, L), mx.gpu(0), np.float16)
    h16 = mx.nd.array(np.zeros((rows, 1)), mx.gpu(0), np.float16)
    _untouched(mx, lambda: f(w16, g, h16, out=w16, lr=0.1), [w16, h16])
    w, h = full(), hempty()
    g16 = rsp(mx, u(3, L), [0, 4, 11], shape, np.float16)
    _untouched(mx, lambda: f(w, g16, h, out=w, lr=0.1), [w, h])
    # a history of the wrong shape: one value per element, or two per row
    w, h = dense(), dense()
    _untouched(mx, lambda: f(w, g, h, out=w, lr=0.1), [w, h])
    w, h = dense(), dense(rows, 2)
    _untouched(mx, lambda: f(w, g, h, out=w, lr=0.1), [w, h])
    w, h = full(), mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
    _untouched(mx, lambda: f(w, g, h, out=w, lr=0.1), [w, h])


# --------------------------------------------------------------------- optimizer trajectories
TRAJ = trajectory_cases()


def _optimizer(name):
    from compat import mxnet_optimizer_contrib as mxopt
    case = TRAJ[name]
    kw = dict(case['opt'], lr_scheduler=ListSched()) if case.get('sched') else case['opt']
    return mxopt.GroupAdaGrad(**kw)


def _store(mx, name, w0s):
    kv = mx.kv.create('device')
    for k, w in enumerate(w0s):
        kv.init(k, rsp(mx, w, np.arange(w.shape[0]), w.shape))
    kv.set_optimizer(_optimizer(name))
    return kv


def _step(mx, kv, case, gs):
    keys = list(range(len(case['shapes'])))
    vals = []
    for (ids, g), s in zip(gs, case['shapes']):
        h = (g / np.float32(2)).astype(np.float32)
        vals.append([rsp(mx, h, ids, s), rsp(mx, h, ids, s)])
    kv.push(keys, vals)
    outs = [mx.nd.sparse.zeros('row_sparse', s, mx.gpu(0)) for s in case['shapes']]
    kv.row_sparse_pull(keys, out=outs, row_ids=[mx.nd.array(np.arange(s[0]), mx.gpu(0), np.int64)
                                               for s in case['shapes']])
    return outs


def _check_step(gold, name, step, ws, states):
    for k, (w, h) in enumerate(zip(ws, states)):
        assert eq(w.asnumpy(), gold["%s_step%d_w%d" % (name, step, k)]), (name, step, k)
        assert eq(h.asnumpy(), gold["%s_step%d_w%d_s0" % (name, step, k)]), (name, step, k)


RSP_CASES = sorted(n for n in TRAJ if TRAJ[n]['form'] == 'rsp')


@pytest.mark.parametrize("name", RSP_CASES)
def test_store_callback_trajectory(mx, golden, name):
    """kv.set_optimizer(<mirror of the reference class>) on row_sparse tables: two values per key, 4
    pushes over different rows, then row_sparse_pull of every row; tables and histories per step"""
    gold = golden("updater_trajectories_group_adagrad")
    case = TRAJ[name]
    kv = _store(mx, name, case['w0'])
    for step, gs in enumerate(case['grads']):
        outs = _step(mx, kv, case, gs)
        states = [kv._updater.states[k] for k in range(len(outs))]
        assert all(s.stype == 'row_sparse' and s.shape == (w.shape[0], 1) for s, w in zip(states, outs))
        _check_step(gold, name, step, outs, states)
    for k, s in enumerate(case['shapes']):
        cold = cold_rows(s)
        assert eq(outs[k].asnumpy()[cold], case['w0'][k][cold]), (name, k)


def test_group_adagrad_checkpoint_restart(mx, golden, tmp_path):
    """save_optimizer_states after step 2 (row_sparse (rows, 1) histories), a fresh store loads
    them: steps 3 and 4 equal the uninterrupted trajectory"""
    name = 'rsp_sched'
    gold = golden("updater_trajectories_group_adagrad")
    case = TRAJ[name]
    fname = os.path.join(str(tmp_path), "%s.states" % name)
    kv = _store(mx, name, case['w0'])
    for gs in case['grads'][:2]:
        outs = _step(mx, kv, case, gs)
    kv.save_optimizer_states(fname, dump_optimizer=True)
    with open(fname, 'rb') as fh:
        states, _ = pickle.loads(fh.read())
    assert all(states[k].stype == 'row_sparse' and states[k].shape == (s[0], 1)
               for k, s in enumerate(case['shapes']))
    kv2 = _store(mx, name, [o.asnumpy() for o in outs])
    kv2.load_optimizer_states(fname)
    for step, gs in list(enumerate(case['grads']))[2:]:
        outs = _step(mx, kv2, case, gs)
        _check_step(gold, name, step, outs, [kv2._updater.states[k] for k in range(len(outs))])


@pytest.mark.parametrize("name", sorted(n for n in TRAJ if TRAJ[n]['form'] == 'dns'))
def test_local_updater_dense_table_trajectory(mx, golden, name):
    """(dense, row_sparse, dense): a local updater over dense tables with row_sparse gradients, the
    calls Trainer's update_on_kvstore=False route makes for Embedding(sparse_grad=True)"""
    from compat import mxnet_optimizer_contrib as mxopt
    gold = golden("updater_trajectories_group_adagrad")
    case = TRAJ[name]
    upd = mxopt.get_updater(_optimizer(name))
    ws = [mx.nd.array(w, mx.gpu(0)) for w in case['w0']]
    for step, gs in enumerate(case['grads']):
        for k, ((ids, g), s) in enumerate(zip(gs, case['shapes'])):
            upd(k, rsp(mx, g, ids, s), ws[k])
        _check_step(gold, name, step, ws, [upd.states[k] for k in range(len(ws))])
