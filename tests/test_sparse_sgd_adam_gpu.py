"""sgd_update, sgd_mom_update and adam_update on row_sparse weights that hold every row, on the GPU,
bit for bit against the reference's own CPU kernels:
- every case of tests/golden/sparse_sgd_adam_ops.npz through mx.nd.sparse (lazy and standard forms,
  row_sparse and dense states, states that hold no rows yet, empty gradients, a table of more than
  one wave of CTAs), with the rows no gradient listed unchanged in the lazy form;
- the refusals, which leave every operand and row count as it was and launch nothing;
- the reference's SGD, ccSGD and Adam classes on row_sparse tables
  (tests/golden/updater_trajectories_sparse_sgd_adam.npz, written by
  oracle/ref_python_sparse_sgd_adam.py) through a local updater, through the store's callback route
  with row_sparse_pull, and across a checkpoint."""
import os

import numpy as np
import pytest

import golden_sparse_sgd_adam as GSA
import golden_sparse_update_ops as GS
import golden_update_ops as GU
from ref_python_sparse_sgd_adam import trajectory_cases, cold_rows, states_of, matches, n_states

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


def nnr(a):
    return a.indices.shape[0] if a.stype == 'row_sparse' else 0


def state(mx, a, sst, n):
    if sst == GSA.DNS:
        return mx.nd.array(a, mx.gpu(0))
    if n == 0:
        return mx.nd.sparse.zeros('row_sparse', a.shape, mx.gpu(0))
    return rsp(mx, a, np.arange(a.shape[0]), a.shape)


@pytest.mark.parametrize("name", sorted(GSA.CASES))
def test_sparse_sgd_adam_golden(mx, golden, name):
    case = GSA.CASES[name]
    op, nst, sst, _ = GSA.FORMS[case['form']]
    tables, steps, st_nnr = GSA.inputs(name)
    shape = tables[0].shape
    w = rsp(mx, tables[0], np.arange(shape[0]), shape)
    sts = [state(mx, s, sst, n) for s, n in zip(tables[1:], st_nnr)]
    lazy = case['params']['lazy_update'] and sst != GSA.DNS
    touched = np.zeros(shape[0], bool)
    f = getattr(mx.nd.sparse, op)
    for ids, g in steps:
        f(w, rsp(mx, g, ids, shape), *sts, out=w, **case['params'])
        touched[ids] = True
    got = [w.asnumpy()] + [s.asnumpy() for s in sts]
    gold = golden(GSA.NAME)
    assert nnr(w) == shape[0]
    if sst == GSA.RSP:                       # a state that held no rows now holds every row
        assert eq(np.array([nnr(s) for s in sts], np.int64), gold['%s|nnr' % name])
        assert all(nnr(s) == shape[0] for s in sts)
    for tag, a in zip(['w'] + ['s%d' % i for i in range(nst)], got):
        if a.size <= GS.FULL_MAX:
            assert eq(a, gold['%s|%s' % (name, tag)]), (name, tag)
        else:
            assert eq(a.reshape(-1)[:GS.HEAD], gold['%s|%s|head' % (name, tag)]), (name, tag)
            assert eq(GU.digest(a), gold['%s|%s|sha256' % (name, tag)]), (name, tag)
    if lazy:                                 # rows no gradient listed: bitwise as they were
        assert eq(got[0][~touched], tables[0][~touched]), name
        for a, before, n in zip(got[1:], tables[1:], st_nnr):
            want = before if n else np.zeros_like(before)
            assert eq(a[~touched], want[~touched]), name


def test_rsp_weight_equals_dense_weight(mx):
    """a row_sparse weight with every row runs the dense weight's kernels: the same bits in the lazy
    form (row_sparse states against dense ones) and in the standard form"""
    rng = np.random.default_rng(3)
    shape = (37, 12)
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    ids = np.array([0, 5, 6, 36])
    g = rng.uniform(-1, 1, (4, 12)).astype(np.float32)
    zeros = lambda: mx.nd.array(np.zeros(shape, np.float32), mx.gpu(0))  # noqa: E731
    for lazy in (True, False):
        a = rsp(mx, w0, np.arange(37), shape)
        if lazy:
            ma, va = [mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0)) for _ in range(2)]
        else:
            ma, va = zeros(), zeros()
        b, mb, vb = mx.nd.array(w0, mx.gpu(0)), zeros(), zeros()
        kw = dict(lr=0.01, wd=0.1, lazy_update=lazy)
        for _ in range(2):
            mx.nd.sparse.adam_update(a, rsp(mx, g, ids, shape), ma, va, out=a, **kw)
            mx.nd.adam_update(b, rsp(mx, g, ids, shape), mb, vb, out=b, **kw)
        assert eq(a.asnumpy(), b.asnumpy()) and eq(ma.asnumpy(), mb.asnumpy()) and eq(va.asnumpy(), vb.asnumpy())


@pytest.mark.parametrize("wst", ['default', 'row_sparse'])
def test_adam_std_absent_row_is_not_a_zero_row(mx, oracle, wst):
    """the standard Adam form tells a row absent from the gradient from a stored row of zeros
    (AdamStdDnsRspDnsKernel, optimizer_op.cc:195-229): with negative weights and wd = 0 an absent
    row's g' = w*wd is -0.0 and keeps a mean of -0.0, where g*rescale + w*wd with g = +0.0f would
    make it +0.0. Bit for bit against the C restatement of the reference's kernel."""
    import kvoracle as K
    rng = np.random.default_rng(5)
    shape = (23, 5)
    w0 = -rng.uniform(0.1, 1, shape).astype(np.float32)
    m0 = np.full(shape, -0.0, np.float32)
    v0 = rng.uniform(0, 0.01, shape).astype(np.float32)
    ids = np.array([2, 7, 11, 20], np.int64)
    g = rng.uniform(-1, 1, (len(ids), 5)).astype(np.float32)
    w = mx.nd.array(w0, mx.gpu(0)) if wst == 'default' else rsp(mx, w0, np.arange(23), shape)
    m, v = mx.nd.array(m0, mx.gpu(0)), mx.nd.array(v0, mx.gpu(0))
    mx.nd.sparse.adam_update(w, rsp(mx, g, ids, shape), m, v, out=w, lr=0.01, wd=0.0, lazy_update=False)
    want = [w0.copy(), m0.copy(), v0.copy()]
    oracle.adam_std_rsp_update(*want, ids, g, K.scalar_param(0.01), wd=0.0)
    absent = np.setdiff1d(np.arange(23), ids)
    assert np.all(np.signbit(want[1][absent])) and np.all(want[1][absent] == 0)
    for got, ref in zip((w, m, v), want):
        assert eq(got.asnumpy(), ref)


# ------------------------------------------------------------------------------------ refusals
def _untouched(mx, call_, arrays):
    before = [(a.asnumpy().copy(), nnr(a)) for a in arrays]
    mx.nd.waitall()
    launches = mx.base.kernel_launch_count()
    with pytest.raises(mx.base.MXNetError):
        call_()
    assert mx.base.kernel_launch_count() == launches
    mx.nd.waitall()
    for a, (b, n) in zip(arrays, before):
        assert eq(a.asnumpy(), b) and nnr(a) == n


def test_sparse_sgd_adam_refusals(mx):
    rng = np.random.default_rng(7)
    rows, L = 12, 8
    shape = (rows, L)
    u = lambda *s: rng.uniform(-1, 1, s).astype(np.float32)  # noqa: E731
    g = rsp(mx, u(3, L), [0, 4, 11], shape)
    full = lambda dt=np.float32: rsp(mx, u(rows, L), np.arange(rows), shape, dt)  # noqa: E731
    empty = lambda: mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))  # noqa: E731
    dense = lambda dt=np.float32: mx.nd.array(u(rows, L), mx.gpu(0), dt)  # noqa: E731
    sp = mx.nd.sparse
    for lazy in (True, False):
        kw = dict(lr=0.1, lazy_update=lazy)
        # a weight that misses one row, first or last
        for ids in (np.arange(rows - 1), np.arange(1, rows)):
            w, m, v = rsp(mx, u(rows - 1, L), ids, shape), empty(), empty()
            _untouched(mx, lambda: sp.sgd_update(w, g, out=w, **kw), [w])
            _untouched(mx, lambda: sp.sgd_mom_update(w, g, m, out=w, momentum=0.9, **kw), [w, m])
            _untouched(mx, lambda: sp.adam_update(w, g, m, v, out=w, **kw), [w, m, v])
        # a state that holds some rows
        w, m, v = full(), rsp(mx, u(3, L), [1, 2, 3], shape), empty()
        _untouched(mx, lambda: sp.sgd_mom_update(w, g, m, out=w, momentum=0.9, **kw), [w, m])
        _untouched(mx, lambda: sp.adam_update(w, g, v, m, out=w, **kw), [w, m, v])
        # out: another row_sparse array, a dense array, none
        w, m, v, o = full(), empty(), empty(), full()
        _untouched(mx, lambda: sp.sgd_update(w, g, out=o, **kw), [w, o])
        _untouched(mx, lambda: sp.adam_update(w, g, m, v, out=o, **kw), [w, m, v, o])
        od = dense()
        _untouched(mx, lambda: sp.sgd_mom_update(w, g, m, out=od, momentum=0.9, **kw), [w, m, od])
        _untouched(mx, lambda: sp.sgd_update(w, g, **kw), [w])
        # mean and var of different stypes
        w, m, v = full(), empty(), dense()
        _untouched(mx, lambda: sp.adam_update(w, g, m, v, out=w, **kw), [w, m, v])
        _untouched(mx, lambda: sp.adam_update(w, g, v, m, out=w, **kw), [w, m, v])
        # a dense gradient with a row_sparse weight
        w, m, gd = full(), empty(), dense()
        _untouched(mx, lambda: sp.sgd_update(w, gd, out=w, **kw), [w, gd])
        _untouched(mx, lambda: sp.sgd_mom_update(w, gd, m, out=w, momentum=0.9, **kw), [w, m, gd])
        # row_sparse states on a dense weight, with either gradient
        w, m, v = dense(), empty(), empty()
        for gg in (g, gd):
            _untouched(mx, lambda: sp.sgd_mom_update(w, gg, m, out=w, momentum=0.9, **kw), [w, m])
            _untouched(mx, lambda: sp.adam_update(w, gg, m, v, out=w, **kw), [w, m, v])
        # 16-bit and float64 operands
        for dt in (np.float16, np.float64):
            w, m = full(dt), empty()
            _untouched(mx, lambda: sp.sgd_mom_update(w, g, m, out=w, momentum=0.9, **kw), [w, m])
            w, m, v = full(), empty(), empty()
            gx = rsp(mx, u(3, L), [0, 4, 11], shape, dt)
            _untouched(mx, lambda: sp.adam_update(w, gx, m, v, out=w, **kw), [w, m, v])
            m, v = dense(dt), dense(dt)
            _untouched(mx, lambda: sp.adam_update(w, g, m, v, out=w, **kw), [w, m, v])
            m = full(dt)
            _untouched(mx, lambda: sp.sgd_mom_update(w, g, m, out=w, momentum=0.9, **kw), [w, m])


# --------------------------------------------------------------------- optimizer trajectories
TRAJ = trajectory_cases()
STORE = sorted(n for n in TRAJ if n.startswith('ccsgd'))


def _optimizer(name):
    from compat import mxnet_optimizer_sparse_sgd as mxopt
    cls, kw = TRAJ[name]['opt']
    return getattr(mxopt, cls)(**kw)


def _check(gold, name, step, ws, states):
    for k, (w, st) in enumerate(zip(ws, states)):
        assert matches(gold, "%s_step%d_w%d" % (name, step, k), w), (name, step, k)
        st = states_of(st)
        assert len(st) == n_states(gold, name, step, k)
        for i, s in enumerate(st):
            assert matches(gold, "%s_step%d_w%d_s%d" % (name, step, k, i), s.asnumpy()), (name, step, k, i)


@pytest.mark.parametrize("name", sorted(TRAJ))
def test_local_updater_trajectory(mx, golden, name):
    """get_updater(<mirror of the reference class>) on row_sparse tables: 4 steps over different rows"""
    from compat.mxnet_optimizer_sparse_sgd import get_updater
    gold = golden("updater_trajectories_sparse_sgd_adam")
    case = TRAJ[name]
    upd = get_updater(_optimizer(name))
    ws = [rsp(mx, w, np.arange(w.shape[0]), w.shape) for w in case['w0']]
    for step, gs in enumerate(case['grads']):
        for k, ((ids, g), s) in enumerate(zip(gs, case['shapes'])):
            upd(k, rsp(mx, g, ids, s), ws[k])
        _check(gold, name, step, [w.asnumpy() for w in ws], [upd.states[k] for k in range(len(ws))])
    for k, w in enumerate(ws):
        assert nnr(w) == w.shape[0]


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


@pytest.mark.parametrize("name", STORE)
def test_store_callback_trajectory(mx, golden, name):
    """kv.set_optimizer(ccSGD(...)) on row_sparse keys: the store calls the optimizer back per key
    with the stored table; two values per key, 4 pushes, then row_sparse_pull of every row"""
    gold = golden("updater_trajectories_sparse_sgd_adam")
    case = TRAJ[name]
    kv = _store(mx, name, case['w0'])
    for step, gs in enumerate(case['grads']):
        outs = _step(mx, kv, case, gs)
        _check(gold, name, step, [o.asnumpy() for o in outs], [kv._updater.states[k] for k in range(len(outs))])
    if 'lazy' in name:
        for k, s in enumerate(case['shapes']):
            cold = cold_rows(s)
            assert eq(outs[k].asnumpy()[cold], case['w0'][k][cold]), (name, k)


@pytest.mark.parametrize("name", ['ccsgd_mom_lazy', 'ccsgd_mom_std'])
def test_sparse_sgd_checkpoint_restart(mx, golden, tmp_path, name):
    """save_optimizer_states after step 2, a fresh store loads them: steps 3 and 4 equal the
    uninterrupted trajectory"""
    gold = golden("updater_trajectories_sparse_sgd_adam")
    case = TRAJ[name]
    fname = os.path.join(str(tmp_path), "%s.states" % name)
    kv = _store(mx, name, case['w0'])
    for gs in case['grads'][:2]:
        outs = _step(mx, kv, case, gs)
    kv.save_optimizer_states(fname, dump_optimizer=True)
    kv2 = _store(mx, name, [o.asnumpy() for o in outs])
    kv2.load_optimizer_states(fname)
    for step, gs in list(enumerate(case['grads']))[2:]:
        outs = _step(mx, kv2, case, gs)
        _check(gold, name, step, [o.asnumpy() for o in outs], [kv2._updater.states[k] for k in range(len(outs))])
