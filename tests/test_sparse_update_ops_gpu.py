"""The row_sparse forms of ftrl_update and _sparse_adagrad_update on the GPU, bit for bit against the
reference's own CPU kernels: every case of tests/golden/sparse_update_ops.npz through mx.nd (rows
outside the gradient untouched in the weight and every state, empty gradients, empty states), the
refusals (operands untouched), and the reference's Ftrl / AdaGrad trajectories on row_sparse tables
(tests/golden/updater_trajectories_sparse.npz, written by oracle/ref_python_sparse_update.py)
through the store's callback route and across a checkpoint."""
import os

import numpy as np
import pytest

import golden_sparse_update_ops as GS
from ref_python_sparse_update import trajectory_cases, cold_rows

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
    if stype == GS.DNS:
        return mx.nd.array(a, mx.gpu(0))
    if empty:
        return mx.nd.sparse.zeros('row_sparse', a.shape, mx.gpu(0))
    return rsp(mx, a, np.arange(a.shape[0]), a.shape)


def nnr(a):
    return a.indices.shape[0] if a.stype == 'row_sparse' else 0


def call(mx, case, name, nds, g):
    if case['form'] == 'ftrl':
        # mx.nd.ftrl_update takes the row_sparse form from its operands; the alias is the same operator
        f = mx.nd.sparse.ftrl_update if 'clip' in name else mx.nd.ftrl_update
    else:
        f = mx.nd.sparse.adagrad_update
    f(nds[0], g, *nds[1:], out=nds[0], **case['params'])


@pytest.mark.parametrize("name", sorted(GS.CASES))
def test_sparse_update_golden(mx, golden, name):
    case = GS.CASES[name]
    tables, steps, st_nnr = GS.inputs(case)
    shape = tables[0].shape
    nds = [table(mx, tables[0], case['wstype'])] + \
          [table(mx, s, case['wstype'], n == 0) for s, n in zip(tables[1:], st_nnr)]
    touched = np.zeros(shape[0], bool)
    for ids, g in steps:
        call(mx, case, name, nds, rsp(mx, g, ids, shape))
        touched[ids] = True
    got = [a.asnumpy() for a in nds]
    g = golden("sparse_update_ops")
    if case['wstype'] == GS.RSP:             # an empty state was zero-filled to every row
        assert eq(np.array([nnr(a) for a in nds[1:]], np.int64), g['%s|nnr' % name])
    for tag, a in zip(['w'] + ['s%d' % i for i in range(len(got) - 1)], got):
        if a.size <= GS.FULL_MAX:
            assert eq(a, g['%s|%s' % (name, tag)]), (name, tag)
        else:
            assert eq(a.reshape(-1)[:GS.HEAD], g['%s|%s|head' % (name, tag)]), (name, tag)
            assert eq(GS.GU.digest(a), g['%s|%s|sha256' % (name, tag)]), (name, tag)
    for a, before in zip(got, tables):       # rows no gradient listed: bitwise as they were
        assert eq(a[~touched], before[~touched]), name


def _untouched(mx, call_, arrays):
    before = [(a.asnumpy().copy(), nnr(a)) for a in arrays]
    with pytest.raises(mx.base.MXNetError):
        call_()
    mx.nd.waitall()
    for a, (b, n) in zip(arrays, before):
        assert eq(a.asnumpy(), b) and nnr(a) == n


def test_sparse_update_refusals(mx):
    rng = np.random.default_rng(5)
    rows, L = 12, 8
    shape = (rows, L)
    u = lambda *s: rng.uniform(-1, 1, s).astype(np.float32)  # noqa: E731
    g = rsp(mx, u(3, L), [0, 4, 11], shape)
    full = lambda: rsp(mx, u(rows, L), np.arange(rows), shape)  # noqa: E731
    empty = lambda: mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))  # noqa: E731
    dense = lambda: mx.nd.array(u(rows, L), mx.gpu(0))  # noqa: E731
    # a row_sparse weight that misses rows
    w, z, n = rsp(mx, u(rows - 1, L), np.arange(rows - 1), shape), empty(), empty()
    _untouched(mx, lambda: mx.nd.ftrl_update(w, g, z, n, out=w, lr=0.1), [w, z, n])
    w, h = rsp(mx, u(rows - 1, L), np.arange(1, rows), shape), empty()
    _untouched(mx, lambda: mx.nd.sparse.adagrad_update(w, g, h, out=w, lr=0.1), [w, h])
    # wd != 0 for AdaGrad, in both forms
    w, h = full(), empty()
    _untouched(mx, lambda: mx.nd.sparse.adagrad_update(w, g, h, out=w, lr=0.1, wd=0.01), [w, h])
    w, h = dense(), dense()
    _untouched(mx, lambda: mx.nd.sparse.adagrad_update(w, g, h, out=w, lr=0.1, wd=0.01), [w, h])
    # a distinct out, and no out
    w, z, n, o = full(), empty(), full(), full()
    _untouched(mx, lambda: mx.nd.ftrl_update(w, g, z, n, out=o, lr=0.1), [w, z, n, o])
    _untouched(mx, lambda: mx.nd.sparse.ftrl_update(w, g, z, n, lr=0.1), [w, z, n])
    w, h, o = dense(), dense(), dense()
    _untouched(mx, lambda: mx.nd.sparse.adagrad_update(w, g, h, out=o, lr=0.1), [w, h, o])
    # mixed storage types
    w, z, n = full(), dense(), empty()
    _untouched(mx, lambda: mx.nd.ftrl_update(w, g, z, n, out=w, lr=0.1), [w, z, n])
    w, h = dense(), empty()
    _untouched(mx, lambda: mx.nd.sparse.adagrad_update(w, g, h, out=w, lr=0.1), [w, h])
    w, h = full(), empty()
    gd = dense()
    _untouched(mx, lambda: mx.nd.sparse.adagrad_update(w, gd, h, out=w, lr=0.1), [w, h, gd])
    w, h = dense(), dense()
    _untouched(mx, lambda: mx.nd.sparse.adagrad_update(w, gd, h, out=w, lr=0.1), [w, h, gd])
    # float16
    w16 = mx.nd.array(u(rows, L), mx.gpu(0), np.float16)
    h16 = mx.nd.array(np.zeros(shape), mx.gpu(0), np.float16)
    _untouched(mx, lambda: mx.nd.sparse.adagrad_update(w16, g, h16, out=w16, lr=0.1), [w16, h16])
    w, z, n = full(), empty(), empty()
    g16 = rsp(mx, u(3, L), [0, 4, 11], shape, np.float16)
    _untouched(mx, lambda: mx.nd.ftrl_update(w, g16, z, n, out=w, lr=0.1), [w, z, n])


# --------------------------------------------------------------------- optimizer trajectories
TRAJ = trajectory_cases()


def _optimizer(name):
    from compat import mxnet_optimizer_sparse as mxopt
    cls, kw = TRAJ[name]['opt']
    return getattr(mxopt, cls)(**kw)


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


def _check_step(kv, gold, name, step, outs):
    for k, o in enumerate(outs):
        assert eq(o.asnumpy(), gold["%s_step%d_w%d" % (name, step, k)]), (name, step, k)
        st = kv._updater.states[k]
        for i, s in enumerate(st if isinstance(st, (tuple, list)) else [st]):
            assert eq(s.asnumpy(), gold["%s_step%d_w%d_s%d" % (name, step, k, i)]), (name, step, k, i)


@pytest.mark.parametrize("name", sorted(TRAJ))
def test_store_callback_trajectory(mx, golden, name):
    """kv.set_optimizer(<mirror of the reference class>) on row_sparse tables: two values per key, 4
    pushes over different rows, then row_sparse_pull of every row; tables and states per step"""
    gold = golden("updater_trajectories_sparse")
    case = TRAJ[name]
    kv = _store(mx, name, case['w0'])
    for step, gs in enumerate(case['grads']):
        outs = _step(mx, kv, case, gs)
        _check_step(kv, gold, name, step, outs)
    for k, s in enumerate(case['shapes']):
        cold = cold_rows(s)
        assert eq(outs[k].asnumpy()[cold], case['w0'][k][cold]), (name, k)


@pytest.mark.parametrize("name", ['ftrl', 'adagrad'])
def test_sparse_checkpoint_restart(mx, golden, tmp_path, name):
    """save_optimizer_states after step 2 (row_sparse states), a fresh store loads them: steps 3
    and 4 equal the uninterrupted trajectory"""
    gold = golden("updater_trajectories_sparse")
    case = TRAJ[name]
    fname = os.path.join(str(tmp_path), "%s.states" % name)
    kv = _store(mx, name, case['w0'])
    for gs in case['grads'][:2]:
        outs = _step(mx, kv, case, gs)
    kv.save_optimizer_states(fname, dump_optimizer=True)
    kv2 = _store(mx, name, [o.asnumpy() for o in outs])
    kv2.load_optimizer_states(fname)
    for step, gs in list(enumerate(case['grads']))[2:]:
        _check_step(kv2, gold, name, step, _step(mx, kv2, case, gs))
