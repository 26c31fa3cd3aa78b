"""Row_sparse values pushed to DENSE keys: the store step gluon.Trainer runs for a dense weight with a
sparse gradient (Embedding(sparse_grad=True); python/mxnet/gluon/trainer.py:141-160, 193-226,
375-388). The merge, the stored value's storage type, every pull form, the fused lazy and standard
updates, the updater callback and the refusals, bit for bit against the checker model
(oracle/kvoracle_sparse_grad.py)."""
import os

import numpy as np
import pytest

import kvoracle as K
import kvoracle_sparse_grad as SG

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def ngpu():
    import torch
    return torch.cuda.device_count()


def rsp_value(mx, rng, shape, nnr, ctx, idx=None):
    if idx is None:
        idx = np.sort(rng.choice(shape[0], nnr, replace=False))
    idx = np.asarray(idx, np.int64)
    val = rng.uniform(-1, 1, (idx.size,) + tuple(shape[1:])).astype(np.float32)
    if idx.size == 0:
        return mx.nd.sparse.zeros('row_sparse', shape, ctx), SG.Rsp(idx, val, shape)
    return mx.nd.sparse.row_sparse_array((val, idx), shape=shape, ctx=ctx), SG.Rsp(idx, val, shape)


def all_rows(mx, shape, ctx):
    return mx.nd.array(np.arange(shape[0]), ctx, np.int64)


def check_value(mx, kv, model, key, shape, ctx):
    """every pull form of the key against the model"""
    dense = [mx.nd.empty(shape, ctx) for _ in range(2)]
    kv.pull(key, out=dense)
    for d in dense:
        assert eq(d.asnumpy(), model.pull(key))
    if model.stype[key] != 'row_sparse':
        return
    want_idx, want_val = model.pull_rsp(key)
    rows2d = want_val.reshape(want_idx.size, int(np.prod(shape[1:])))
    outs = [mx.nd.sparse.zeros('row_sparse', shape, ctx) for _ in range(2)]
    kv.pull(key, out=outs, ignore_sparse=False)
    for o in outs:
        assert np.array_equal(o.indices.asnumpy(), want_idx)
        assert eq(o.data.asnumpy(), want_val)
    # row_sparse_pull works on the key now: every row, then a subset with duplicates
    o = mx.nd.sparse.zeros('row_sparse', shape, ctx)
    kv.row_sparse_pull(key, out=o, row_ids=all_rows(mx, shape, ctx))
    if want_idx.size == 0:   # an all-zero value: FillZerosRspImpl (sparse_retain-inl.h:271-275)
        assert o.indices.shape[0] == 0
        return
    ri, rv = K.get_oracle().sparse_retain(want_idx, rows2d, np.arange(shape[0]))
    assert np.array_equal(o.indices.asnumpy(), ri) and eq(o.data.asnumpy().reshape(ri.size, -1), rv)
    req = np.random.default_rng(1).integers(0, shape[0], 40)
    kv.row_sparse_pull(key, out=o, row_ids=mx.nd.array(req, ctx, np.int64))
    ri, rv = K.get_oracle().sparse_retain(want_idx, rows2d, np.unique(req))
    assert np.array_equal(o.indices.asnumpy(), ri) and eq(o.data.asnumpy().reshape(ri.size, -1), rv)


@pytest.mark.parametrize("row_len", [1, 3, 4, 512])
@pytest.mark.parametrize("nsrc", [1, 2, 3, 8, 9])
def test_merge_and_pulls_without_updater(mx, nsrc, row_len):
    rng = np.random.default_rng(nsrc * 1000 + row_len)
    shape = (300, row_len)
    ctx = mx.gpu(0)
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    kv = mx.kv.create('device')
    model = SG.DenseKeySparseGradModel('device')
    kv.init(3, mx.nd.array(w0, ctx))
    model.init(3, w0)
    for rep in range(2):
        srcs = [rsp_value(mx, rng, shape, 0 if (i == 1 and nsrc >= 3) else 40, ctx) for i in range(nsrc)]
        kv.push(3, [s[0] for s in srcs])
        model.push(3, [s[1] for s in srcs])
        assert model.stype[3] == 'row_sparse'
        check_value(mx, kv, model, 3, shape, ctx)


def test_empty_overlapping_and_every_row_layouts(mx):
    rng = np.random.default_rng(7)
    shape = (64, 5)
    ctx = mx.gpu(0)
    kv = mx.kv.create('device')
    model = SG.DenseKeySparseGradModel('device')
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    kv.init('w', mx.nd.array(w0, ctx))
    model.init('w', w0)
    layouts = [
        [[], []],                                   # all-empty push: the value is all zeros
        [np.arange(64), np.arange(64), np.arange(64)],  # every row in every source
        [[0, 5, 63], [5, 6], [63]],                 # overlapping
        [[], [10]],
    ]
    for ids in layouts:
        srcs = [rsp_value(mx, rng, shape, None, ctx, idx=i) for i in ids]
        kv.push('w', [s[0] for s in srcs])
        model.push('w', [s[1] for s in srcs])
        check_value(mx, kv, model, 'w', shape, ctx)
    out = mx.nd.sparse.zeros('row_sparse', shape, ctx)
    kv.push('w', [rsp_value(mx, rng, shape, None, ctx, idx=[])[0]])
    kv.pull('w', out=out, ignore_sparse=False)
    assert out.indices.shape[0] == 0 and not out.asnumpy().any()


def test_storage_type_transitions(mx):
    """dense init -> row_sparse push -> pulls -> dense push -> row_sparse push with an optimizer"""
    rng = np.random.default_rng(11)
    shape = (50, 8)
    ctx = mx.gpu(0)
    kv = mx.kv.create('device')
    model = SG.DenseKeySparseGradModel('device')
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    kv.init(0, mx.nd.array(w0, ctx))
    model.init(0, w0)
    o = mx.nd.sparse.zeros('row_sparse', shape, ctx)
    with pytest.raises(mx.base.MXNetError, match="PullRowSparse expects row_sparse src NDArray"):
        kv.row_sparse_pull(0, out=o, row_ids=all_rows(mx, shape, ctx))
    # ignore_sparse=True (the default) skips row_sparse outs
    sentinel = mx.nd.sparse.row_sparse_array((np.full((1, 8), 7, np.float32), np.array([2])), shape=shape, ctx=ctx)
    kv.pull(0, out=sentinel)
    assert np.array_equal(sentinel.indices.asnumpy(), [2]) and np.all(sentinel.data.asnumpy() == 7)
    a, ra = rsp_value(mx, rng, shape, 9, ctx)
    kv.push(0, [a])
    model.push(0, [ra])
    check_value(mx, kv, model, 0, shape, ctx)
    kv.pull(0, out=sentinel)
    assert np.array_equal(sentinel.indices.asnumpy(), [2]) and np.all(sentinel.data.asnumpy() == 7)
    g = rng.uniform(-1, 1, shape).astype(np.float32)
    kv.push(0, [mx.nd.array(g, ctx)])
    model.push(0, [g])
    assert model.stype[0] == 'default'
    check_value(mx, kv, model, 0, shape, ctx)
    with pytest.raises(mx.base.MXNetError, match="PullRowSparse expects row_sparse src NDArray"):
        kv.row_sparse_pull(0, out=o, row_ids=all_rows(mx, shape, ctx))
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9))
    model.set_optimizer('sgd', lr=0.1, momentum=0.9)
    a, ra = rsp_value(mx, rng, shape, 9, ctx)
    kv.push(0, [a, a])
    model.push(0, [ra, ra])
    assert model.stype[0] == 'default'
    check_value(mx, kv, model, 0, shape, ctx)


def test_optimizer_after_row_sparse_value(mx):
    """an optimizer set while the value is row_sparse updates zeros plus the stored rows"""
    rng = np.random.default_rng(12)
    shape = (40, 4)
    ctx = mx.gpu(0)
    kv = mx.kv.create('device')
    model = SG.DenseKeySparseGradModel('device')
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    kv.init(0, mx.nd.array(w0, ctx))
    model.init(0, w0)
    a, ra = rsp_value(mx, rng, shape, 5, ctx)
    kv.push(0, [a])
    model.push(0, [ra])
    kv.set_optimizer(mx.optimizer.Adam(learning_rate=0.01))
    model.set_optimizer('adam', lr=0.01)
    a, ra = rsp_value(mx, rng, shape, 5, ctx)
    kv.push(0, [a])
    model.push(0, [ra])
    check_value(mx, kv, model, 0, shape, ctx)


def _optimizers(mx, name, lazy):
    kw = dict(learning_rate=0.1, wd=1e-3, rescale_grad=0.5, clip_gradient=0.3, lazy_update=lazy)
    mk = dict(lr=0.1, wd=1e-3, rescale_grad=0.5, clip_gradient=0.3, lazy_update=lazy)
    if name == 'sgd':
        return mx.optimizer.SGD(**kw), ('sgd', dict(mk))
    if name == 'sgd_mom':
        return mx.optimizer.SGD(momentum=0.9, **kw), ('sgd', dict(mk, momentum=0.9))
    kw['learning_rate'] = mk['lr'] = 1e-2
    return mx.optimizer.Adam(**kw), ('adam', mk)


@pytest.mark.parametrize("lazy", [True, False])
@pytest.mark.parametrize("name", ['sgd', 'sgd_mom', 'adam'])
def test_fused_updates_share_state_with_dense_pushes(mx, name, lazy, tmp_path):
    rng = np.random.default_rng(21)
    shape = (200, 12)
    ctx = mx.gpu(0)
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    opt, (kind, mk) = _optimizers(mx, name, lazy)
    kv = mx.kv.create('device')
    kv.init(5, mx.nd.array(w0, ctx))
    kv.set_optimizer(opt)
    model = SG.DenseKeySparseGradModel('device')
    model.init(5, w0)
    model.set_optimizer(kind, **mk)
    fname = os.path.join(str(tmp_path), "states")
    steps = ['rsp', 'rsp', 'dense', 'save', 'rsp', 'dense', 'rsp']
    for step in steps:
        if step == 'save':
            kv.save_optimizer_states(fname, dump_optimizer=True)
            out = mx.nd.empty(shape, ctx)
            kv.pull(5, out=out)
            kv = mx.kv.create('device')
            kv.init(5, out)
            kv.set_optimizer(_optimizers(mx, name, lazy)[0])
            kv.load_optimizer_states(fname)
            continue
        before = model.pull(5)
        if step == 'rsp':
            srcs = [rsp_value(mx, rng, shape, 30, ctx) for _ in range(3)]
            kv.push(5, [s[0] for s in srcs])
            model.push(5, [s[1] for s in srcs])
            if lazy:   # rows no gradient names stay as they were
                touched = np.unique(np.concatenate([s[1].idx for s in srcs]))
                cold = np.setdiff1d(np.arange(shape[0]), touched)
                assert eq(model.pull(5)[cold], before[cold])
        else:
            gs = [rng.uniform(-1, 1, shape).astype(np.float32) for _ in range(2)]
            kv.push(5, [mx.nd.array(g, ctx) for g in gs])
            model.push(5, gs)
        out = mx.nd.empty(shape, ctx)
        kv.pull(5, out=out)
        assert eq(out.asnumpy(), model.pull(5)), step
        assert model.stype[5] == 'default'


def _callback_optimizer(name):
    if name == 'sgd':
        from compat import mxnet_optimizer as M
        return M.SGD(learning_rate=0.1, momentum=0.9, wd=1e-3), M.get_updater
    if name == 'adam':
        from compat import mxnet_optimizer as M
        return M.Adam(learning_rate=0.01), M.get_updater
    if name == 'adagrad':
        from compat import mxnet_optimizer_sparse as M
        return M.AdaGrad(learning_rate=0.1), M.get_updater
    from compat import mxnet_optimizer_contrib as M
    return M.GroupAdaGrad(learning_rate=0.1), M.get_updater


@pytest.mark.parametrize("name", ['sgd', 'adam', 'adagrad', 'group_adagrad'])
def test_callback_route(mx, name, monkeypatch):
    """the updater receives (row_sparse merged gradient, dense stored weight): the store's trajectory
    equals the same updater applied to the merged gradient by hand"""
    monkeypatch.setenv('B200KV_FUSED_OPTIMIZER', '0')
    rng = np.random.default_rng(31)
    shape = (120, 16)
    ctx = mx.gpu(0)
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    kv = mx.kv.create('device')
    kv.init(1, mx.nd.array(w0, ctx))
    opt, get_updater = _callback_optimizer(name)
    kv.set_optimizer(opt)
    upd = get_updater(_callback_optimizer(name)[0])
    w = mx.nd.array(w0, ctx)
    oracle = K.get_oracle()
    for _ in range(3):
        srcs = [rsp_value(mx, rng, shape, 25, ctx) for _ in range(2)]
        kv.push(1, [s[0] for s in srcs])
        gi, gv = oracle.rsp_reduce([s[1].idx for s in srcs], [s[1].val for s in srcs])
        upd(1, mx.nd.sparse.row_sparse_array((gv.reshape((gi.size,) + shape[1:]), gi), shape=shape, ctx=ctx), w)
        out = mx.nd.empty(shape, ctx)
        kv.pull(1, out=out)
        assert eq(out.asnumpy(), w.asnumpy())


def test_trainer_loop_update_on_kvstore_false_and_true_agree(mx):
    """Trainer._allreduce_grads + _update restated for 2 devices and 3 steps with lazy SGD:
    update_on_kvstore=False (push, pull into the row_sparse grads, local sgd_update per device) and
    True (the store's fused step, pull into the dense weights) give identical weights"""
    rng = np.random.default_rng(41)
    shape = (500, 32)
    ctx = mx.gpu(0)
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    ndev = 2
    kw = dict(learning_rate=0.1, wd=1e-4, rescale_grad=1.0 / ndev)
    # update_on_kvstore=False
    kv_f = mx.kv.create('device')
    ws_f = [mx.nd.array(w0, ctx) for _ in range(ndev)]
    kv_f.init(0, ws_f[0])
    kv_f.pull(0, out=ws_f)
    from compat import mxnet_optimizer as M
    upds = [M.get_updater(M.SGD(**kw)) for _ in range(ndev)]
    # update_on_kvstore=True
    kv_t = mx.kv.create('device')
    ws_t = [mx.nd.array(w0, ctx) for _ in range(ndev)]
    kv_t.init(0, ws_t[0])
    kv_t.pull(0, out=ws_t)
    kv_t.set_optimizer(mx.optimizer.SGD(**kw))
    model = SG.DenseKeySparseGradModel('device')
    model.init(0, w0)
    model.set_optimizer('sgd', lr=0.1, wd=1e-4, rescale_grad=1.0 / ndev)
    for _ in range(3):
        srcs = [rsp_value(mx, rng, shape, 60, ctx) for _ in range(ndev)]
        grads = [s[0].copy() for s in srcs]
        kv_f.push(0, grads)
        kv_f.pull(0, out=grads, ignore_sparse=False)
        for d in range(ndev):
            upds[d](0, grads[d], ws_f[d])
        kv_t.push(0, [s[0] for s in srcs])
        kv_t.pull(0, out=ws_t)
        model.push(0, [s[1] for s in srcs])
        for d in range(ndev):
            assert eq(ws_f[d].asnumpy(), ws_t[d].asnumpy())
            assert eq(ws_t[d].asnumpy(), model.pull(0))


def test_queued_dense_calls_then_row_sparse_push(mx):
    """single-key dense calls are queued; a row_sparse push runs them first, and a repeated dense
    pull (a cached call) sees the row_sparse value, then the dense one again"""
    rng = np.random.default_rng(51)
    shape = (80, 8)
    ctx = mx.gpu(0)
    kv = mx.kv.create('device')
    model = SG.DenseKeySparseGradModel('device')
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    kv.init(0, mx.nd.array(w0, ctx))
    model.init(0, w0)
    out = mx.nd.empty(shape, ctx)
    for _ in range(2):
        g = rng.uniform(-1, 1, shape).astype(np.float32)
        kv.push(0, mx.nd.array(g, ctx))
        model.push(0, [g])
        kv.pull(0, out=out)
        kv.pull(0, out=out)
        a, ra = rsp_value(mx, rng, shape, 10, ctx)
        kv.push(0, [a])
        model.push(0, [ra])
        for _ in range(2):
            kv.pull(0, out=out)
            assert eq(out.asnumpy(), model.pull(0))


def test_refusals_leave_value_and_state_unchanged(mx, tmp_path):
    rng = np.random.default_rng(61)
    shape = (30, 4)
    ctx = mx.gpu(0)
    kv = mx.kv.create('device')
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    kv.init(0, mx.nd.array(w0, ctx))
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9))
    kv.push(0, [rsp_value(mx, rng, shape, 6, ctx)[0]])

    def snapshot():
        out = mx.nd.empty(shape, ctx)
        kv.pull(0, out=out)
        f = os.path.join(str(tmp_path), "s")
        kv.save_optimizer_states(f)
        with open(f, 'rb') as fh:
            return out.asnumpy(), fh.read()
    w_before, s_before = snapshot()
    bad_shape = rsp_value(mx, rng, (31, 4), 3, ctx)[0]
    with pytest.raises(mx.base.MXNetError, match="shape mismatch"):
        kv.push(0, [bad_shape])
    idx = np.array([1, 2])
    bad_dtype = mx.nd.sparse.row_sparse_array((np.ones((2, 4), np.float16), idx), shape=shape, ctx=ctx,
                                              dtype=np.float16)
    with pytest.raises(mx.base.MXNetError, match="dtype mismatch"):
        kv.push(0, [bad_dtype])
    w_after, s_after = snapshot()
    assert eq(w_after, w_before) and s_after == s_before
    # a float16 dense key
    kv16 = mx.kv.create('device')
    kv16.init(0, mx.nd.array(w0, ctx, np.float16))
    with pytest.raises(mx.base.MXNetError, match="float32"):
        kv16.push(0, [bad_dtype])
    out = mx.nd.empty(shape, ctx, np.float16)
    kv16.pull(0, out=out)
    assert eq(out.asnumpy(), w0.astype(np.float16))
    # kvstore 'nccl' takes dense values only
    kvn = mx.kv.create('nccl')
    kvn.init(0, mx.nd.array(w0, ctx))
    with pytest.raises(mx.base.MXNetError, match="nccl"):
        kvn.push(0, [rsp_value(mx, rng, shape, 3, ctx)[0]])
    out = mx.nd.empty(shape, ctx)
    kvn.pull(0, out=out)
    assert eq(out.asnumpy(), w0)


@pytest.mark.skipif(ngpu() < 2, reason="needs 2 GPUs")
def test_two_gpus_striped_whole_striped(mx):
    """a key striped over 2 GPUs by dense pushes is made whole for a row_sparse push (values and
    outs on both GPUs, outs on GPU 1 written by peer stores) and striped again by the next dense
    push; the momentum carries across"""
    rng = np.random.default_rng(71)
    shape = (70001, 3)
    ctxs = [mx.gpu(0), mx.gpu(1)]
    kv = mx.kv.create('device')
    model = SG.DenseKeySparseGradModel('device')
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    kv.init(0, mx.nd.array(w0, ctxs[0]))
    model.init(0, w0)
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9))
    model.set_optimizer('sgd', lr=0.1, momentum=0.9)
    for step in ['dense', 'rsp', 'dense', 'rsp']:
        if step == 'dense':
            gs = [rng.uniform(-1, 1, shape).astype(np.float32) for _ in ctxs]
            kv.push(0, [mx.nd.array(g, c) for g, c in zip(gs, ctxs)])
            model.push(0, gs)
        else:
            srcs = [rsp_value(mx, rng, shape, 3000, c) for c in ctxs]
            kv.push(0, [s[0] for s in srcs])
            model.push(0, [s[1] for s in srcs])
        outs = [mx.nd.empty(shape, c) for c in ctxs]
        kv.pull(0, out=outs)
        for o in outs:
            assert eq(o.asnumpy(), model.pull(0)), step
    # no updater: a row_sparse value pulled into outs on both GPUs
    kv2 = mx.kv.create('device')
    kv2.init(1, mx.nd.array(w0, ctxs[0]))
    model2 = SG.DenseKeySparseGradModel('device')
    model2.init(1, w0)
    gs = [rng.uniform(-1, 1, shape).astype(np.float32) for _ in ctxs]
    kv2.push(1, [mx.nd.array(g, c) for g, c in zip(gs, ctxs)])
    model2.push(1, gs)
    srcs = [rsp_value(mx, rng, shape, 3000, c) for c in ctxs]
    kv2.push(1, [s[0] for s in srcs])
    model2.push(1, [s[1] for s in srcs])
    check_value(mx, kv2, model2, 1, shape, ctxs[1])
    outs = [mx.nd.sparse.zeros('row_sparse', shape, c) for c in ctxs] + [mx.nd.empty(shape, c) for c in ctxs]
    kv2.pull(1, out=outs, ignore_sparse=False)
    want_idx, want_val = model2.pull_rsp(1)
    for o in outs[:2]:
        assert np.array_equal(o.indices.asnumpy(), want_idx) and eq(o.data.asnumpy(), want_val)
    for o in outs[2:]:
        assert eq(o.asnumpy(), model2.pull(1))
