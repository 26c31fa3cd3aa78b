"""nag_mom_update, signsgd_update, signum_update, rmsprop_update, rmspropalex_update, ftml_update and
ftrl_update with a dense weight, dense states and a row_sparse gradient, on the GPU, bit for bit
against the reference, which densifies the gradient and runs the dense operator:
- every case of tests/golden/rsp_grad_update_ops.npz through mx.nd.<op> (out as the weight, as a
  separate array, and on slices that start off a 16-byte boundary);
- a 100 000 x 512 table against the gradient densified on the GPU followed by the dense operator;
- the refusals, which leave every operand and row count as it was and launch nothing;
- the reference's NAG, Signum, RMSProp, FTML and Ftrl classes on dense tables with row_sparse
  gradients (tests/golden/updater_trajectories_rsp_grad.npz, written by
  oracle/ref_python_rsp_grad_update.py) through a local updater, through the store's callback route
  on dense keys, and across a checkpoint."""
import os

import numpy as np
import pytest

import golden_rsp_grad_update_ops as GR
import golden_update_ops as GU
from ref_python_rsp_grad_update import trajectory_cases, states_of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def rsp(mx, vals, ids, shape, dtype=np.float32, ctx=None):
    ctx = ctx or mx.gpu(0)
    if len(ids) == 0:
        return mx.nd.sparse.zeros('row_sparse', shape, ctx, dtype)
    return mx.nd.sparse.row_sparse_array((vals.reshape((len(ids),) + tuple(shape[1:])), np.asarray(ids)),
                                         shape=shape, ctx=ctx, dtype=dtype)


def nnr(a):
    return a.indices.shape[0] if a.stype == 'row_sparse' else 0


def check(gold, name, out, states):
    assert GR.matches(gold, '%s|out' % name, out), (name, 'out')
    for i, s in enumerate(states):
        assert GR.matches(gold, '%s|s%d' % (name, i), s), (name, i)


@pytest.mark.parametrize("name", sorted(GR.CASES))
def test_rsp_grad_golden(mx, golden, name):
    case = GR.CASES[name]
    w, ids, vals, states = GR.inputs(case)
    shape = case['shape']
    wd = mx.nd.array(w, mx.gpu(0))
    sts = [mx.nd.array(s, mx.gpu(0)) for s in states]
    g = rsp(mx, vals, ids, shape)
    out = mx.nd.empty(shape, mx.gpu(0)) if case['distinct_out'] else wd
    getattr(mx.nd, case['op'])(wd, g, *sts, out=out, **case['params'])
    check(golden("rsp_grad_update_ops"), name, out.asnumpy(), [s.asnumpy() for s in sts])
    if case['distinct_out']:
        assert eq(wd.asnumpy(), w), "the weight must stay untouched"
    assert nnr(g) == len(ids)


@pytest.mark.parametrize("op", GR.OPS)
@pytest.mark.parametrize("sname", ['r1', 'r5'])
def test_rsp_grad_unaligned_slices(mx, golden, op, sname):
    """weight and states that start one row (4 or 20 bytes) past a 16-byte boundary: base[1:]"""
    name = sorted(n for n, c in GR.CASES.items()
                  if c['op'] == op and c['shape'] == GR.SHAPES[sname] and c['rows'] == 'ends')[-1]
    case = GR.CASES[name]
    w, ids, vals, states = GR.inputs(case)
    bases = [mx.nd.array(np.concatenate([a[:1], a]), mx.gpu(0)) for a in [w] + states]
    views = [b[1:] for b in bases]
    getattr(mx.nd, op)(views[0], rsp(mx, vals, ids, case['shape']), *views[1:], out=views[0], **case['params'])
    check(golden("rsp_grad_update_ops"), name, views[0].asnumpy(), [v.asnumpy() for v in views[1:]])
    for b, a in zip(bases, [w] + states):
        assert eq(b.asnumpy()[:1], a[:1]), "the row before the slice must stay untouched"


@pytest.mark.parametrize("op", GR.OPS)
def test_rsp_grad_large_equals_densified(mx, op):
    """100 000 x 512 with 10 % of the rows: the row_sparse pass equals the gradient cast to a dense
    array on the GPU (the reference's fallback, CastStorageRspDnsImpl) followed by the dense
    operator, bit for bit"""
    name = sorted(n for n, c in GR.CASES.items()
                  if c['op'] == op and c['shape'] == GR.SHAPES['r64'] and c['rows'] == 'all'
                  and not c['distinct_out'])[-1]
    params = GR.CASES[name]['params']               # clip, rescale and wd
    rows, L = 100000, 512
    shape = (rows, L)
    ins = [x.reshape(shape) for x in GU.inputs(dict(op=op, dtype='float32', n=rows * L))]
    ids = np.sort(np.random.default_rng(2024).choice(rows, rows // 10, replace=False))
    g = rsp(mx, ins[1][ids], ids, shape)
    a = [mx.nd.array(x, mx.gpu(0)) for x in [ins[0]] + ins[2:]]
    b = [mx.nd.array(x, mx.gpu(0)) for x in [ins[0]] + ins[2:]]
    getattr(mx.nd, op)(a[0], g, *a[1:], out=a[0], **params)
    gd = mx.nd.empty(shape, mx.gpu(0))
    g.copyto(gd)
    getattr(mx.nd, op)(b[0], gd, *b[1:], out=b[0], **params)
    for x, y in zip(a, b):
        assert eq(x.asnumpy(), y.asnumpy()), op
    cold = np.setdiff1d(np.arange(rows), ids)
    assert not eq(a[0].asnumpy()[cold], ins[0][cold]), "rows absent from the gradient move too"


# ------------------------------------------------------------------------------------ refusals
def _untouched(mx, call_, arrays, match=None):
    before = [(a.asnumpy().copy(), nnr(a)) for a in arrays]
    mx.nd.waitall()
    launches = mx.base.kernel_launch_count()
    with pytest.raises(mx.base.MXNetError, match=match):
        call_()
    assert mx.base.kernel_launch_count() == launches
    mx.nd.waitall()
    for a, (b, n) in zip(arrays, before):
        assert eq(a.asnumpy(), b) and nnr(a) == n


NSTATES = {'nag_mom_update': 1, 'signsgd_update': 0, 'signum_update': 1, 'rmsprop_update': 1,
           'rmspropalex_update': 3, 'ftml_update': 3, 'ftrl_update': 2}


def _kw(op):
    return dict(lr=0.1, t=1) if op == 'ftml_update' else dict(lr=0.1)


def ngpu():
    import torch
    return torch.cuda.device_count()


def test_rsp_grad_refusals(mx):
    rng = np.random.default_rng(9)
    rows, L = 12, 8
    shape = (rows, L)
    u = lambda *s: rng.uniform(-1, 1, s).astype(np.float32)  # noqa: E731
    g = rsp(mx, u(3, L), [0, 4, 11], shape)
    full = lambda: rsp(mx, u(rows, L), np.arange(rows), shape)  # noqa: E731
    empty = lambda: mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))  # noqa: E731
    dense = lambda s=shape, dt=np.float32, ctx=None: mx.nd.array(u(*s), ctx or mx.gpu(0), dt)  # noqa: E731
    for op, ns in NSTATES.items():
        f = getattr(mx.nd, op)
        kw = _kw(op)
        named = None if op == 'ftrl_update' else op   # Ftrl checks z / n against the weight first
        # a row_sparse weight, with row_sparse states that hold no rows or every row, or dense
        # states, or a dense gradient; Ftrl's all-row_sparse form is served
        if op != 'ftrl_update':
            for mk in (empty, full):
                w, sts = full(), [mk() for _ in range(ns)]
                _untouched(mx, lambda: f(w, g, *sts, out=w, **kw), [w] + sts,
                           match="Operator %s is not implemented for storage types" % op)
            w, sts, gd = full(), [dense() for _ in range(ns)], dense()
            _untouched(mx, lambda: f(w, g, *sts, out=w, **kw), [w] + sts, match=op)
            _untouched(mx, lambda: f(w, gd, *sts, out=w, **kw), [w, gd] + sts, match=op)
        # a dense weight with a row_sparse state, with either gradient
        if ns:
            w, sts, gd = dense(), [empty()] + [dense() for _ in range(ns - 1)], dense()
            for gg in (g, gd):
                _untouched(mx, lambda: f(w, gg, *sts, out=w, **kw), [w] + sts, match=named)
        # a float16 row_sparse gradient
        w, sts = dense(), [dense() for _ in range(ns)]
        g16 = rsp(mx, u(3, L), [0, 4, 11], shape, np.float16)
        _untouched(mx, lambda: f(w, g16, *sts, out=w, **kw), [w, g16] + sts, match="float32")
        # shapes: another row count, the same size in another shape, states and out of the same size
        for gs in (rsp(mx, u(3, L), [0, 4, 12], (rows + 1, L)), rsp(mx, u(2, 2 * L), [0, 5], (rows // 2, 2 * L))):
            _untouched(mx, lambda: f(w, gs, *sts, out=w, **kw), [w] + sts, match="shape mismatch")
        if ns:
            flat = [dense((rows * L,)) for _ in range(ns)]
            _untouched(mx, lambda: f(w, g, *flat, out=w, **kw), [w] + flat, match="shape mismatch")
        o = dense((rows * L,))
        _untouched(mx, lambda: f(w, g, *sts, out=o, **kw), [w, o] + sts, match="shape mismatch")
        # host operands
        wh = dense(ctx=mx.cpu())
        _untouched(mx, lambda: f(wh, g, *sts, out=wh, **kw), [wh] + sts)
        if ns:
            sh = [dense(ctx=mx.cpu())] + [dense() for _ in range(ns - 1)]
            _untouched(mx, lambda: f(w, g, *sh, out=w, **kw), [w] + sh, match="same GPU")
    # mp_nag_mom_update: 16-bit weights would need 16-bit row_sparse values
    w16, mom, w32 = dense(dt=np.float16), dense(), dense()
    g16 = rsp(mx, u(3, L), [0, 4, 11], shape, np.float16)
    for gg in (g, g16):
        _untouched(mx, lambda: mx.nd.mp_nag_mom_update(w16, gg, mom, w32, out=w16, lr=0.1, momentum=0.9),
                   [w16, mom, w32], match="mp_nag_mom_update: a row_sparse gradient")


@pytest.mark.skipif(ngpu() < 2, reason="needs 2 GPUs")
def test_rsp_grad_other_gpu_refused(mx):
    rng = np.random.default_rng(10)
    shape = (6, 4)
    w = mx.nd.array(rng.uniform(-1, 1, shape).astype(np.float32), mx.gpu(0))
    m = mx.nd.array(rng.uniform(-1, 1, shape).astype(np.float32), mx.gpu(1))
    g = rsp(mx, rng.uniform(-1, 1, (2, 4)).astype(np.float32), [1, 3], shape)
    _untouched(mx, lambda: mx.nd.nag_mom_update(w, g, m, out=w, lr=0.1, momentum=0.9), [w, m], match="same GPU")


# --------------------------------------------------------------------- optimizer trajectories
TRAJ = trajectory_cases()


def _optimizer(name):
    from compat import mxnet_optimizer_update as mxopt
    cls, kw = TRAJ[name]['opt']
    return getattr(mxopt, cls)(**kw)


def _check(gold, name, step, ws, states):
    for k, (w, st) in enumerate(zip(ws, states)):
        assert GR.matches(gold, "%s_step%d_w%d" % (name, step, k), w), (name, step, k)
        st = states_of(st)
        pre = "%s_step%d_w%d_s" % (name, step, k)
        assert len(st) == len({f.split('|')[0] for f in gold.files if f.startswith(pre)})
        for i, s in enumerate(st):
            assert GR.matches(gold, "%s_step%d_w%d_s%d" % (name, step, k, i), s.asnumpy()), (name, step, k, i)


@pytest.mark.parametrize("name", sorted(TRAJ))
def test_local_updater_trajectory(mx, golden, name):
    """update_on_kvstore=False: the local updater of <mirror of the reference class> with each
    device's row_sparse gradient and a dense weight"""
    from compat.mxnet_optimizer_update import get_updater
    gold = golden("updater_trajectories_rsp_grad")
    case = TRAJ[name]
    upd = get_updater(_optimizer(name))
    ws = [mx.nd.array(w, mx.gpu(0)) for w in case['w0']]
    for step, gs in enumerate(case['grads']):
        for k, ((ids, g), s) in enumerate(zip(gs, case['shapes'])):
            upd(k, rsp(mx, g, ids, s), ws[k])
        _check(gold, name, step, [w.asnumpy() for w in ws], [upd.states[k] for k in range(len(ws))])


def _store(mx, name, w0s):
    kv = mx.kv.create('device')
    for k, w in enumerate(w0s):
        kv.init(k, mx.nd.array(w, mx.gpu(0)))
    kv.set_optimizer(_optimizer(name))
    return kv


def _step(mx, kv, case, gs):
    """two halves of each gradient pushed from two sources (g/2 + g/2 == g exactly), dense pull"""
    keys = list(range(len(case['shapes'])))
    vals = []
    for (ids, g), s in zip(gs, case['shapes']):
        h = (g / np.float32(2)).astype(np.float32)
        vals.append([rsp(mx, h, ids, s), rsp(mx, h, ids, s)])
    kv.push(keys, vals)
    outs = [mx.nd.empty(s, mx.gpu(0)) for s in case['shapes']]
    kv.pull(keys, out=outs)
    return outs


@pytest.mark.parametrize("name", sorted(TRAJ))
def test_store_callback_trajectory(mx, golden, name, monkeypatch):
    """kv.set_optimizer(<mirror>) on dense keys: the store merges the row_sparse pushes and calls
    the optimizer back with (merged row_sparse gradient, stored dense weight)"""
    monkeypatch.setenv('B200KV_FUSED_OPTIMIZER', '0')
    gold = golden("updater_trajectories_rsp_grad")
    case = TRAJ[name]
    kv = _store(mx, name, case['w0'])
    for step, gs in enumerate(case['grads']):
        outs = _step(mx, kv, case, gs)
        _check(gold, name, step, [o.asnumpy() for o in outs], [kv._updater.states[k] for k in range(len(outs))])


@pytest.mark.parametrize("name", ['ftml', 'nag_mom'])
def test_rsp_grad_checkpoint_restart(mx, golden, tmp_path, name, monkeypatch):
    """save_optimizer_states(dump_optimizer=True) after step 2, a fresh store loads them: steps 3
    and 4 equal the uninterrupted trajectory (FTML's t resumes with the update count)"""
    monkeypatch.setenv('B200KV_FUSED_OPTIMIZER', '0')
    gold = golden("updater_trajectories_rsp_grad")
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
