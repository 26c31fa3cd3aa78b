"""The dense-gradient branches of the reference's AdaGrad and GroupAdaGrad on the GPU, bit for bit:

- square on float16, bfloat16, float32, float64, int32 and int64, mean over the last axis on the
  four float dtypes, and broadcast_add / _sub / _mul / _div / _maximum with an rhs of one value per
  row, against tests/golden/dense_adagrad_ops.npz (written from the reference's own code by
  oracle/golden_dense_adagrad.py) and its restatement; through the operators, mx.nd.square /
  mx.nd.mean, NDArray.mean, `/` and mx.nd.maximum; in place (`state[:] += mean(...)`,
  `x[:] /= row`);
- refusals raise and leave `out` as it was;
- the tests/compat mirror of the two classes against the trajectories the reference's own classes
  reach (tests/golden/updater_trajectories_dense_adagrad.npz): through the store's per-key callback
  (kv.set_optimizer, two pushed values per key) and through a local updater; and its row_sparse
  branches against the existing row_sparse trajectories.

NaN compares as NaN (the GPU writes its canonical NaN)."""
import numpy as np
import pytest

import golden_dense_adagrad as GD
import golden_ndarray_ops as G
import ref_python_dense_adagrad as RPD

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


@pytest.fixture(scope="module")
def fixture():
    d = np.load(G.os.path.join(GD.GOLD, "dense_adagrad_ops.npz"))
    return {str(n): (s, h) for n, s, h in zip(d['names'], d['sha256'], d['head'])}


def up(mx, x, dt):
    if dt == 'bfloat16':
        return mx.nd.array(G.bf16_to_f32(x), mx.gpu(0), dtype='bfloat16')
    return mx.nd.array(np.ascontiguousarray(x, G.STORE[dt]), mx.gpu(0), dtype=G.STORE[dt])


def down(nd, dt):
    x = nd.asnumpy()
    if dt == 'bfloat16':
        return (x.view(np.uint32) >> 16).astype(np.uint16)
    return x


def check(got, want, dt, what):
    """bit equality with NaN positions and the shape compared, the first differences named"""
    if G.same(got, want, dt):
        return
    a, b = np.ravel(G.canon(got, dt)), np.ravel(G.canon(want, dt))
    if np.shape(got) != np.shape(want):
        pytest.fail('%s: shape %s, want %s' % (what, np.shape(got), np.shape(want)))
    u = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.itemsize]
    bad = np.nonzero(a.view(u) != b.view(u))[0]
    lines = ['%s: %d of %d elements differ' % (what, len(bad), b.size)]
    for i in bad[:6]:
        lines.append('  [%d] got %r want %r' % (i, a[i], b[i]))
    pytest.fail('\n'.join(lines))


def check_fixture(fixture, name, got, dt):
    sha, head = fixture[name]
    got = np.ravel(got)
    assert np.array_equal(G.head_bytes(got, dt), head), name + ': head differs from the reference'
    assert np.array_equal(G.sha256(got, dt), sha), name + ': differs from the reference'


# --------------------------------------------------------------------------------- operators
@pytest.mark.parametrize("case", GD.square_cases(), ids=lambda c: c[0])
def test_square(mx, fixture, case):
    name, dt, n = case
    a = GD.inputs('square', case)[0]
    want = GD.restate('square', case)
    A = up(mx, a, dt)
    got = down(mx.nd._invoke('square', [A]), dt)
    check(got, want, dt, name)
    check_fixture(fixture, name, got, dt)
    check(down(mx.nd.square(A), dt), want, dt, name + ' nd.square')
    check(down(A, dt), a, dt, name + ' input kept')
    mx.nd.square(A, out=A)
    check(down(A, dt), want, dt, name + ' in place')


@pytest.mark.parametrize("case", GD.mean_cases(), ids=lambda c: c[0])
def test_mean(mx, fixture, case):
    name, dt, shape, axis, keepdims, _ = case
    x = GD.inputs('mean', case)[0]
    want = GD.restate('mean', case)
    X = up(mx, x, dt)
    got = down(mx.nd._invoke('mean', [X], axis=axis, keepdims=keepdims), dt)
    check(got, want, dt, name)
    check_fixture(fixture, name, got, dt)
    keep = keepdims == 'True'
    check(down(mx.nd.mean(X, axis=-1, keepdims=keep), dt), want, dt, name + ' nd.mean')
    check(down(X.mean(axis=len(shape) - 1, keepdims=keep), dt), want, dt, name + ' NDArray.mean')
    O = up(mx, np.zeros(want.shape, G.STORE[dt]), dt)
    mx.nd.mean(X, axis=(len(shape) - 1,), keepdims=keep, out=O)
    check(down(O, dt), want, dt, name + ' out=')
    check(down(X, dt), x, dt, name + ' input kept')


@pytest.mark.parametrize("case", GD.broadcast_cases(), ids=lambda c: c[0])
def test_row_broadcast(mx, fixture, case):
    name, op, dt, shape = case
    a, b = GD.inputs('broadcast', case)
    want = GD.restate('broadcast', case)
    A, B = up(mx, a, dt), up(mx, b, dt)
    got = down(mx.nd._invoke(op, [A, B]), dt)
    check(got, want, dt, name)
    check_fixture(fixture, name, got, dt)
    # this package's NDArray lowers `a + b`, `a - b`, `a * b` to the equal-shape _plus / _minus / _mul;
    # `a / b` is broadcast_div, which the reference's GroupAdaGrad calls with a row operand
    if op == 'broadcast_div':
        check(down(A / B, dt), want, dt, name + ' a / row')
    elif op == 'broadcast_maximum':
        check(down(mx.nd.maximum(A, B), dt), want, dt, name + ' nd.maximum')
    check(down(B, dt), b, dt, name + ' rhs kept')
    if op == 'broadcast_div':
        A[:] /= B                                              # x[:] /= row writes x
        check(down(A, dt), want, dt, name + ' x[:] /= row')
    else:
        mx.nd._invoke(op, [A, B], out=A)
        check(down(A, dt), want, dt, name + ' in place')


@pytest.mark.parametrize("dt", G.FLOATS)
def test_history_accumulates_in_place(mx, dt):
    """state[:] += mean(square(g), axis=1, keepdims=True), GroupAdaGrad's history step"""
    g = GD.mean_operand('hist|' + dt, dt, (300, 45), 'signed')
    h = GD.mean_operand('hist0|' + dt, dt, (300, 1), 'mixed')
    want = GD.row_broadcast('broadcast_add', h, GD.mean_rows(GD.square(g, dt), dt).reshape(300, 1), dt)
    H = up(mx, h, dt)
    H[:] += mx.nd.mean(mx.nd.square(up(mx, g, dt)), axis=1, keepdims=True)
    check(down(H, dt), want, dt, 'state[:] += mean(square(g))')


# --------------------------------------------------------------------------------- refusals
def _refused(mx, call, out, match):
    before = out.asnumpy().copy()
    with pytest.raises(mx.base.MXNetError, match=match):
        call()
    mx.nd.waitall()
    after = out.asnumpy()
    assert np.array_equal(np.ascontiguousarray(after).view(np.uint8), np.ascontiguousarray(before).view(np.uint8))


def test_refusals_leave_out_untouched(mx):
    g = mx.gpu(0)
    rng = np.random.default_rng(5)
    f = lambda s, dt=np.float32: mx.nd.array(rng.uniform(1, 2, s).astype(dt), g, dt)  # noqa: E731
    x, o = f((4, 5)), f((4,))
    mean = lambda out=o, data=x, **kw: mx.nd._invoke('mean', [data], out=out, **kw)  # noqa: E731
    for axis in ('0', '-2', '()', 'None', '(0, 1)', '(1, 1)', '5'):
        _refused(mx, lambda: mean(axis=axis), o, 'only the last axis')
    _refused(mx, lambda: mean(), o, 'only the last axis')
    _refused(mx, lambda: mean(axis='1', exclude='True'), o, 'exclude=True')
    _refused(mx, lambda: mean(axis='0', data=f((5,)), out=f((1,))), o, 'rank 2 or more')
    for dt in (np.int32, np.int64):
        io = f((4,), dt)
        _refused(mx, lambda: mean(axis='1', data=f((4, 5), dt), out=io), io, 'float16, bfloat16')
    host = mx.nd.array(np.ones((4, 5), np.float32), mx.cpu(0))
    _refused(mx, lambda: mean(axis='1', data=host), o, 'GPU arrays only')
    _refused(mx, lambda: mean(axis='1', out=mx.nd.array(np.ones(4, np.float32), mx.cpu(0))), o, 'same GPU')
    rsp = mx.nd.row_sparse_array((np.ones((1, 5), np.float32), np.array([2], np.int64)), shape=(4, 5), ctx=g)
    _refused(mx, lambda: mean(axis='1', data=rsp), o, 'dense arrays only')
    o2 = f((4, 1))
    _refused(mx, lambda: mean(axis='1', out=o2), o2, 'wrong shape')
    _refused(mx, lambda: mean(axis='1', keepdims='True'), o, 'wrong shape')
    o16 = f((4,), np.float16)
    _refused(mx, lambda: mean(axis='1', out=o16), o16, 'dtype')
    _refused(mx, lambda: mean(axis='1', keepdim='True'), o, "Cannot find argument 'keepdim'")
    # the row broadcast takes exactly lhs.shape[:-1] + (1,); the rest keeps today's refusal
    out = f((4, 5))
    for op in ('broadcast_add', 'broadcast_sub', 'broadcast_mul', 'broadcast_div', 'broadcast_maximum'):
        for lhs, rhs in (((4, 5), (1, 5)), ((4, 5), (4, 5, 1)), ((4, 5), (4,)), ((4, 5), (2, 1)),
                         ((4, 1), (4, 5)), ((5,), (1,))):
            _refused(mx, lambda: mx.nd._invoke(op, [f(lhs), f(rhs)], out=out), out, 'would broadcast')
    for dt in (np.int32, np.int64):
        iout = f((4, 5), dt)
        _refused(mx, lambda: mx.nd._invoke('broadcast_div', [f((4, 5), dt), f((4, 1), dt)], out=iout), iout,
                 'integer division')
    _refused(mx, lambda: mx.nd._invoke('broadcast_div', [x, f((4, 1), np.float16)], out=out), out, 'dtype')
    _refused(mx, lambda: mx.nd._invoke('broadcast_mul', [x, mx.nd.array(np.ones((4, 1), np.float32), mx.cpu(0))],
                                       out=out), out, 'same GPU')
    _refused(mx, lambda: mx.nd._invoke('broadcast_div', [x, f((4, 1))], out=f((4, 4))), out, 'shape mismatch')
    _refused(mx, lambda: mx.nd._invoke('square', [x], out=host), host, 'GPU arrays only')


# --------------------------------------------------------------------------------- optimizers
TRAJ = RPD.trajectory_cases()


def _optimizer(name):
    from compat import mxnet_optimizer_dense_adagrad as mxopt
    cls, kw = TRAJ[name]['opt']
    return getattr(mxopt, cls)(**kw)


def _halves(mx, g, dtype):
    h = (g / g.dtype.type(2)).astype(g.dtype)
    return [mx.nd.array(h, mx.gpu(0), dtype) for _ in range(2)]


def _eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("name", sorted(TRAJ))
def test_store_callback_trajectory(mx, golden, name):
    """kv.set_optimizer(<mirror of the reference class>): two values per key, 4 pushpulls, the
    store's per-key updater callback running the operators; weights after every step"""
    gold = golden("updater_trajectories_dense_adagrad")
    case = TRAJ[name]
    dt = case['dtype']
    keys = list(range(len(case['shapes'])))
    kv = mx.kv.create('device')
    for k in keys:
        kv.init(k, mx.nd.array(case['w0'][k], mx.gpu(0), dt))
    kv.set_optimizer(_optimizer(name))
    outs = [mx.nd.empty(s, mx.gpu(0), dt) for s in case['shapes']]
    for step, gs in enumerate(case['grads']):
        kv.pushpull(keys, [_halves(mx, gk, dt) for gk in gs], out=outs)
        for k in keys:
            assert _eq(outs[k].asnumpy(), gold["%s_step%d_w%d" % (name, step, k)]), (name, step, k)


@pytest.mark.parametrize("name", sorted(TRAJ))
def test_local_updater_trajectory(mx, golden, name):
    """update_on_kvstore=False: in-place pushpull of the two values, then the local updater;
    weights and histories after every step"""
    from compat import mxnet_optimizer_dense_adagrad as mxopt
    gold = golden("updater_trajectories_dense_adagrad")
    case = TRAJ[name]
    dt = case['dtype']
    keys = list(range(len(case['shapes'])))
    kv = mx.kv.create('device')
    for k in keys:
        kv.init(k, mx.nd.zeros(case['shapes'][k], mx.gpu(0), dt))
    upd = mxopt.get_updater(_optimizer(name))
    ws = [mx.nd.array(w, mx.gpu(0), dt) for w in case['w0']]
    for step, gs in enumerate(case['grads']):
        vals = [_halves(mx, gk, dt) for gk in gs]
        for k in keys:
            kv.pushpull(k, vals[k], out=vals[k])
            upd(k, vals[k][0], ws[k])
        for k in keys:
            key = "%s_step%d_w%d" % (name, step, k)
            assert _eq(ws[k].asnumpy(), gold[key]), key
            assert _eq(RPD.history(upd.states[k]).asnumpy(), gold[key + "_s0"]), key


def test_row_sparse_branches_unchanged(mx, golden):
    """the mirror classes' row_sparse branches still reach the existing row_sparse trajectories:
    GroupAdaGrad on dense tables with row_sparse gradients, AdaGrad through _sparse_adagrad_update"""
    import ref_python_group_adagrad as RPG
    from compat import mxnet_optimizer_dense_adagrad as mxopt
    gold = golden("updater_trajectories_group_adagrad")
    case = RPG.trajectory_cases()['dns_clip']
    upd = mxopt.get_updater(mxopt.GroupAdaGrad(**case['opt']))
    ws = [mx.nd.array(w, mx.gpu(0)) for w in case['w0']]
    for step, gs in enumerate(case['grads']):
        for k, (ids, g) in enumerate(gs):
            grad = mx.nd.row_sparse_array((g, ids), shape=case['shapes'][k], ctx=mx.gpu(0))
            upd(k, grad, ws[k])
        for k in range(len(ws)):
            key = "dns_clip_step%d_w%d" % (step, k)
            assert _eq(ws[k].asnumpy(), gold[key]), key
            assert _eq(upd.states[k].asnumpy(), gold[key + "_s0"]), key
    # AdaGrad's row_sparse branch is one _sparse_adagrad_update with the optimizer's parameters
    opt = mxopt.AdaGrad(learning_rate=0.1, clip_gradient=0.5)
    w0 = np.random.default_rng(7).uniform(-1, 1, (10, 4)).astype(np.float32)
    g = np.random.default_rng(8).uniform(-1, 1, (3, 4)).astype(np.float32)
    ids = np.array([1, 4, 9], np.int64)
    W = mx.nd.array(w0, mx.gpu(0))
    state = opt.create_state(0, W)
    opt.update(0, W, mx.nd.row_sparse_array((g, ids), shape=(10, 4), ctx=mx.gpu(0)), state)
    W2 = mx.nd.array(w0, mx.gpu(0))
    h2 = mx.nd.zeros((10, 4), mx.gpu(0))
    mx.nd.sparse.adagrad_update(W2, mx.nd.row_sparse_array((g, ids), shape=(10, 4), ctx=mx.gpu(0)), h2,
                                out=W2, lr=0.1, wd=0.0, epsilon=1e-7, rescale_grad=1.0, clip_gradient=0.5)
    assert _eq(W.asnumpy(), W2.asnumpy()) and _eq(state.asnumpy(), h2.asnumpy())
    rows = np.setdiff1d(np.arange(10), ids)
    assert _eq(W.asnumpy()[rows], w0[rows])
