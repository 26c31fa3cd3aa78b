"""The arithmetic of the reference's Adamax, Nadam and AdaDelta optimizers on the GPU, bit for bit:

- broadcast_add / _sub / _mul / _div / _maximum, _div_scalar, abs and clip on float16, bfloat16,
  float32, float64, int32 and int64 (division on the float types) against tests/golden/arith_ops.npz,
  written from the reference's own functors by oracle/golden_arith_ops.py, and its restatement;
  through the operators, the NDArray methods (`/`, `/=`) and mx.nd.clip / abs / maximum;
- refusals (operands that would broadcast, integer division, row_sparse and host operands, an
  unknown clip argument, a missing bound) raise and leave `out` as it was;
- the tests/compat mirror of the three classes against the trajectories the reference's own classes
  reach (tests/golden/updater_trajectories_arith.npz, from oracle/ref_python_arith.py): through the
  store's per-key callback (kv.set_optimizer, two pushed values per key) and through a local
  updater (update_on_kvstore=False), float32 and float16 with multi_precision; AdaDelta's gradient
  after each step too, since it rescales the caller's array in place.

NaN compares as NaN (the GPU writes its canonical NaN)."""
import numpy as np
import pytest

import golden_arith_ops as GA
import golden_ndarray_ops as G
import ref_python_arith as RPA

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


@pytest.fixture(scope="module")
def fixture():
    d = np.load(G.os.path.join(GA.GOLD, "arith_ops.npz"))
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
    """bit equality with NaN positions compared, the first differences named"""
    if G.same(got, want, dt):
        return
    a, b = G.canon(got, dt), G.canon(want, dt)
    u = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.itemsize]
    bad = np.nonzero(a.view(u) != b.view(u))[0] if a.shape == b.shape else []
    lines = ['%s: %d of %d elements differ' % (what, len(bad), b.size)]
    for i in bad[:6]:
        lines.append('  [%d] got %r want %r' % (i, a[i], b[i]))
    pytest.fail('\n'.join(lines))


def check_fixture(fixture, name, got, dt):
    sha, head = fixture[name]
    assert np.array_equal(G.head_bytes(got, dt), head), name + ': head differs from the reference'
    assert np.array_equal(G.sha256(got, dt), sha), name + ': differs from the reference'


def seeded_out(mx, n, dt):
    return up(mx, G.operands('arith-out|%s|%d' % (dt, n), n, dt, 'plus')[0], dt)


# --------------------------------------------------------------------------------- operators
METHOD = {'broadcast_add': '__add__', 'broadcast_sub': '__sub__', 'broadcast_mul': '__mul__',
          'broadcast_div': '__truediv__'}


@pytest.mark.parametrize("case", GA.array_cases(), ids=lambda c: c[0])
def test_array_operator(mx, fixture, case):
    name, op, dt, n = case
    ins = GA.inputs('array', case)
    want = GA.restate('array', case)
    nds = [up(mx, a, dt) for a in ins]
    got = down(mx.nd._invoke(op, nds), dt)
    check(got, want, dt, name)
    check_fixture(fixture, name, got, dt)
    O = seeded_out(mx, n, dt)
    mx.nd._invoke(op, nds, out=O)                              # a distinct out
    check(down(O, dt), want, dt, name + ' out=')
    for nd, a in zip(nds, ins):
        check(down(nd, dt), a, dt, name + ' input kept')
    if op in METHOD:
        check(down(getattr(nds[0], METHOD[op])(nds[1]), dt), want, dt, name + ' ' + METHOD[op])
    elif op == 'broadcast_maximum':
        check(down(mx.nd.maximum(*nds), dt), want, dt, name + ' nd.maximum')
    else:
        check(down(mx.nd.abs(nds[0]), dt), want, dt, name + ' nd.abs')
    if op == 'broadcast_div':
        R = nds[0].__itruediv__(nds[1])
        assert R is nds[0]
        check(down(nds[0], dt), want, dt, name + ' /=')
    else:
        mx.nd._invoke(op, nds, out=nds[0])                     # out = the first input
        check(down(nds[0], dt), want, dt, name + ' in place')


@pytest.mark.parametrize("case", GA.scalar_cases(), ids=lambda c: c[0])
def test_div_scalar(mx, fixture, case):
    name, dt, s = case
    a = GA.inputs('scalar', case)[0]
    want = GA.restate('scalar', case)
    A = up(mx, a, dt)
    got = down(mx.nd._invoke('_div_scalar', [A], scalar=s), dt)
    check(got, want, dt, name)
    check_fixture(fixture, name, got, dt)
    if repr(float(s)) == s:                                    # the method formats float(s) with str()
        check(down(A / float(s), dt), want, dt, name + ' /')
        A /= float(s)
        check(down(A, dt), want, dt, name + ' /=')


@pytest.mark.parametrize("case", GA.clip_cases(), ids=lambda c: c[0])
def test_clip(mx, fixture, case):
    name, dt, lo, hi, n = case
    a = GA.inputs('clip', case)[0]
    want = GA.restate('clip', case)
    A = up(mx, a, dt)
    got = down(mx.nd._invoke('clip', [A], a_min=lo, a_max=hi), dt)
    check(got, want, dt, name)
    check_fixture(fixture, name, got, dt)
    if repr(float(lo)) == lo and repr(float(hi)) == hi:
        check(down(mx.nd.clip(A, float(lo), float(hi)), dt), want, dt, name + ' nd.clip')
    mx.nd.clip(A, lo, hi, out=A)
    check(down(A, dt), want, dt, name + ' in place')


@pytest.mark.parametrize("dt", G.DTYPES)
def test_views_and_aliasing(mx, dt):
    """x[:] op= y on a view of the whole array, and an operator whose two inputs are one array"""
    a, b = GA.operands('view|%s' % dt, 'broadcast_maximum', dt, 4099)
    A, B = up(mx, a, dt), up(mx, b, dt)
    A[:] = mx.nd.maximum(A[:], B)
    check(down(A, dt), GA.maximum(a, b, dt), dt, 'x[:] = maximum(x[:], y)')
    A = up(mx, a, dt)
    mx.nd._invoke('broadcast_maximum', [A, A], out=A)
    check(down(A, dt), a, dt, 'maximum(a, a)')
    if dt in G.FLOATS:
        A = up(mx, a, dt)
        A[:] /= B
        check(down(A, dt), GA.div(a, b, dt), dt, 'x[:] /= y')


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
    rng = np.random.default_rng(3)
    f = lambda s, dt=np.float32: mx.nd.array(rng.uniform(1, 2, s).astype(dt), g, dt)  # noqa: E731
    a, b, out = f((4, 5)), f((4, 5)), f((4, 5))
    for op in ('broadcast_add', 'broadcast_sub', 'broadcast_mul', 'broadcast_div', 'broadcast_maximum'):
        _refused(mx, lambda: mx.nd._invoke(op, [a, f((1, 5))], out=out), out, 'would broadcast')
        _refused(mx, lambda: mx.nd._invoke(op, [f((5, 4)), a], out=out), out, 'would broadcast')
    for dt in (np.int32, np.int64):
        ia, ib, iout = f((4, 5), dt), f((4, 5), dt), f((4, 5), dt)
        _refused(mx, lambda: mx.nd._invoke('broadcast_div', [ia, ib], out=iout), iout, 'integer division')
        _refused(mx, lambda: mx.nd._invoke('_div_scalar', [ia], out=iout, scalar=2.0), iout,
                 'integer division')
    _refused(mx, lambda: mx.nd._invoke('clip', [a], out=out, a_min=0.0, a_max=1.0, a_mx=2), out,
             "Cannot find argument 'a_mx'")
    _refused(mx, lambda: mx.nd._invoke('clip', [a], out=out, a_min=0.0), out, 'Required parameter a_max')
    _refused(mx, lambda: mx.nd._invoke('_div_scalar', [a], out=out), out, 'Required parameter scalar')
    _refused(mx, lambda: mx.nd._invoke('_div_scalar', [a], out=out, scalar='x'), out, 'cannot parse')
    host = mx.nd.array(np.ones((4, 5), np.float32), mx.cpu(0))
    _refused(mx, lambda: mx.nd._invoke('broadcast_mul', [a, host], out=out), out, 'same GPU')
    _refused(mx, lambda: mx.nd._invoke('abs', [a], out=host), host, 'GPU arrays only')
    rsp = mx.nd.row_sparse_array((np.ones((1, 5), np.float32), np.array([2], np.int64)), shape=(4, 5), ctx=g)
    _refused(mx, lambda: mx.nd._invoke('broadcast_add', [a, rsp], out=out), out, 'dense arrays only')
    _refused(mx, lambda: mx.nd._invoke('clip', [rsp], out=out, a_min=0.0, a_max=1.0), out, 'dense arrays only')
    _refused(mx, lambda: mx.nd._invoke('broadcast_add', [a, f((4, 5), np.float16)], out=out), out, 'dtype')
    check(down(a, 'float32'), a.asnumpy(), 'float32', 'operand kept')


# --------------------------------------------------------------------------------- optimizers
TRAJ = RPA.trajectory_cases()


def _optimizer(name):
    from compat import mxnet_optimizer_arith as mxopt
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
    gold = golden("updater_trajectories_arith")
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
    weights, and AdaDelta's rescaled gradient, after every step"""
    from compat import mxnet_optimizer_arith as mxopt
    gold = golden("updater_trajectories_arith")
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
            assert _eq(ws[k].asnumpy(), gold["%s_step%d_w%d" % (name, step, k)]), (name, step, k)
            if case['opt'][0] == 'AdaDelta':
                assert _eq(vals[k][0].asnumpy(), gold["%s_step%d_g%d" % (name, step, k)]), (name, step, k)
