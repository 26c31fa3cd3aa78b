"""The NAG / Signum / RMSProp / FTML / Ftrl operators on the GPU, bit for bit against the reference's
own CPU code: every case of tests/golden/update_ops.npz through mx.nd.<op> (out as the weight, as a
separate array, and on unaligned slices), and the reference optimizers' trajectories
(tests/golden/updater_trajectories_ext.npz, written by oracle/ref_python_update.py) through the
store's callback route, through update_on_kvstore=False local updaters, and across a checkpoint."""
import os

import numpy as np
import pytest

import golden_update_ops as GU
from ref_python_update import trajectory_cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def to_gpu(mx, a, dtype='float32'):
    if dtype == 'bfloat16':
        return mx.nd.array(GU.bf16_bits_to_f32(a), mx.gpu(0), 'bfloat16')
    return mx.nd.array(a, mx.gpu(0), a.dtype)


def from_gpu(nd, dtype='float32'):
    a = nd.asnumpy()
    return GU.to_bf16_bits(a) if dtype == 'bfloat16' else a


def check_case(g, name, case, out, states):
    for tag, a in [('out', out)] + [('s%d' % i, s) for i, s in enumerate(states)]:
        a = np.ascontiguousarray(a)
        if case['n'] <= GU.FULL_MAX:
            assert eq(a, g['%s|%s' % (name, tag)]), (name, tag)
        else:
            assert eq(a[:GU.HEAD], g['%s|%s|head' % (name, tag)]), (name, tag)
            assert eq(GU.digest(a), g['%s|%s|sha256' % (name, tag)]), (name, tag)


@pytest.mark.parametrize("name", sorted(GU.CASES))
def test_update_op_golden(mx, golden, name):
    case = GU.CASES[name]
    g = golden("update_ops")
    ins = GU.inputs(case)
    dt = case['dtype']
    nds = [to_gpu(mx, a, dt) for a in ins[:2]] + [to_gpu(mx, a) for a in ins[2:]]
    out = mx.nd.empty(nds[0].shape, mx.gpu(0), nds[0].dtype) if case['distinct_out'] else nds[0]
    getattr(mx.nd, case['op'])(*nds, out=out, **case['params'])
    check_case(g, name, case, from_gpu(out, dt), [s.asnumpy() for s in nds[2:]])
    if case['distinct_out']:
        assert eq(from_gpu(nds[0], dt), ins[0]), "the weight must stay untouched"


@pytest.mark.parametrize("op", GU.OPS)
def test_update_op_unaligned_slice(mx, golden, op):
    """operands that start 1 element past a 16-byte boundary: the scalar path over the whole tensor"""
    name = sorted(n for n, c in GU.CASES.items() if c['op'] == op and c['n'] == 4097 and not c['distinct_out'])[0]
    case = GU.CASES[name]
    g = golden("update_ops")
    ins = GU.inputs(case)
    dt = case['dtype']
    bases, views = [], []
    for i, a in enumerate(ins):
        pad = np.concatenate([a[:1], a])
        base = to_gpu(mx, pad, dt if i < 2 else 'float32')
        bases.append(base)
        views.append(base[1:])
    getattr(mx.nd, op)(*views, out=views[0], **case['params'])
    check_case(g, name, case, from_gpu(views[0], dt), [v.asnumpy() for v in views[2:]])
    assert eq(from_gpu(bases[0], dt)[:1], ins[0][:1]), "the element before the slice must stay untouched"


def _weight_untouched(mx, call, w):
    before = w.asnumpy().copy()
    with pytest.raises(mx.base.MXNetError):
        call()
    assert eq(w.asnumpy(), before)


def test_update_op_errors(mx):
    rng = np.random.default_rng(3)
    a = lambda n=64, dt=np.float32: mx.nd.array(rng.uniform(-1, 1, n).astype(dt), mx.gpu(0), dt)  # noqa: E731
    w, g, s = a(), a(), a()
    rsp = mx.nd.sparse.row_sparse_array((rng.uniform(-1, 1, (2, 8)).astype(np.float32), np.array([1, 3])),
                                        shape=(8, 8), ctx=mx.gpu(0))
    w2 = mx.nd.array(rng.uniform(-1, 1, (8, 8)).astype(np.float32), mx.gpu(0))
    _weight_untouched(mx, lambda: mx.nd.ftrl_update(w2, rsp, a(64), a(64), out=w2, lr=0.1), w2)
    w16 = a(dt=np.float16)
    for op, extra in [('rmsprop_update', 1), ('nag_mom_update', 1), ('ftml_update', 3), ('ftrl_update', 2),
                      ('signum_update', 1), ('signsgd_update', 0), ('rmspropalex_update', 3)]:
        states = [a() for _ in range(extra)]
        kw = dict(lr=0.1, t=1) if op == 'ftml_update' else dict(lr=0.1)
        _weight_untouched(mx, lambda: getattr(mx.nd, op)(w16, a(dt=np.float16), *states, out=w16, **kw), w16)
    _weight_untouched(mx, lambda: mx.nd.nag_mom_update(w, g, s, out=w, momentum=0.9), w)
    _weight_untouched(mx, lambda: mx.nd.ftml_update(w, g, a(), a(), a(), out=w, lr=0.1), w)
    _weight_untouched(mx, lambda: mx.nd.rmsprop_update(w, a(63), s, out=w, lr=0.1), w)
    _weight_untouched(mx, lambda: mx.nd.ftml_update(w, g, a(), a(), a(), out=w, lr=0.1, t=1, beta1=1.5), w)
    _weight_untouched(mx, lambda: mx.nd.mp_nag_mom_update(w, g, s, a(), out=w, lr=0.1), w)


# --------------------------------------------------------------------- optimizer trajectories
TRAJ = trajectory_cases()


def _optimizer(name):
    from compat import mxnet_optimizer_update as mxopt
    cls, kw = TRAJ[name]['opt']
    return getattr(mxopt, cls)(**kw)


def _halves(mx, g, dtype):
    h = (g / g.dtype.type(2)).astype(g.dtype)
    return [mx.nd.array(h, mx.gpu(0), dtype) for _ in range(2)]


@pytest.mark.parametrize("name", sorted(TRAJ))
def test_store_callback_trajectory(mx, golden, name):
    """kv.set_optimizer(<mirror of the reference class>): two values per key, 4 pushpulls, the
    store's per-key updater callback running the operators; weights after every step"""
    gold = golden("updater_trajectories_ext")
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
            assert eq(outs[k].asnumpy(), gold["%s_step%d_w%d" % (name, step, k)]), (name, step, k)


@pytest.mark.parametrize("name", sorted(TRAJ))
def test_local_updater_trajectory(mx, golden, name):
    """update_on_kvstore=False: in-place pushpull of the two values, then the local updater"""
    from compat import mxnet_optimizer_update as mxopt
    gold = golden("updater_trajectories_ext")
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
            assert eq(ws[k].asnumpy(), gold["%s_step%d_w%d" % (name, step, k)]), (name, step, k)


def test_ftml_checkpoint_restart(mx, golden, tmp_path):
    """save_optimizer_states(dump_optimizer=True) after step 2, a fresh store loads them: FTML's t
    (the update count) resumes, so steps 3 and 4 equal the uninterrupted trajectory"""
    gold = golden("updater_trajectories_ext")
    case = TRAJ['ftml']
    keys = list(range(len(case['shapes'])))
    fname = os.path.join(str(tmp_path), "ftml.states")
    kv = mx.kv.create('device')
    for k in keys:
        kv.init(k, mx.nd.array(case['w0'][k], mx.gpu(0)))
    kv.set_optimizer(_optimizer('ftml'))
    outs = [mx.nd.empty(s, mx.gpu(0)) for s in case['shapes']]
    for gs in case['grads'][:2]:
        kv.pushpull(keys, [_halves(mx, gk, 'float32') for gk in gs], out=outs)
    kv.save_optimizer_states(fname, dump_optimizer=True)
    weights = [o.asnumpy() for o in outs]
    kv2 = mx.kv.create('device')
    for k in keys:
        kv2.init(k, mx.nd.array(weights[k], mx.gpu(0)))
    kv2.set_optimizer(_optimizer('ftml'))
    kv2.load_optimizer_states(fname)
    for step, gs in list(enumerate(case['grads']))[2:]:
        kv2.pushpull(keys, [_halves(mx, gk, 'float32') for gk in gs], out=outs)
        for k in keys:
            assert eq(outs[k].asnumpy(), gold["ftml_step%d_w%d" % (step, k)]), (step, k)
