"""CUDA store (fused reduce + optimizer step) against trajectories produced by the REFERENCE's own
Python front-end over the reference's own compiled operators (tests/golden/updater_trajectories.npz,
written by oracle/gen_golden.py through oracle/ref_python.py: python/mxnet/optimizer/optimizer.py
Updater / SGD / Adam / Test + lr_scheduler.FactorScheduler, src/operator/optimizer_op.cc
FCompute<cpu>). No oracle in between; weights bit for bit after every case's last step -- update
counts, multipliers, the scheduler call, Adam's bias correction and the python-repr -> dmlc::stof
scalar route (std::stod for Test's `grad * rescale_grad`, a _mul_scalar) all have to agree for that."""
import numpy as np
import pytest

from gen_golden import updater_cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


STORE_CASES = sorted(n for n, c in updater_cases().items() if c['model'])


@pytest.mark.parametrize("fused", ['1', '0'])
@pytest.mark.parametrize("name", STORE_CASES)
def test_store_trajectory_golden(mx, golden, name, fused, monkeypatch):
    """fused = '1': the optimizer step inside the reduce kernel (native replay of the bookkeeping);
    fused = '0': the reference's callback route (store -> Updater -> optimizer operators)"""
    from compat import mxnet_optimizer as mxopt
    monkeypatch.setenv('B200KV_FUSED_OPTIMIZER', fused)
    g = golden("updater_trajectories")
    case = updater_cases()[name]
    shapes, keys = case['shapes'], list(range(len(case['shapes'])))
    cls, kw = case['opt']
    kw = dict(kw)
    if 'sched' in case:
        class Sched(object):                 # lr_scheduler.py FactorScheduler(step=2, factor=0.5)'s values
            base_lr = case['lr_at'][0]

            def __call__(self, num_update):
                return case['lr_at'][min(max(num_update, 1), len(case['lr_at'])) - 1]
        kw['lr_scheduler'] = Sched()
    if cls == 'Test':
        # fused: the package's record; callback: the reference's Test class, whose update() runs
        # `weight += grad * rescale_grad` through _mul_scalar and _plus
        opt = mx.optimizer.Test(**kw) if fused == '1' else mxopt.Test(**kw)
    else:
        opt = getattr(mxopt, cls)(**kw)
    if case.get('lr_mult'):
        opt.set_lr_mult(case['lr_mult'])
    if case.get('wd_mult'):
        opt.set_wd_mult(case['wd_mult'])
    kv = mx.kv.create('device')
    for k in keys:
        kv.init(k, mx.nd.array(case['w0'][k], mx.gpu(0)))
    kv.set_optimizer(opt)
    outs = [mx.nd.empty(s, mx.gpu(0)) for s in shapes]
    for gs in case['grads']:
        kv.pushpull(keys, [[mx.nd.array(a, mx.gpu(0))] for a in gs], out=outs)
    for k in keys:
        assert eq(outs[k].asnumpy(), g["%s_w%d" % (name, k)]), (name, fused, k)


def test_store_mixed_precision_fp16_golden(mx, golden):
    """fp16 weights / gradients, fp32 master weights and momentum on the store (multi_precision): the
    fused kernel against the reference Updater's multi_mp_sgd_mom_update trajectory, fp16 bits equal"""
    g = golden("updater_trajectories")
    case = updater_cases()['sgd_mp_fp16']
    shapes, keys = case['shapes'], list(range(len(case['shapes'])))
    kv = mx.kv.create('device')
    for k in keys:
        kv.init(k, mx.nd.array(case['w0'][k], mx.gpu(0), np.float16))
    kv.set_optimizer(mx.optimizer.SGD(**case['opt'][1]))
    outs = [mx.nd.empty(s, mx.gpu(0), np.float16) for s in shapes]
    for gs in case['grads']:
        kv.pushpull(keys, [[mx.nd.array(a, mx.gpu(0), np.float16)] for a in gs], out=outs)
    for k in keys:
        got = outs[k].asnumpy()
        assert got.dtype == np.float16
        assert eq(got.view(np.uint16), g["sgd_mp_fp16_w%d" % k].view(np.uint16)), k


@pytest.mark.parametrize("name", ['lars_list', 'lamb_list'])
def test_local_updater_lars_lamb_golden(mx, golden, name):
    """update_on_kvstore=False: the LARS / LAMB front-end (tests/compat mirror, pinned to the reference's
    on the CPU side) over this library's multi-tensor operators on the GPU, against the trajectory of
    the reference's own classes over its own operators. Layers whose step involves a norm depend on
    the association of a float sum of squares (2e-6 relative per operator call): held to 1e-5 after
    three steps; gamma / beta / bias under LARS see no norm and must be bit-equal."""
    from compat import mxnet_optimizer as mxopt
    g = golden("updater_trajectories")
    case = updater_cases()[name]
    cls, kw = case['opt']
    kw = dict(kw, param_idx2name=dict(enumerate(case['names'])))
    if 'sched' in case:
        class Sched(object):
            base_lr = case['lr_at'][0]

            def __call__(self, num_update):
                return case['lr_at'][min(max(num_update, 1), len(case['lr_at'])) - 1]
        kw['lr_scheduler'] = Sched()
    opt = getattr(mxopt, cls)(**kw)
    upd = mxopt.get_updater(opt)
    ws = [mx.nd.array(w, mx.gpu(0)) for w in case['w0']]
    for gs in case['grads']:
        upd(list(range(len(ws))), [mx.nd.array(a, mx.gpu(0)) for a in gs], ws)
    for k, nm in enumerate(case['names']):
        got, want = ws[k].asnumpy().astype(np.float64), g["%s_w%d" % (name, k)].astype(np.float64)
        assert np.all(np.abs(got - want) <= 1e-5 * np.abs(want) + 1e-7), (name, nm)
        if cls == 'LARS' and nm.endswith(('gamma', 'beta', 'bias')):
            assert eq(ws[k].asnumpy(), g["%s_w%d" % (name, k)]), (name, nm)
