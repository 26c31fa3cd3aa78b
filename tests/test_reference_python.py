"""Host orchestration pinned to the reference's OWN Python front-end.

oracle/ref_python.py loads /root/reference/python/mxnet/optimizer/optimizer.py and lr_scheduler.py
unmodified and runs them over the reference's own compiled operators (oracle/_ref/libmxref.so), so
update counts, schedulers, lr / wd multipliers, Adam's bias correction, SGD's aggregation, mixed
precision states, LARS's layer split and LAMB's step counts are all the reference's code. Against it:

  * ``kvoracle.LocalKVStoreModel`` -- the checker of the GPU store's fused route -- bit for bit;
  * the mirror under tests/compat/ -- the checker of the GPU store's callback route -- bit for bit
    AND call for call (same operators, same parameter strings, same order);
  * tests/golden/updater_trajectories.npz (written from it by oracle/gen_golden.py; the reference
    Python cannot travel to the GPU box, the fixture does) -- checked here against the model, and
    against the CUDA store in tests/test_updater_reference_fixture_gpu.py.

The live halves need /root/reference and are skipped where it is absent (the GPU box)."""
import numpy as np
import pytest

import kvoracle as K
import ref_python as RP
from gen_golden import updater_cases, run_updater_case

live = pytest.mark.skipif(not RP.available(), reason="needs /root/reference and oracle/_ref/libmxref.so")


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def model_run(case):
    """the same plan through kvoracle.LocalKVStoreModel: per step, per key, push the gradient"""
    shapes, w0, grads = case['shapes'], case['w0'], case['grads']
    model = K.LocalKVStoreModel('device')
    for k, w in enumerate(w0):
        model.init(k, w)
    model.set_optimizer(lr_mult=case.get('lr_mult'), wd_mult=case.get('wd_mult'), **case['model'])
    for step in range(len(grads)):
        if 'lr_at' in case:
            model.opt['lr'] = case['lr_at'][step]
        for k in range(len(shapes)):
            model.push(k, [grads[step][k]])
    return [model.pull(k) for k in range(len(shapes))]


@pytest.mark.parametrize("name", sorted(n for n, c in updater_cases().items() if c['model']))
def test_model_vs_golden_trajectories(golden, name):
    g = golden("updater_trajectories")
    case = updater_cases()[name]
    got = model_run(case)
    for k, w in enumerate(got):
        assert eq(w, g["%s_w%d" % (name, k)]), (name, k)


@live
@pytest.mark.parametrize("name", sorted(updater_cases()))
def test_golden_trajectories_are_the_live_reference(golden, name):
    g = golden("updater_trajectories")
    case = updater_cases()[name]
    with RP.reference_python() as (opt, sched):
        got = run_updater_case(opt, sched, case)
    for k, w in enumerate(got):
        assert eq(w, g["%s_w%d" % (name, k)]), (name, k)


# ---------------------------------------------------------------- the tests/compat mirror
def _mirror():
    """tests/compat/mxnet_optimizer.py with its operator imports replaced by the harness's, so it
    runs on the same numpy buffers and the same reference operators as the reference front-end"""
    from compat import mxnet_optimizer as M
    saved = dict(M.__dict__)
    M.__dict__.update(RP.op_table())
    M._contrib = type('contrib', (), {'multi_lamb_update': staticmethod(RP.multi_lamb_update),
                                      'multi_mp_lamb_update': staticmethod(RP.multi_mp_lamb_update)})
    return M, saved


NAMES = ['conv0_weight', 'conv0_bias', 'bn0_gamma', 'bn0_beta', 'fc_weight', 'fc_bias', 'emb_weight']
SHAPES = [(8, 3, 3, 3), (8,), (8,), (8,), (10, 72), (10,), (37, 5)]


def _plan(rng, steps, dtype=np.float32):
    w0 = [rng.uniform(-1, 1, s).astype(dtype) for s in SHAPES]
    grads = [[rng.uniform(-1, 1, s).astype(dtype) for s in SHAPES] for _ in range(steps)]
    return w0, grads


def _drive(mod, sched_mod, make, w0, grads, mode, devices=1, lr_changes=None, restart_at=None):
    """mode 'single': updater(index, grad, weight) per key, as the store's callback does;
    mode 'list': updater([indices], [grads], [weights]) as Trainer._update does.
    devices > 1: one Updater per device sharing ONE optimizer (gluon/trainer.py:321-323).
    restart_at: pickle the updater states (dump_optimizer=True) before that step and continue from a
    fresh Updater, as Trainer.save_states / load_states do."""
    RP.LOG[:] = []
    opt = make(mod, sched_mod)
    upds = [mod.get_updater(opt) for _ in range(devices)]
    ws = [[RP.NDArray(w.copy(), RP.Context(d, 'gpu')) for w in w0] for d in range(devices)]
    for step, gs in enumerate(grads):
        if lr_changes and step in lr_changes:
            opt.set_learning_rate(lr_changes[step])
        if restart_at == step:
            blobs = [u.get_states(dump_optimizer=True) for u in upds]
            upds = [mod.get_updater(make(mod, sched_mod)) for _ in range(devices)]
            for u, b in zip(upds, blobs):
                u.set_states(b)
            opt = upds[0].optimizer
            for u in upds:
                u.optimizer = opt
        for d, upd in enumerate(upds):
            garr = [RP.NDArray(g.copy(), RP.Context(d, 'gpu')) for g in gs]
            if mode == 'single':
                for k in range(len(w0)):
                    upd(k, garr[k], ws[d][k])
            else:
                upd(list(range(len(w0))), garr, ws[d])
    states = {}
    for d, upd in enumerate(upds):
        for k, st in upd.states.items():
            flat = RP._flat([st]) if isinstance(st, (list, tuple)) else [st]
            states[(d, k)] = [s.a.copy() for s in flat if s is not None]
    return [[w.a.copy() for w in dev] for dev in ws], states, list(RP.LOG), opt.num_update


CONFIGS = {
    'sgd_mom': lambda m, s: m.SGD(learning_rate=0.1, momentum=0.9, wd=1e-4, rescale_grad=1 / 32,
                                  param_idx2name=dict(enumerate(NAMES))),
    'sgd_plain_clip': lambda m, s: m.SGD(learning_rate=0.05, wd=1e-3, clip_gradient=0.3),
    'sgd_mults': lambda m, s: _with_mults(m.SGD(learning_rate=0.1, momentum=0.9, wd=1e-4,
                                                param_idx2name=dict(enumerate(NAMES)))),
    'sgd_factor_sched': lambda m, s: m.SGD(momentum=0.9, wd=1e-4,
                                           lr_scheduler=s.FactorScheduler(step=2, factor=0.5, base_lr=0.2)),
    'sgd_multifactor_warmup': lambda m, s: m.SGD(
        momentum=0.9, lr_scheduler=s.MultiFactorScheduler(step=[2, 4], factor=0.1, base_lr=0.4,
                                                          warmup_steps=2, warmup_begin_lr=0.01)),
    'sgd_cosine': lambda m, s: m.SGD(learning_rate=0.3, momentum=0.5,
                                     lr_scheduler=s.CosineScheduler(max_update=5, base_lr=0.3, final_lr=0.01)),
    'sgd_begin_num_update': lambda m, s: m.SGD(learning_rate=0.1, begin_num_update=7,
                                               lr_scheduler=s.PolyScheduler(max_update=20, base_lr=0.1, pwr=2)),
    'adam': lambda m, s: m.Adam(learning_rate=1e-3, wd=0.01, rescale_grad=0.5,
                                param_idx2name=dict(enumerate(NAMES))),
    'adam_clip_betas': lambda m, s: m.Adam(learning_rate=3e-4, beta1=0.8, beta2=0.98, epsilon=1e-6,
                                           clip_gradient=0.25),
    'adam_begin_num_update': lambda m, s: m.Adam(learning_rate=1e-3, begin_num_update=100),
    'lars': lambda m, s: m.LARS(learning_rate=0.2, momentum=0.9, wd=1e-4, eta=0.001, eps=1e-9,
                                rescale_grad=1 / 32, param_idx2name=dict(enumerate(NAMES))),
    'lars_sched_correction': lambda m, s: m.LARS(momentum=0.9, wd=1e-4, eta=0.002, rescale_grad=1 / 8,
                                                 param_idx2name=dict(enumerate(NAMES)),
                                                 lr_scheduler=s.FactorScheduler(step=2, factor=0.5, base_lr=0.4)),
    'lars_no_momentum': lambda m, s: m.LARS(learning_rate=0.1, wd=1e-3, eta=0.01, clip_gradient=0.5,
                                            param_idx2name=dict(enumerate(NAMES))),
    'lamb': lambda m, s: m.LAMB(learning_rate=2e-3, wd=0.01, rescale_grad=0.25,
                                param_idx2name=dict(enumerate(NAMES))),
    'lamb_bounds_nobias': lambda m, s: m.LAMB(learning_rate=1e-3, lower_bound=0.01, upper_bound=2.0,
                                              bias_correction=False, clip_gradient=0.4),
    'test': lambda m, s: m.Test(rescale_grad=2.0),
    # dmlc::stof and std::stod-then-float parse this rescale_grad to different floats
    'test_rescale_stod': lambda m, s: m.Test(rescale_grad=1.2345e-05),
}


def _with_mults(opt):
    opt.set_lr_mult({1: 0.5, 'fc_weight': 2.0, 6: 0.25})
    opt.set_wd_mult({0: 0.0, 'bn0_beta': 0.5})
    return opt


def _norm(call):
    """(operator, parameters) with tuple-valued parameters as token lists: the mirror hands python
    tuples to the operators where the reference hands lists -- '(0.1,)' and '[0.1]' are the same
    value to the Tuple<float> parser (include/mxnet/tuple.h); every token must still be identical"""
    name, params = call
    out = {}
    for k, v in params.items():
        out[k] = [t.strip() for t in v.strip('()[]').split(',') if t.strip()] if v[:1] in '([' else v
    return name, out


def _compare(cfg, mode, dtype=np.float32, steps=5, monkeypatch=None, agg=None, mp=False, **kw):
    if agg is not None:
        monkeypatch.setenv('MXNET_OPTIMIZER_AGGREGATION_SIZE', str(agg))
    make = CONFIGS[cfg]
    if mp:
        base = make

        def make(m, s):                     # noqa: E306
            o = base(m, s)
            o.multi_precision = True
            return o
    w0, grads = _plan(np.random.default_rng(len(cfg) + steps), steps, dtype)
    with RP.reference_python() as (opt, sched):
        want = _drive(opt, sched, make, w0, grads, mode, **kw)
        M, saved = _mirror()
        try:
            got = _drive(M, sched, make, w0, grads, mode, **kw)
        finally:
            M.__dict__.clear()
            M.__dict__.update(saved)
    assert got[3] == want[3]                                  # num_update
    assert len(got[2]) == len(want[2]) and len(want[2]) > 0
    for a, b in zip(got[2], want[2]):                         # operator, parameter strings, order
        assert _norm(a) == _norm(b)
    for dev_g, dev_w in zip(got[0], want[0]):
        for k, (a, b) in enumerate(zip(dev_g, dev_w)):
            assert eq(a, b), (cfg, mode, k)
    assert got[1].keys() == want[1].keys()
    for key in want[1]:
        assert len(got[1][key]) == len(want[1][key])
        for a, b in zip(got[1][key], want[1][key]):
            assert eq(a, b), (cfg, mode, key)


@live
@pytest.mark.parametrize("mode", ['single', 'list'])
@pytest.mark.parametrize("cfg", sorted(c for c in CONFIGS if not c.startswith('test')))
def test_compat_mirror_vs_reference(cfg, mode):
    _compare(cfg, mode)


@live
def test_compat_mirror_test_optimizer():
    _compare('test', 'single')


@live
def test_compat_mirror_test_optimizer_stod_rescale():
    """grad * rescale_grad is _mul_scalar: the reference's registered parser, not dmlc::stof"""
    _compare('test_rescale_stod', 'single')


@live
@pytest.mark.parametrize("cfg", ['sgd_mom', 'sgd_plain_clip', 'lars', 'lars_no_momentum', 'lamb', 'adam'])
@pytest.mark.parametrize("agg", [1, 3, 45])
def test_compat_mirror_aggregation_sizes(cfg, agg, monkeypatch):
    if cfg == 'lamb' and agg == 1:
        pytest.skip("LAMB's one-tensor form calls NDArray.norm(), an operator outside the harness")
    _compare(cfg, 'list', monkeypatch=monkeypatch, agg=agg)


@live
@pytest.mark.parametrize("cfg", ['sgd_mom', 'sgd_plain_clip', 'lars', 'lars_no_momentum', 'lamb', 'adam'])
@pytest.mark.parametrize("mode", ['single', 'list'])
def test_compat_mirror_multi_precision_fp16(cfg, mode):
    _compare(cfg, mode, dtype=np.float16, mp=True)


@live
@pytest.mark.parametrize("cfg", ['sgd_mom', 'adam', 'lars_sched_correction', 'sgd_factor_sched'])
def test_compat_mirror_shared_optimizer_two_devices(cfg):
    _compare(cfg, 'list', devices=2)


@live
@pytest.mark.parametrize("cfg", ['sgd_mom', 'adam', 'lamb'])
def test_compat_mirror_set_learning_rate_between_steps(cfg):
    _compare(cfg, 'single', lr_changes={2: 0.01, 4: 0.3})


@live
@pytest.mark.parametrize("cfg", ['sgd_mom', 'adam', 'sgd_factor_sched'])
def test_compat_mirror_state_pickle_restart(cfg):
    _compare(cfg, 'list', restart_at=3)


# ---------------------------------------------------------------- the product's hyper-parameter record
@live
def test_fused_record_vs_reference_optimizer():
    """anand_mxnet_b200.optimizer.FusedOptimizer (what kv.set_optimizer turns into the native replay's
    inputs) against the reference's Optimizer: multiplier lookup order (Parameter object, index, name),
    default wd_mult of non-weights, scheduler / explicit learning rate precedence -- for records built
    directly and for records taken from an object of the reference's own classes (record_of)."""
    from anand_mxnet_b200 import optimizer as P

    class Param(object):
        def __init__(self, lr_mult, wd_mult):
            self.lr_mult, self.wd_mult = lr_mult, wd_mult
    idx2name = dict(enumerate(NAMES))
    variants = [
        dict(),
        dict(param_idx2name=idx2name),
        dict(param_idx2name=idx2name, param_dict={2: Param(0.3, 0.7), 4: Param(5.0, 0.0)}),
        dict(param_dict={0: Param(0.5, 2.0)}),
    ]
    setters = [
        ({}, {}),
        ({1: 0.5, 'fc_weight': 2.0, 6: 0.25}, {0: 0.0, 'bn0_beta': 0.5, 'fc_bias': 3.0}),
        ({'conv0_weight': 0.1, 0: 0.2}, {'emb_weight': 0.0}),          # index beats name
    ]
    with RP.reference_python() as (opt, sched):
        for cls in ('SGD', 'Adam', 'Test'):
            for kw in variants:
                for lr_mult, wd_mult in setters:
                    ref = getattr(opt, cls)(learning_rate=1.0, wd=1.0, **kw)
                    mine = getattr(P, cls)(learning_rate=1.0, wd=1.0, **kw)
                    for o in (ref, mine):
                        o.set_lr_mult(lr_mult)
                        o.set_wd_mult(wd_mult)
                    assert P.fused_kind(ref) == cls.lower()
                    rec = P.record_of(ref)
                    for i in list(range(len(NAMES) + 2)) + ['fc_weight']:
                        want = (ref._get_lr(i), ref._get_wd(i))       # lr = wd = 1: the multipliers
                        assert mine.multipliers(i) == want, (cls, kw.keys(), i)
                        assert rec.multipliers(i) == want, (cls, kw.keys(), i)
        # learning rate: scheduler(num_update), an explicit rate overriding the scheduler's base
        for mk in (lambda m: dict(lr_scheduler=sched.FactorScheduler(step=3, factor=0.5, base_lr=0.4)),
                   lambda m: dict(lr_scheduler=sched.FactorScheduler(step=3, factor=0.5, base_lr=0.4),
                                  learning_rate=0.8),
                   lambda m: dict(learning_rate=0.25), lambda m: dict()):
            ref, mine = opt.SGD(**mk(0)), P.SGD(**mk(0))
            for n in (0, 1, 3, 4, 7, 20):
                ref.num_update = mine.num_update = n
                assert ref.learning_rate == mine.learning_rate == P.record_of(ref).learning_rate
            for o in (ref, mine):
                if o.lr_scheduler is None:
                    o.set_learning_rate(0.03)
                    assert o.learning_rate == 0.03
                else:
                    with pytest.raises(UserWarning):
                        o.set_learning_rate(0.03)
        # operator parameters handed to the library: the reference object's own attribute values
        ref = opt.Adam(learning_rate=2e-3, beta1=0.8, beta2=0.97, epsilon=1e-5, wd=0.1, rescale_grad=0.5,
                       clip_gradient=0.7, begin_num_update=11)
        p = P.record_of(ref).op_params()
        assert (p['learning_rate'], p['beta1'], p['beta2'], p['epsilon'], p['wd'], p['rescale_grad'],
                p['clip_gradient'], p['begin_num_update']) == (2e-3, 0.8, 0.97, 1e-5, 0.1, 0.5, 0.7, 11)
        ref = opt.SGD(momentum=0.9, clip_gradient=None)
        p = P.record_of(ref).op_params()
        assert p['momentum'] == 0.9 and p['clip_gradient'] == 0.0 and p['learning_rate'] == 0.01
