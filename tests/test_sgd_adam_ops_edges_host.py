"""Pins the SGD and Adam restatements of oracle/kvoracle.c, which
tests/test_sgd_adam_ops_edges_gpu.py trusts, at the cases that file adds: NaN, +-Inf, -0.0 and
subnormals in the weight, the gradient and every state, and clip_gradient absent, negative,
zero and 0.5 with gradients whose rescaled value is exactly +-clip. Each restatement is compared
bit for bit (NaN as NaN) with the reference's own FCompute<cpu> (oracle/_ref/libmxref.so; skipped
where it is not built).

It also records why the non-mp forms take float32 weights only: the reference's float16
sgd_update computes in half precision, rounding lr, wd and every intermediate, so its result is
not the float32 update rounded once to float16, which is what the fused kernel would compute."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import kvoracle as K  # noqa: E402
import golden_ndarray_ops as GN  # noqa: E402

N = 1031
SPECIALS = np.array([np.nan, np.inf, -np.inf, -0.0, 1e-40, -1e-40], np.float32)
CLIPS = [None, -1.0, 0.0, 0.5]


@pytest.fixture(scope="module")
def ref():
    r = K.ref()
    if r is None or not r.has_ops():
        pytest.skip("oracle/_ref/libmxref.so is not built")
    return r


def sp(v):
    return K.scalar_param(v)


def same(a, b):
    if a.dtype == np.float16:
        return GN.same(a, b, 'float16')
    return GN.same(a, b, 'float32')


def operands(seed, specials):
    """float32 w, g, mom, mean, var with the special values spread over every operand, or the
    gradients +-5 (rescaled by 0.1: exactly +-0.5) and one ulp either side"""
    rng = np.random.default_rng(seed)
    f = {'w': rng.uniform(-1, 1, N), 'g': rng.uniform(-2, 2, N), 'mom': rng.uniform(-0.1, 0.1, N),
         'mean': rng.uniform(-0.1, 0.1, N), 'var': rng.uniform(0, 0.1, N)}
    f = {k: v.astype(np.float32) for k, v in f.items()}
    if specials:
        for i, k in enumerate(f):
            for j, v in enumerate(SPECIALS):
                f[k][7 * j + i] = v
                f[k][N - 1 - 7 * j - i] = v
    else:
        g = np.array([5.0, -5.0, 0.5, -0.5], np.float32)
        g = np.concatenate([g, np.nextafter(g, np.float32(np.inf)), np.nextafter(g, np.float32(-np.inf))])
        f['g'][:g.size] = g
    return f


def params_of(op, clip):
    p = dict(lr=0.0123, wd=0.021, rescale_grad=0.1)
    if 'mom' in op:
        p['momentum'] = 0.9
    if op == 'adam_update':
        p.update(beta1=0.9, beta2=0.999, epsilon=1e-8)
    if clip is not None:
        p['clip_gradient'] = clip
    return p


OPS = ['sgd_update', 'sgd_mom_update', 'adam_update', 'mp_sgd_update', 'mp_sgd_mom_update',
       'multi_sgd_mom_update', 'multi_mp_sgd_mom_update']


@pytest.mark.parametrize("case", ['specials'] + ['clip-%s' % c for c in CLIPS])
@pytest.mark.parametrize("op", OPS)
def test_restatement_matches_reference(ref, op, case):
    clip = None if case in ('specials', 'clip-None') else float(case[5:])
    f = operands(len(op) * 10 + len(case), case == 'specials')
    p = params_of(op, clip)
    mp, multi = 'mp_' in op, op.startswith('multi_')
    states = ['mean', 'var'] if op == 'adam_update' else (['mom'] if 'mom' in op else [])
    # the reference: float16 weight and gradient of the mp forms, float32 everything else
    r = {k: f[k].copy() for k in ['w', 'g'] + states}
    if mp:
        r['w32'] = r['w'].astype(np.float16).astype(np.float32)
        r['w'], r['g'] = r['w'].astype(np.float16), r['g'].astype(np.float16)
    names = ['w', 'g'] + states + (['w32'] if mp else [])
    rp = dict(p)
    if multi:
        rp.update(num_weights=1, lrs=(p['lr'],), wds=(p['wd'],))
        del rp['lr'], rp['wd']
    ref.op_invoke(op, [r[k] for k in names], [r['w']], **rp)
    # the restatement, on the same values
    o = {k: (f[k].astype(np.float16) if mp and k in ('w', 'g') else f[k]).copy() for k in ['w', 'g'] + states}
    if mp:
        o['w32'] = o['w'].astype(np.float32)
        o['w'], o['g'] = o['w'].view(np.uint16), o['g'].view(np.uint16)
    O = K.get_oracle()
    lr, wd = (K.f32(p['lr']), K.f32(p['wd'])) if multi else (sp(p['lr']), sp(p['wd']))
    c = None if clip is None else sp(clip)
    rescale, mom = sp(p['rescale_grad']), sp(p.get('momentum', 0.0))
    if op == 'sgd_update':
        O.sgd_update(o['w'], o['g'], lr, wd, rescale, c)
    elif op == 'sgd_mom_update':
        O.sgd_mom_update(o['w'], o['g'], o['mom'], lr, mom, wd, rescale, c)
    elif op == 'multi_sgd_mom_update':
        O.multi_sgd_update(o['w'], o['g'], o['mom'], lr, mom, wd, rescale, c)
    elif op == 'adam_update':
        O.adam_update(o['w'], o['g'], o['mean'], o['var'], lr, sp(0.9), sp(0.999), sp(1e-8), wd, rescale, c)
    elif op == 'mp_sgd_update':
        O.mp_sgd_update(o['w'], o['w32'], o['g'], 0, lr, wd, rescale, c)
    else:
        O.multi_mp_sgd_update(o['w'], o['w32'], o['g'], o['mom'], 0, lr, mom, wd, rescale, c)
    if mp:
        o['w'] = o['w'].view(np.float16)
    for k in ['w'] + states + (['w32'] if mp else []):
        assert same(o[k], r[k]), (op, case, k)


def test_reference_float16_sgd_is_not_float32_rounded_once(ref):
    """sgd_update on float16 weights in the reference rounds lr (0.1 -> 0.0999755859375), wd and
    every intermediate to half precision; the float32 update rounded once to float16 differs from
    it, so the operator's non-mp forms cannot take 16-bit weights"""
    assert float(np.float16(0.1)) == 0.0999755859375
    rng = np.random.default_rng(16)
    w = rng.uniform(-1, 1, N).astype(np.float16)
    g = rng.uniform(-1, 1, N).astype(np.float16)
    got = w.copy()
    ref.op_invoke('sgd_update', [got, g], [got], lr=0.1, wd=0.01, rescale_grad=0.37)
    once = w.astype(np.float32)
    K.get_oracle().sgd_update(once, g.astype(np.float32), sp(0.1), sp(0.01), sp(0.37))
    once = once.astype(np.float16)
    differ = np.count_nonzero(got.view(np.uint16) != once.view(np.uint16))
    assert differ > N // 20, differ
