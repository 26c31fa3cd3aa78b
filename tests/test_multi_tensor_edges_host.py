"""Pins the multi-tensor optimizer restatements of oracle/kvoracle.c, which
tests/test_multi_tensor_edges_gpu.py trusts, at the shapes that file uses: multi-chunk tensors,
65-weight multi AdamW, 45-tensor multi LAMB and 1000-tensor multi_lars.

float32 and float16 are compared bit for bit against the reference's own FCompute<cpu> functions
(oracle/_ref/libmxref.so; skipped where it is not built). The reference has no bfloat16 form of
these operators (its MSHADOW_REAL_TYPE_SWITCH lacks the type), so the bfloat16 restatement
(kind 1) is checked against the float32 expression tree of the same restatement fed with the
same values: 16-bit data only enters by widening and leaves by rounding, plus the rounded
16-bit product of lamb phase 1, which the float32 tree is given already rounded."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import kvoracle as K  # noqa: E402
import golden_ops as G  # noqa: E402

CHUNK = 8192
MULTI = 3 * CHUNK + 5
P = K._ptr


def same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _arr(rng, n, dt, lo=-1.0, hi=1.0):
    return rng.uniform(lo, hi, n).astype(np.float32).astype(dt)


def _sizes(rng, count, big):
    sizes = [int(s) for s in rng.integers(1, 3000, count)]
    for k, n in big:
        sizes[k] = n
    return sizes


def _adamw(b, rng, dt, multi, count):
    mp = dt == np.float16
    sizes = _sizes(rng, count, [(0, MULTI), (count - 1, 2 * CHUNK + 4099)] if multi else [(0, MULTI)])
    ts = []
    for n in sizes:
        w = _arr(rng, n, dt)
        t = [w, _arr(rng, n, dt, -2, 2), _arr(rng, n, np.float32, -0.1, 0.1), _arr(rng, n, np.float32, 0, 0.1)]
        ts.append(t + ([w.astype(np.float32)] if mp else []))
    ins = [a for t in ts for a in t] + [np.array([0.37], np.float32)]
    kw = dict(beta1=0.9, beta2=0.98, epsilon=1e-6, clip_gradient=0.5)
    if multi:
        kw.update(num_weights=count, lrs=[0.001 * (1 + k / 37.0) for k in range(count)],
                  wds=[0.01 * (1 + k / 53.0) for k in range(count)], etas=[1 - k / 301.0 for k in range(count)])
    else:
        kw.update(lr=0.0123, wd=0.021, eta=0.87)
    name = '_%s%sadamw_update' % ('multi_' if multi else '', 'mp_' if mp else '')
    b.invoke(name, ins, [t[0] for t in ts], **kw)
    return {'%s%d' % (k, i): a for i, t in enumerate(ts) for k, a in zip(('w', 'g', 'mean', 'var', 'w32'), t)}


def _lamb_phases(b, rng, dt):
    mp = dt == np.float16
    n = 2 * CHUNK + 4099
    w, g = _arr(rng, n, dt), _arr(rng, n, dt, -2, 2)
    mean, var = _arr(rng, n, np.float32, -0.1, 0.1), _arr(rng, n, np.float32, 0, 0.1)
    w32 = (w.astype(np.float32) * np.float32(1.001)).astype(np.float32)
    gout = np.zeros(n, np.float32)
    kw = dict(t=3, wd=0.01, rescale_grad=0.37, clip_gradient=0.4, beta1=0.9, beta2=0.98, epsilon=1e-6)
    b.invoke('mp_lamb_update_phase1' if mp else 'lamb_update_phase1',
             [w, g, mean, var] + ([w32] if mp else []), [gout], **kw)
    r1 = np.array([np.sqrt(np.dot(w.astype(np.float64), w.astype(np.float64)))], np.float32)
    r2 = np.array([np.sqrt(np.dot(gout.astype(np.float64), gout))], np.float32)
    out = np.zeros(n, dt)
    b.invoke('mp_lamb_update_phase2' if mp else 'lamb_update_phase2',
             [w, gout, r1, r2] + ([w32] if mp else []), [out], lr=0.0031, lower_bound=float(r1[0]) * 2)
    return dict(mean=mean, var=var, gout=gout, out=out, w32=w32)


def _multi_lamb(b, rng, dt):
    mp = dt == np.float16
    count = 45
    sizes = _sizes(rng, count, [(3, 21 * CHUNK + 5), (20, 2 * CHUNK + 4099), (44, CHUNK + 1)])
    ts = []
    for n in sizes:
        w = _arr(rng, n, dt)
        t = [w, _arr(rng, n, dt, -3, 3), _arr(rng, n, np.float32, -0.1, 0.1), _arr(rng, n, np.float32, 0, 0.1)]
        ts.append(t + ([(w.astype(np.float32) * np.float32(1.001)).astype(np.float32)] if mp else []))
    ts[12][0][...] = 0
    if mp:
        ts[12][4][...] = 0
    norms = [float(np.sqrt(np.dot(t[0].astype(np.float64), t[0].astype(np.float64)))) for t in ts]
    nz = [x for x in norms if x > 0]
    kw = dict(learning_rates=[0.02 * (1 + k / 45.0) for k in range(count)],
              wds=[0.001 * (1 + k) for k in range(count)], beta1=0.9, beta2=0.98, epsilon=1e-6,
              rescale_grad=0.37, clip_gradient=1.5, num_tensors=count,
              step_count=[k + 1 for k in range(count)], lower_bound=2 * min(nz), upper_bound=0.5 * max(nz))
    b.invoke('_multi_mp_lamb_update' if mp else '_multi_lamb_update', [a for t in ts for a in t],
             [t[0] for t in ts], **kw)
    return {'%s%d' % (k, i): a for i, t in enumerate(ts) for k, a in zip(('w', 'g', 'mean', 'var', 'w32'), t)}


def _lars(b, rng):
    n = 1000
    lrs, wsq, gsq = rng.uniform(0.01, 1, n), rng.uniform(0, 50, n), rng.uniform(0, 50, n)
    wds = rng.uniform(0, 0.01, n)
    lrs, wsq, gsq, wds = (a.astype(np.float32) for a in (lrs, wsq, gsq, wds))
    wsq[0::3] = 0
    gsq[1::4] = 0
    out = np.zeros(n, np.float32)
    b.invoke('multi_lars', [lrs, wsq, gsq, wds], [out], eta=0.0013, eps=0.0, rescale_grad=0.37)
    return dict(out=out)


def _sum_sq(b, rng, dt):
    xs = [_arr(rng, n, dt) for n in (MULTI, 1, 2 * CHUNK + 4099, 300 * CHUNK + 7)]
    out = np.zeros(len(xs), np.float32)
    b.invoke('multi_sum_sq', xs, [out], num_arrays=len(xs))
    return dict(out=out)


CASES = {
    'adamw_f32': lambda b, r: _adamw(b, r, np.float32, False, 1),
    'mp_adamw_f16': lambda b, r: _adamw(b, r, np.float16, False, 1),
    'multi_adamw_65_f32': lambda b, r: _adamw(b, r, np.float32, True, 65),
    'multi_mp_adamw_65_f16': lambda b, r: _adamw(b, r, np.float16, True, 65),
    'lamb_phases_f32': lambda b, r: _lamb_phases(b, r, np.float32),
    'mp_lamb_phases_f16': lambda b, r: _lamb_phases(b, r, np.float16),
    'multi_lamb_45_f32': lambda b, r: _multi_lamb(b, r, np.float32),
    'multi_mp_lamb_45_f16': lambda b, r: _multi_lamb(b, r, np.float16),
    'multi_lars_1000': _lars,
    'sum_sq_f32': lambda b, r: _sum_sq(b, r, np.float32),
    'sum_sq_f16': lambda b, r: _sum_sq(b, r, np.float16),
}


class _RefAdamW50(G._RefBackend):
    """The reference's multi AdamW kernel parameters hold 50 tensors (adamw-inl.h:328-346,
    MultiAdamKernelParam::N, unchecked): a longer call is run there as consecutive calls of at most
    50 weights. Every tensor's update depends only on its own operands and scalars, so the split
    does not change what is compared."""

    def invoke(self, op, inputs, outputs, **params):
        n = params.get('num_weights')
        if n is None or n <= 50:
            return G._RefBackend.invoke(self, op, inputs, outputs, **params)
        stride = (len(inputs) - 1) // n
        for k0 in range(0, n, 50):
            k1 = min(n, k0 + 50)
            p = dict(params, num_weights=k1 - k0, lrs=params['lrs'][k0:k1], wds=params['wds'][k0:k1],
                     etas=params['etas'][k0:k1])
            G._RefBackend.invoke(self, op, inputs[k0 * stride:k1 * stride] + inputs[-1:], outputs[k0:k1], **p)


@pytest.mark.parametrize("case", sorted(CASES))
def test_restatement_matches_live_reference(case):
    ref = K.ref()
    if ref is None or not ref.has_ops():
        pytest.skip("oracle/_ref/libmxref.so not built here")
    seed = int.from_bytes(case.encode(), 'little') % (2 ** 31)
    want = CASES[case](_RefAdamW50(ref), np.random.default_rng(seed))
    got = CASES[case](G.OracleOps(K.get_oracle()), np.random.default_rng(seed))
    assert sorted(want) == sorted(got)
    for k in want:
        assert same(got[k], want[k]), (case, k)


# --------------------------------------------------------------------------------- bfloat16
def _bf16(rng, n, lo=-1.0, hi=1.0):
    """bfloat16 bit patterns of random values"""
    return K.Oracle._to_half_np(rng.uniform(lo, hi, n).astype(np.float32), 1)


def _wide(h):
    return K.Oracle.from_half(h, 1)


def _round(f):
    return K.Oracle._to_half_np(np.ascontiguousarray(f, np.float32), 1)


N = 2 * CHUNK + 4099
ADAM = dict(rescale=0.37, clip=0.5, beta1=0.9, beta2=0.98, eta=0.87, lr=0.0123, wd=0.021, eps=1e-6)


def _states(rng, n):
    return _arr(rng, n, np.float32, -0.1, 0.1), _arr(rng, n, np.float32, 0, 0.1)


def test_bf16_mp_adamw_is_the_float32_tree():
    L, a = K.get_oracle().lib, ADAM
    rng = np.random.default_rng(1)
    g16 = _bf16(rng, N, -2, 2)
    w32 = _arr(rng, N, np.float32)
    mean, var = _states(rng, N)
    m1, v1, w1, out16 = mean.copy(), var.copy(), w32.copy(), np.zeros(N, np.uint16)
    L.kvo_mp_adamw_update(N, P(out16), P(m1), P(v1), P(w1), P(g16), 1, a['rescale'], a['clip'], a['beta1'],
                          a['beta2'], a['eta'], a['lr'], a['wd'], a['eps'])
    m0, v0, w0, g0 = mean.copy(), var.copy(), w32.copy(), _wide(g16).copy()
    L.kvo_adamw_update(N, P(w0), P(m0), P(v0), P(w0), P(g0), a['rescale'], a['clip'], a['beta1'], a['beta2'],
                       a['eta'], a['lr'], a['wd'], a['eps'])
    assert same(m1, m0) and same(v1, v0) and same(w1, w0)
    assert same(out16, _round(w0))


@pytest.mark.parametrize("mp", [False, True])
def test_bf16_multi_adamw_is_the_float32_tree(mp):
    L, a = K.get_oracle().lib, ADAM
    rng = np.random.default_rng(2 + mp)
    g16 = _bf16(rng, N, -2, 2)
    w32 = _arr(rng, N, np.float32)
    mean, var = _states(rng, N)
    m1, v1, w1, w16 = mean.copy(), var.copy(), w32.copy(), np.zeros(N, np.uint16)
    L.kvo_multi_adamw_update(N, P(w1), None, P(w16), P(g16), 1, P(m1), P(v1), a['rescale'], a['clip'],
                             a['beta1'], a['beta2'], a['eta'], a['lr'], a['wd'], a['eps'])
    m0, v0, w0, g0 = mean.copy(), var.copy(), w32.copy(), _wide(g16).copy()
    L.kvo_multi_adamw_update(N, P(w0), P(g0), None, None, 0, P(m0), P(v0), a['rescale'], a['clip'],
                             a['beta1'], a['beta2'], a['eta'], a['lr'], a['wd'], a['eps'])
    assert same(m1, m0) and same(v1, v0) and same(w1, w0)
    assert same(w16, _round(w0))


@pytest.mark.parametrize("bias", [True, False])
def test_bf16_lamb_phase1_rounds_the_product_to_bf16(bias):
    """mp_lamb_update_phase1's `grad * rescale_grad` is a 16-bit product: the bfloat16 form equals
    the float32 tree given that product already rounded to bfloat16 (and rescale 1)"""
    L = K.get_oracle().lib
    rng = np.random.default_rng(4 + bias)
    g16 = _bf16(rng, N, -2, 2)
    w32 = _arr(rng, N, np.float32)
    mean, var = _states(rng, N)
    b1, b2, t = K.f32(0.9), K.f32(0.98), 3
    common = (0.4, None, b1, K.Oracle.beta_pow(b1, t), b2, K.Oracle.beta_pow(b2, t), 0.01, 1e-6, int(bias))
    m1, v1, o1 = mean.copy(), var.copy(), np.empty(N, np.float32)
    L.kvo_lamb_phase1(N, P(o1), P(m1), P(v1), P(w32), None, P(g16), 1, common[0], 0.37, *common[2:])
    g0 = _wide(_round(_wide(g16) * np.float32(0.37)))
    assert not same(g0, _wide(g16) * np.float32(0.37)), "the product must need rounding"
    m0, v0, o0 = mean.copy(), var.copy(), np.empty(N, np.float32)
    L.kvo_lamb_phase1(N, P(o0), P(m0), P(v0), P(w32), P(g0), None, -1, common[0], 1.0, *common[2:])
    assert same(m1, m0) and same(v1, v0) and same(o1, o0)


def test_bf16_lamb_phase2_rounds_the_float32_result():
    L = K.get_oracle().lib
    rng = np.random.default_rng(6)
    w32, g = _arr(rng, N, np.float32), _arr(rng, N, np.float32)
    for lb, ub in ((-1.0, -1.0), (9.0, -1.0), (-1.0, 0.25)):
        out16, out = np.zeros(N, np.uint16), np.zeros(N, np.float32)
        L.kvo_lamb_phase2(N, None, P(out16), 1, P(w32), P(g), 1.7, 0.9, 0.0031, lb, ub)
        L.kvo_lamb_phase2(N, P(out), None, 0, P(w32), P(g), 1.7, 0.9, 0.0031, lb, ub)
        assert same(out16, _round(out)), (lb, ub)


def test_bf16_multi_lamb_steps_are_the_float32_tree():
    L = K.get_oracle().lib
    rng = np.random.default_rng(7)
    g16 = _bf16(rng, N, -3, 3)
    w32 = _arr(rng, N, np.float32)
    mean, var = _states(rng, N)
    m1, v1, t1 = mean.copy(), var.copy(), np.empty(N, np.float32)
    L.kvo_multi_lamb_step1(N, P(t1), P(m1), P(v1), P(w32), None, P(g16), 1, 1.5, 0.37, K.f32(0.9),
                           K.f32(0.98), 1e-6, 0.004, 5, 1)
    m0, v0, t0, g0 = mean.copy(), var.copy(), np.empty(N, np.float32), _wide(g16).copy()
    L.kvo_multi_lamb_step1(N, P(t0), P(m0), P(v0), P(w32), P(g0), None, -1, 1.5, 0.37, K.f32(0.9),
                           K.f32(0.98), 1e-6, 0.004, 5, 1)
    assert same(m1, m0) and same(v1, v0) and same(t1, t0)
    w1, w16, w0 = w32.copy(), np.zeros(N, np.uint16), w32.copy()
    L.kvo_multi_lamb_step2(N, P(w1), P(w16), 1, P(t1), 123.0, 45.0, 0.02, 2.0, 20.0)
    L.kvo_multi_lamb_step2(N, P(w0), None, 0, P(t1), 123.0, 45.0, 0.02, 2.0, 20.0)
    assert same(w1, w0) and same(w16, _round(w0))


def test_bf16_sum_sq_adds_bf16_rounded_squares():
    """the restatement's bfloat16 sum of squares (the reference CPU's 16-bit product form): each
    square rounded to bfloat16, added in float32 in index order"""
    rng = np.random.default_rng(8)
    x = _bf16(rng, N)
    sq = _wide(_round(_wide(x) * _wide(x)))
    want = np.add.accumulate(sq, dtype=np.float32)[-1]
    got = K.get_oracle().lib.kvo_sum_sq(P(x), N, 1)
    assert np.float32(got) == want
