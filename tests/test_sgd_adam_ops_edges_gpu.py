"""The SGD and Adam optimizer operators (ops.cc: SgdAdam, MpSgd, MultiSgd) at the edges of the
fused launch they share with the store's step (dense_kernels.cu, dense_fused_kernel):

  * chunks: a tensor is cut into kChunkElems = 4096-element chunks, one CTA each; inside a chunk
    the vector body runs on 16-byte packs (4 float32 or 8 16-bit values) and a scalar tail takes
    the rest;
  * alignment: one vec_ok flag per tensor picks the vector or the scalar path for all of its
    operands, so one misaligned operand moves the whole tensor to the scalar path;
  * many tensors per launch, each with its own lr and wd, from tuples or from device arrays;
  * the plan cache: device tables keyed by the operands' addresses, cleared past 512 plans;
  * out distinct from the weight, clip_gradient at its edges, NaN, +-Inf, -0 and subnormals;
  * the weight dtypes each form refuses, before anything is enqueued;
  * float16 / bfloat16 keys on the store: the 16-bit sum in both association orders and the Test
    optimizer's half-precision arithmetic.

Every result is compared bit for bit (NaN as NaN) with the plain-C restatements of
oracle/kvoracle.c, which tests/test_sgd_adam_ops_edges_host.py pins to the reference's operators
at the special-value and clip cases."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import kvoracle as K  # noqa: E402
import golden_ndarray_ops as GN  # noqa: E402
import golden_update_ops as GU  # noqa: E402

pytestmark = pytest.mark.gpu

CHUNK = 4096                          # kChunkElems
SIZES32 = [1, 3, 4, 5, CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 5, (1 << 20) + 3]
SIZES16 = [7, 8, 9, 17, CHUNK + 9]
KIND = {'float16': 0, 'bfloat16': 1}
SPECIALS = np.array([np.nan, np.inf, -np.inf, -0.0, 1e-40, -1e-40], np.float32)

# operator -> (state names after weight and grad, whether it takes a 16-bit weight + fp32 master)
SINGLE = {
    'sgd_update': ((), False),
    'sgd_mom_update': (('mom',), False),
    'adam_update': (('mean', 'var'), False),
    'mp_sgd_update': (('w32',), True),
    'mp_sgd_mom_update': (('mom', 'w32'), True),
}
HYPER = dict(lr=0.0123, wd=0.021, momentum=0.9, beta1=0.9, beta2=0.999, epsilon=1e-8)


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200
    return anand_mxnet_b200


def sp(v):
    """the float32 value a scalar operator parameter takes (str() -> dmlc::stof)"""
    return K.scalar_param(v)


def narrow(f, dtype):
    """float32 values -> 16-bit bit patterns (round to nearest even)"""
    f = np.ascontiguousarray(f, np.float32)
    return f.astype(np.float16).view(np.uint16) if dtype == 'float16' else GU.to_bf16_bits(f)


def wide(h, dtype):
    return K.Oracle.from_half(h, KIND[dtype])


def up(mx, a, dtype):
    """host array (float32 values or 16-bit bit patterns) -> GPU NDArray of `dtype`"""
    if dtype == 'float32':
        return mx.nd.array(a, mx.gpu(0), np.float32)
    if dtype == 'float16':
        return mx.nd.array(a.view(np.float16), mx.gpu(0), np.float16)
    return mx.nd.array(GU.bf16_bits_to_f32(a), mx.gpu(0), 'bfloat16')


def down(nd, dtype):
    a = nd.asnumpy().reshape(-1)
    if dtype == 'float32':
        return a
    if dtype == 'float16':
        return a.view(np.uint16)
    return GU.to_bf16_bits(a)


def same(a, b, dtype):
    """bit equality with NaN as NaN (16-bit arrays are bit patterns)"""
    if dtype == 'float16':
        a, b = np.ascontiguousarray(a).view(np.float16), np.ascontiguousarray(b).view(np.float16)
    return GN.same(a, b, dtype)


class Tensor(object):
    """host copies (h) and GPU arrays (d) of one weight's operands: w and g in the weight's dtype,
    the states and the fp32 master in float32"""

    def __init__(self, mx, rng, n, dtype, states, specials=False):
        self.dtype, self.n = dtype, n
        f = {'w': rng.uniform(-1, 1, n), 'g': rng.uniform(-2, 2, n), 'mom': rng.uniform(-0.1, 0.1, n),
             'mean': rng.uniform(-0.1, 0.1, n), 'var': rng.uniform(0, 0.1, n)}
        f = {k: v.astype(np.float32) for k, v in f.items()}
        if specials:
            # each special value in every operand, in the vector body and in the scalar tail
            for i, k in enumerate(('w', 'g', 'mom', 'mean', 'var')):
                for j, v in enumerate(SPECIALS):
                    for p in (3 * j + i, n - 1 - 3 * j - i):
                        if 0 <= p < n:
                            f[k][p] = v
        self.names = ('w', 'g') + tuple(states)
        self.h = {}
        for k in self.names:
            if k == 'w32':
                self.h[k] = wide(self.h['w'], dtype) if specials else \
                    (wide(self.h['w'], dtype) * np.float32(1.001)).astype(np.float32)
                if specials:
                    self.h[k][1::7] = SPECIALS[np.arange(self.h[k][1::7].size) % SPECIALS.size]
            elif k in ('w', 'g') and dtype != 'float32':
                self.h[k] = narrow(f[k], dtype)
            else:
                self.h[k] = f[k].copy()
        self.d = {k: up(mx, self.h[k], self.dt(k)) for k in self.names}

    def dt(self, k):
        return self.dtype if k in ('w', 'g') else 'float32'

    def inputs(self):
        return [self.d[k] for k in self.names]

    def check(self, what, names=None):
        for k in names or self.names:
            assert same(down(self.d[k], self.dt(k)), self.h[k], self.dt(k)), (what, self.n, k)


def single_oracle(op, t, params):
    """the restated update of one tensor, in place on its host copies"""
    O = K.get_oracle()
    lr, wd, mom = sp(params['lr']), sp(params.get('wd', 0.0)), sp(params.get('momentum', 0.0))
    rescale = sp(params.get('rescale_grad', 1.0))
    clip = sp(params['clip_gradient']) if 'clip_gradient' in params else None
    h = t.h
    if op == 'sgd_update':
        O.sgd_update(h['w'], h['g'], lr, wd, rescale, clip)
    elif op == 'sgd_mom_update':
        O.sgd_mom_update(h['w'], h['g'], h['mom'], lr, mom, wd, rescale, clip)
    elif op == 'adam_update':
        O.adam_update(h['w'], h['g'], h['mean'], h['var'], lr, sp(params['beta1']), sp(params['beta2']),
                      sp(params['epsilon']), wd, rescale, clip)
    elif op == 'mp_sgd_update':
        O.mp_sgd_update(h['w'], h['w32'], h['g'], KIND[t.dtype], lr, wd, rescale, clip)
    else:
        O.multi_mp_sgd_update(h['w'], h['w32'], h['g'], h['mom'], KIND[t.dtype], lr, mom, wd, rescale,
                              clip)


def single_params(op, **kw):
    keys = {'sgd_update': ('lr', 'wd'), 'sgd_mom_update': ('lr', 'wd', 'momentum'),
            'adam_update': ('lr', 'wd', 'beta1', 'beta2', 'epsilon'), 'mp_sgd_update': ('lr', 'wd'),
            'mp_sgd_mom_update': ('lr', 'wd', 'momentum')}[op]
    p = {k: HYPER[k] for k in keys}
    p.update(kw)
    return p


def single_cases():
    out = []
    for op, (_, mp) in SINGLE.items():
        for dtype in (('float16', 'bfloat16') if mp else ('float32',)):
            for n in (SIZES16 if mp else SIZES32):
                out.append(pytest.param(op, dtype, n, id='%s-%s-%d' % (op, dtype, n)))
    return out


# ------------------------------------------------------------------------------ chunk edges
@pytest.mark.parametrize("op,dtype,n", single_cases())
def test_single_chunk_edges(mx, op, dtype, n):
    """one tensor at every chunk and vector-tail edge, two steps so the states carry over (the
    second one clipped, with a rescale_grad float32 cannot hold)"""
    rng = np.random.default_rng(n * 7 + len(op))
    t = Tensor(mx, rng, n, dtype, SINGLE[op][0])
    for step, kw in enumerate([dict(rescale_grad=0.5), dict(rescale_grad=0.1, clip_gradient=0.3)]):
        params = single_params(op, **kw)
        mx.nd._invoke(op, t.inputs(), out=t.d['w'], **params)
        single_oracle(op, t, params)
        t.check('step %d' % step)


# ------------------------------------------------------------------------------- alignment
def misaligned_cases():
    out = []
    for op, (states, mp) in SINGLE.items():
        for dtype in (('float16', 'bfloat16') if mp else ('float32',)):
            for k in ('w', 'g') + states:
                out.append(pytest.param(op, dtype, k, id='%s-%s-%s' % (op, dtype, k)))
    return out


@pytest.mark.parametrize("op,dtype,which", misaligned_cases())
def test_single_misaligned_operand(mx, op, dtype, which):
    """one operand a base[1:] view: the tensor takes the scalar path for all of its operands; the
    results are those of aligned operands and the elements around the view stay untouched"""
    mp = SINGLE[op][1]
    n = CHUNK + 9 if mp else 3 * CHUNK + 5
    rng = np.random.default_rng(len(op) * 11 + len(which))
    t = Tensor(mx, rng, n, dtype, SINGLE[op][0])
    dt = t.dt(which)
    pad = rng.uniform(-1, 1, 2).astype(np.float32)
    pad = narrow(pad, dt) if dt != 'float32' else pad
    base = up(mx, np.concatenate([pad[:1], t.h[which], pad[1:]]), dt)
    t.d[which] = base[1:1 + n]
    params = single_params(op, rescale_grad=0.37)
    mx.nd._invoke(op, t.inputs(), out=t.d['w'], **params)
    single_oracle(op, t, params)
    t.check('view of ' + which)
    b = down(base, dt)
    assert same(b[:1], pad[:1], dt) and same(b[-1:], pad[1:], dt), 'padding written'


# -------------------------------------------------------------------------------- out != w
@pytest.mark.parametrize("op,dtype", [('sgd_update', 'float32'), ('sgd_mom_update', 'float32'),
                                      ('adam_update', 'float32'), ('mp_sgd_update', 'float16'),
                                      ('mp_sgd_mom_update', 'bfloat16')])
def test_single_distinct_out(mx, op, dtype):
    """out is not the weight: the weight keeps its value, out and the states are the oracle's"""
    n = 3 * CHUNK + 5
    rng = np.random.default_rng(len(op) + 3)
    t = Tensor(mx, rng, n, dtype, SINGLE[op][0])
    w0 = t.h['w'].copy()
    out = up(mx, np.zeros(n, np.float32) if dtype == 'float32' else np.zeros(n, np.uint16), dtype)
    params = single_params(op, rescale_grad=0.25, clip_gradient=0.4)
    mx.nd._invoke(op, t.inputs(), out=out, **params)
    single_oracle(op, t, params)
    assert same(down(out, dtype), t.h['w'], dtype)
    t.h['w'] = w0
    t.check('distinct out')


# ----------------------------------------------------------------------------- clip, rescale
@pytest.mark.parametrize("clip", [None, -1.0, 0.0, 0.5], ids=['none', 'negative', 'zero', 'half'])
@pytest.mark.parametrize("op", list(SINGLE))
def test_single_clip_and_rescale(mx, op, clip):
    """clip_gradient absent, negative (off), zero and 0.5, with rescale_grad 0.1 (not a float32);
    the gradients include values whose rescaled value is exactly +-clip and one ulp either side"""
    mp = SINGLE[op][1]
    dtype = 'float16' if mp else 'float32'
    n = CHUNK + 9 if mp else CHUNK + 5
    rng = np.random.default_rng(len(op) * 3 + (0 if clip is None else int(clip * 10) + 2))
    t = Tensor(mx, rng, n, dtype, SINGLE[op][0])
    g = np.array([5.0, -5.0, 0.5, -0.5], np.float32)
    g = np.concatenate([g, np.nextafter(g, np.float32(np.inf)), np.nextafter(g, np.float32(-np.inf))])
    g = np.tile(g, 3)
    t.h['g'][:g.size] = narrow(g, dtype) if mp else g
    t.h['g'][-g.size:] = t.h['g'][:g.size]
    t.d['g'] = up(mx, t.h['g'], dtype)
    params = single_params(op, rescale_grad=0.1, **({} if clip is None else dict(clip_gradient=clip)))
    mx.nd._invoke(op, t.inputs(), out=t.d['w'], **params)
    single_oracle(op, t, params)
    t.check('clip %s' % clip)


# ---------------------------------------------------------------------------- special values
@pytest.mark.parametrize("op,dtype", [(op, dt) for op, (_, mp) in SINGLE.items()
                                      for dt in (('float16', 'bfloat16') if mp else ('float32',))])
def test_single_special_values(mx, op, dtype):
    """NaN, +-Inf, -0.0 and +-1e-40 in the weight, the gradient and every state, in the vector
    body and in the scalar tail, with and without clipping"""
    n = 2 * CHUNK + (9 if SINGLE[op][1] else 5)
    rng = np.random.default_rng(len(op) * 5 + len(dtype))
    t = Tensor(mx, rng, n, dtype, SINGLE[op][0], specials=True)
    for kw in (dict(rescale_grad=0.1), dict(rescale_grad=0.1, clip_gradient=0.5)):
        params = single_params(op, **kw)
        mx.nd._invoke(op, t.inputs(), out=t.d['w'], **params)
        single_oracle(op, t, params)
        t.check('specials %s' % kw)


# ----------------------------------------------------------------------------- multi forms
def multi_name(mom, mp, preloaded):
    return '%smulti_%ssgd_%supdate' % ('preloaded_' if preloaded else '', 'mp_' if mp else '',
                                       'mom_' if mom else '')


def multi_sizes(count, mp):
    sizes = SIZES16 if mp else SIZES32
    out = [sizes[(3 * k + 1) % len(sizes)] for k in range(count)]
    if count > 1:
        out[count // 2] = 0
    return out


class Multi(object):
    """`count` tensors of one multi call; every third one (from the second) has a misaligned
    weight view, so aligned and scalar-path tensors share the launch"""

    def __init__(self, mx, rng, count, mom, mp, dtype):
        self.mom, self.mp = mom, mp
        states = (('mom',) if mom else ()) + (('w32',) if mp else ())
        self.t = []
        self.bases = []
        for k, n in enumerate(multi_sizes(count, mp)):
            t = Tensor(mx, rng, n, dtype, states)
            if k % 3 == 1 and n > 0:
                pad = t.h['w'][:1].copy()
                base = up(mx, np.concatenate([pad, t.h['w']]), dtype)
                t.d['w'] = base[1:1 + n]
                self.bases.append((base, pad, dtype))
            self.t.append(t)

    def inputs(self):
        return [a for t in self.t for a in t.inputs()]

    def run(self, mx, name, preloaded, lrs, wds, **kw):
        count = len(self.t)
        if preloaded:
            ins = self.inputs() + [mx.nd.array(np.array(lrs, np.float32), mx.gpu(0)),
                                   mx.nd.array(np.array(wds, np.float32), mx.gpu(0))]
            mx.nd._invoke(name, ins, out=[t.d['w'] for t in self.t], num_weights=count, **kw)
        else:
            mx.nd._invoke(name, self.inputs(), out=[t.d['w'] for t in self.t], num_weights=count,
                          lrs=tuple(lrs), wds=tuple(wds), **kw)
        O = K.get_oracle()
        rescale = sp(kw.get('rescale_grad', 1.0))
        mom = sp(kw.get('momentum', 0.0))
        clip = sp(kw['clip_gradient']) if 'clip_gradient' in kw else None
        for t, lr, wd in zip(self.t, lrs, wds):
            h = t.h
            if self.mp:
                O.multi_mp_sgd_update(h['w'], h['w32'], h['g'], h.get('mom'), KIND[t.dtype], K.f32(lr), mom,
                                      K.f32(wd), rescale, clip)
            else:
                O.multi_sgd_update(h['w'], h['g'], h.get('mom'), K.f32(lr), mom, K.f32(wd), rescale, clip)

    def check(self, what):
        for k, t in enumerate(self.t):
            t.check('%s, tensor %d' % (what, k))
        for base, pad, dtype in self.bases:
            assert same(down(base, dtype)[:1], pad, dtype), 'padding written'


def multi_cases():
    out = []
    for preloaded in (False, True):
        for mp in (False, True):
            for mom in (False, True):
                for dtype in (('float16', 'bfloat16') if mp else ('float32',)):
                    for count in (1, 4, 60):
                        name = multi_name(mom, mp, preloaded)
                        out.append(pytest.param(name, preloaded, mp, mom, dtype, count,
                                                id='%s-%s-%d' % (name, dtype, count)))
    return out


@pytest.mark.parametrize("name,preloaded,mp,mom,dtype,count", multi_cases())
def test_multi_forms(mx, name, preloaded, mp, mom, dtype, count):
    """1, 4 and 60 tensors of the size list, one of them empty, a distinct lr and wd per tensor;
    then the same arrays again with new lrs (a plan-cache hit that must re-upload them)"""
    rng = np.random.default_rng(count * 13 + len(name) + len(dtype))
    M = Multi(mx, rng, count, mom, mp, dtype)
    kw = dict(rescale_grad=0.37, clip_gradient=0.6)
    if mom:
        kw['momentum'] = 0.85
    lrs = [0.01 * (1 + k / 37.0) for k in range(count)]
    wds = [0.001 * (1 + k / 53.0) for k in range(count)]
    M.run(mx, name, preloaded, lrs, wds, **kw)
    M.check('first call')
    M.run(mx, name, preloaded, [3.0 * lr for lr in lrs], wds, **kw)
    M.check('new lrs')


@pytest.mark.parametrize("op,dtype", [('multi_sgd_mom_update', 'float32'),
                                      ('multi_mp_sgd_mom_update', 'bfloat16')])
def test_multi_distinct_out(mx, op, dtype):
    """multi forms with outs that are not the weights"""
    mp = 'mp_' in op
    rng = np.random.default_rng(len(op))
    M = Multi(mx, rng, 4, True, mp, dtype)
    w0 = [t.h['w'].copy() for t in M.t]
    w_dev = [t.d['w'] for t in M.t]
    outs = [up(mx, np.zeros(t.n, np.uint16 if mp else np.float32), dtype) for t in M.t]
    for t, o in zip(M.t, outs):
        t.d['w'] = o
    lrs, wds = [0.01, 0.02, 0.03, 0.04], [0.001, 0.0, 0.003, 0.004]
    kw = dict(momentum=0.9, rescale_grad=0.5, num_weights=4, lrs=tuple(lrs), wds=tuple(wds))
    ins = []
    for t, w in zip(M.t, w_dev):
        ins += [w] + [t.d[k] for k in t.names[1:]]
    mx.nd._invoke(op, ins, out=outs, **kw)
    O = K.get_oracle()
    for t, lr, wd in zip(M.t, lrs, wds):
        if mp:
            O.multi_mp_sgd_update(t.h['w'], t.h['w32'], t.h['g'], t.h['mom'], KIND[dtype], K.f32(lr),
                                  sp(0.9), K.f32(wd), sp(0.5))
        else:
            O.multi_sgd_update(t.h['w'], t.h['g'], t.h['mom'], K.f32(lr), sp(0.9), K.f32(wd), sp(0.5))
    M.check('outs')
    for t, w, h in zip(M.t, w_dev, w0):
        assert same(down(w, dtype), h, dtype), 'weight written'


# ------------------------------------------------------------------------------ plan cache
def test_plan_cache_churn_in_flight(mx):
    """600 distinct single-tensor calls with no synchronisation in between (the cache is cleared
    after 512 plans while earlier launches may still be queued), each with its own lr, then every
    result"""
    rng = np.random.default_rng(600)
    ts, params = [], []
    for k in range(600):
        t = Tensor(mx, rng, 1 + (k * 37) % (CHUNK + 3), 'float32', ('mom',))
        p = single_params('sgd_mom_update', lr=0.001 * (1 + k), rescale_grad=0.5)
        mx.nd._invoke('sgd_mom_update', t.inputs(), out=t.d['w'], **p)
        ts.append(t)
        params.append(p)
    for k, (t, p) in enumerate(zip(ts, params)):
        single_oracle('sgd_mom_update', t, p)
        t.check('call %d' % k)


# -------------------------------------------------------------------------------- refusals
def refusal_cases():
    out = []
    for dtype in ('float16', 'bfloat16', 'float64'):
        for op in ('sgd_update', 'sgd_mom_update', 'adam_update', 'multi_sgd_update',
                   'multi_sgd_mom_update', 'preloaded_multi_sgd_update',
                   'preloaded_multi_sgd_mom_update'):
            out.append(pytest.param(op, dtype, id='%s-%s' % (op, dtype)))
    for op in ('mp_sgd_update', 'mp_sgd_mom_update', 'multi_mp_sgd_update', 'multi_mp_sgd_mom_update',
               'preloaded_multi_mp_sgd_update', 'preloaded_multi_mp_sgd_mom_update'):
        out.append(pytest.param(op, 'float64', id='%s-float64' % op))
    return out


@pytest.mark.parametrize("op,dtype", refusal_cases())
def test_refused_weight_dtypes(mx, op, dtype):
    """16-bit weights in every non-mp form (with float32 states, where the form has states) and
    float64 weights in every form: an MXNetError before anything is enqueued, with out and every
    state byte-identical"""
    n = CHUNK + 9
    ctx = mx.gpu(0)
    rng = np.random.default_rng(len(op))
    multi, preloaded = 'multi_' in op, op.startswith('preloaded_')
    mom, mp = 'mom_' in op or op == 'adam_update', 'mp_' in op
    nstates = 2 if op == 'adam_update' else int(mom) + int(mp)
    npdt = {'float16': np.float16, 'bfloat16': 'bfloat16', 'float64': np.float64}[dtype]

    def arr(v, dt):
        return mx.nd.array(v, ctx, dt)
    w = arr(rng.uniform(-1, 1, n).astype(np.float32), npdt)
    g = arr(rng.uniform(-1, 1, n).astype(np.float32), npdt)
    states = [arr(rng.uniform(0, 1, n).astype(np.float32), np.float32) for _ in range(nstates)]
    out = arr(rng.uniform(-1, 1, n).astype(np.float32), npdt)
    before = [a.asnumpy().tobytes() for a in [w, out] + states]
    ins = [w, g] + states
    kw = dict(rescale_grad=0.5)
    if multi:
        kw['num_weights'] = 1
        if preloaded:
            ins += [arr(np.array([0.1], np.float32), np.float32), arr(np.array([0.0], np.float32), np.float32)]
        else:
            kw.update(lrs=(0.1,), wds=(0.0,))
    else:
        kw['lr'] = 0.1
    mx.nd.waitall()
    launches = mx.base.kernel_launch_count()
    with pytest.raises(mx.MXNetError, match='takes float32'):
        mx.nd._invoke(op, ins, out=[out] if multi else out, **kw)
    mx.nd.waitall()
    assert mx.base.kernel_launch_count() == launches
    assert [a.asnumpy().tobytes() for a in [w, out] + states] == before


# ------------------------------------------------------------------- the store on 16-bit keys
STORE_SHAPES = [(3,), (4097,), (1000, 513)]


def sum16(srcs, order, dtype):
    """the 16-bit sum of the store: float32 adds, each rounded to the key's dtype, in the 'local'
    order g0 + (((g1+g2)+g3)+g4) + (((g5+... or the 'device' order ((g0+g1)+g2)+..."""
    r = lambda x: narrow(x, dtype)  # noqa: E731
    f = lambda h: wide(h, dtype)    # noqa: E731
    acc = srcs[0]
    if order == 'device':
        for s in srcs[1:]:
            acc = r(f(acc) + f(s))
        return acc
    for i in range(1, len(srcs), 4):
        t = srcs[i]
        for s in srcs[i + 1:i + 4]:
            t = r(f(t) + f(s))
        acc = r(f(acc) + f(t))
    return acc


def step_test16(w, g, rescale, dtype):
    """weight[:] += grad * rescale_grad in the key's dtype: the scalar, the product and the sum
    each rounded to it"""
    r = narrow(np.array([rescale], np.float32), dtype)
    prod = narrow(wide(g, dtype) * wide(r, dtype)[0], dtype)
    return narrow(wide(w, dtype) + wide(prod, dtype), dtype)


@pytest.mark.parametrize("n", [1, 2, 3, 5, 9])
@pytest.mark.parametrize("dtype", ['float16', 'bfloat16'])
@pytest.mark.parametrize("kvtype", ['local', 'device'])
@pytest.mark.parametrize("opt", ['none', 'test'])
def test_store_16bit_keys(mx, kvtype, dtype, n, opt):
    """n values per 16-bit key (one per MAXSRC instantiation of the fused kernel), no optimizer or
    Test(rescale_grad=0.1), two steps, against the 16-bit restatement of the store's order; Test
    also against the callback route, an updater running weight += grad * 0.1 through this
    library's _mul_scalar and _plus"""
    rng = np.random.default_rng(n * 4 + len(kvtype) + len(dtype) + len(opt))
    keys = list(range(len(STORE_SHAPES)))
    sizes = [int(np.prod(s)) for s in STORE_SHAPES]
    w0 = {k: narrow(rng.uniform(-1, 1, m).astype(np.float32), dtype) for k, m in zip(keys, sizes)}
    grads = [{k: [narrow(rng.uniform(-1, 1, m).astype(np.float32), dtype) for _ in range(n)]
              for k, m in zip(keys, sizes)} for _ in range(2)]
    routes = ['fused'] + (['callback'] if opt == 'test' else [])
    got = {}
    for route in routes:
        kv = mx.kv.create(kvtype)
        for k, s in zip(keys, STORE_SHAPES):
            kv.init(k, up(mx, w0[k], dtype).reshape(s))
        if route == 'fused' and opt == 'test':
            kv.set_optimizer(mx.optimizer.Test(rescale_grad=0.1))
        elif route == 'callback':
            def updater(key, recv, local):
                local += recv * 0.1
            kv._set_updater(updater)
        outs = [up(mx, np.zeros(m, np.uint16), dtype).reshape(s) for m, s in zip(sizes, STORE_SHAPES)]
        w = dict(w0)
        for step in range(2):
            kv.pushpull(keys, [[up(mx, g, dtype).reshape(s) for g in grads[step][k]]
                               for k, s in zip(keys, STORE_SHAPES)], out=outs)
            for k in keys:
                merged = sum16(grads[step][k], kvtype, dtype)
                w[k] = step_test16(w[k], merged, 0.1, dtype) if opt == 'test' else merged
                assert same(down(outs[k], dtype), w[k], dtype), (route, step, k)
        got[route] = [down(o, dtype) for o in outs]
    if opt == 'test':
        for a, b in zip(got['fused'], got['callback']):
            assert same(a, b, dtype)
