"""The multi-tensor optimizer operators (multi_tensor_kernels.cu / multi_ops.cc) at the edges of
their launch machinery, which the small-shape fixture cases of test_ops_gpu.py never reach:

  * chunks: a tensor is cut into kMTChunk = 8192-element chunks, one CTA each; inside a chunk the
    vector body runs on 4-element groups and a scalar tail takes the rest;
  * launch groups: a call is split into groups of kMTMaxTensors = 64 tensors, and each group's
    per-tensor scalars (lr, wd, eta, ...) are re-based to the group;
  * alignment: one vec_ok flag per tensor picks the vector or the scalar path for all of its
    operands (16-byte alignment for float32, 8 for the 16-bit types);
  * the plan cache: device tables keyed by a signature of the operands, cleared past 512 plans;
  * the sums of squares: per-chunk partials folded by a second kernel;
  * bfloat16 in every multi-precision form.

References: the plain-C restatements of oracle/kvoracle.c (pinned to the reference's operators
by tests/test_oracle_ops.py and tests/test_multi_tensor_edges_host.py; kind 1 is their bfloat16
form) and float64 numpy for sums of squares. Elementwise results are compared bit for bit. A
result that goes through a sum of squares is compared within sum_sq_rel_bound(), derived from
the kernel's summation structure."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import kvoracle as K  # noqa: E402
import golden_update_ops as GU  # noqa: E402

pytestmark = pytest.mark.gpu

CHUNK = 8192                 # kMTChunk: elements per CTA
U = 2.0 ** -24               # unit roundoff of float32
SIZES = [1, 3, CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 5,
         2 * CHUNK + 4099]   # the last: multi-chunk, 4099 = 1024 groups of 4 + a scalar tail of 3
MULTI = 3 * CHUNK + 5
DTYPES = ['float32', 'float16', 'bfloat16']
KIND = {'float32': -1, 'float16': 0, 'bfloat16': 1}
P = K._ptr


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200
    return anand_mxnet_b200


def lib():
    return K.get_oracle().lib


def sum_sq_rel_bound(n, squares_exact):
    """Relative error bound of the GPU's float32 sum of squares of n elements against the exact
    sum (all terms are non-negative, so the bound is relative to the sum itself). Along every
    term's path the kernel rounds at most: 32 sequential adds per thread in its chunk (8192
    elements over 256 threads), 5 shuffle levels and 8 warp leaders in the chunk's block_sum,
    ceil(chunks / 256) sequential adds per thread in the fold kernel and 5 + 8 more levels in its
    block_sum: 58 + ceil(chunks / 256) additions, plus one rounding of the square itself unless
    the square is exact (a widened 16-bit value has at most 11 significant bits)."""
    chunks = max(1, -(-n // CHUNK))
    m = 58 + -(-chunks // 256) + (0 if squares_exact else 1)
    return m * U / (1 - m * U)


def narrow(f, dtype):
    """float32 values -> 16-bit bit patterns (round to nearest even)"""
    return K.Oracle._to_half_np(np.ascontiguousarray(f, np.float32), KIND[dtype])


def wide(a, dtype):
    return a if dtype == 'float32' else K.Oracle.from_half(a, KIND[dtype])


def rand(rng, n, dtype='float32', lo=-1.0, hi=1.0):
    f = rng.uniform(lo, hi, n).astype(np.float32)
    return f if dtype == 'float32' else narrow(f, dtype)


def up(mx, a, dtype='float32'):
    """host array (float32 values or 16-bit bit patterns) -> GPU NDArray of `dtype`"""
    if dtype == 'float32':
        return mx.nd.array(a, mx.gpu(0), np.float32)
    if dtype == 'float16':
        return mx.nd.array(a.view(np.float16), mx.gpu(0), np.float16)
    return mx.nd.array(GU.bf16_bits_to_f32(a), mx.gpu(0), 'bfloat16')


def down(nd, dtype='float32'):
    a = nd.asnumpy().reshape(-1)
    if dtype == 'float32':
        return a
    if dtype == 'float16':
        return a.view(np.uint16)
    return GU.to_bf16_bits(a)


def same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def sp(v):
    """the float32 value a scalar operator parameter takes (str() -> dmlc::stof)"""
    return K.scalar_param(v)


# ------------------------------------------------------------------------------------- AdamW
ADAMW = dict(beta1=0.9, beta2=0.98, epsilon=1e-6)


class Tensors(object):
    """host copies and GPU arrays of an optimizer's tensors: w, g (dtype), mean, var and, for
    16-bit weights, the float32 master w32"""

    def __init__(self, mx, rng, sizes, dtype, master_skew=0.0):
        self.dtype = dtype
        self.mp = dtype != 'float32'
        self.h = []
        for n in sizes:
            t = dict(w=rand(rng, n, dtype), g=rand(rng, n, dtype, -2, 2),
                     mean=rand(rng, n, 'float32', -0.1, 0.1), var=rand(rng, n, 'float32', 0, 0.1))
            if self.mp:
                t['w32'] = (wide(t['w'], dtype) * np.float32(1 + master_skew)).astype(np.float32)
            self.h.append(t)
        self.d = [{k: up(mx, v, self.dt(k)) for k, v in t.items()} for t in self.h]

    def dt(self, key):
        return self.dtype if key in ('w', 'g') else 'float32'

    def names(self):
        return ('w', 'g', 'mean', 'var') + (('w32',) if self.mp else ())

    def inputs(self):
        return [t[k] for t in self.d for k in self.names()]

    def new_grads(self, mx, rng):
        for t, d in zip(self.h, self.d):
            t['g'] = rand(rng, t['w'].size, self.dtype, -2, 2)
            d['g'] = up(mx, t['g'], self.dtype)

    def check(self, what, keys=None):
        for i, (t, d) in enumerate(zip(self.h, self.d)):
            for k in keys or self.names():
                assert same(down(d[k], self.dt(k)), t[k]), (what, 'tensor %d' % i, k)


def adamw_gpu(mx, T, multi, rescale, params):
    op = '_%s%sadamw_update' % ('multi_' if multi else '', 'mp_' if T.mp else '')
    if multi:
        params = dict(params, num_weights=len(T.d))
    mx.nd._invoke(op, T.inputs() + [mx.nd.array([rescale], mx.gpu(0))], out=[d['w'] for d in T.d],
                  **params)


def adamw_oracle(T, multi, rescale, params):
    """the restated update of every tensor, in place on the host copies"""
    r = float(np.float32(rescale))
    if not np.isfinite(r) or r == 0:
        return  # adamw-inl.h:449-461: the update is skipped
    L, kind = lib(), KIND[T.dtype]
    clip = sp(params.get('clip_gradient', -1.0))
    b1, b2, eps = sp(params['beta1']), sp(params['beta2']), sp(params['epsilon'])
    for k, t in enumerate(T.h):
        n = t['w'].size
        if multi:
            lr, wd, eta = K.f32(params['lrs'][k]), K.f32(params['wds'][k]), K.f32(params['etas'][k])
            if T.mp:
                L.kvo_multi_adamw_update(n, P(t['w32']), None, P(t['w']), P(t['g']), kind, P(t['mean']),
                                         P(t['var']), r, clip, b1, b2, eta, lr, wd, eps)
            else:
                L.kvo_multi_adamw_update(n, P(t['w']), P(t['g']), None, None, 0, P(t['mean']),
                                         P(t['var']), r, clip, b1, b2, eta, lr, wd, eps)
        else:
            lr, wd, eta = sp(params['lr']), sp(params.get('wd', 0.0)), sp(params['eta'])
            if T.mp:
                L.kvo_mp_adamw_update(n, P(t['w']), P(t['mean']), P(t['var']), P(t['w32']), P(t['g']),
                                      kind, r, clip, b1, b2, eta, lr, wd, eps)
            else:  # rewrites g with the rescaled gradient, as the reference does
                L.kvo_adamw_update(n, P(t['w']), P(t['mean']), P(t['var']), P(t['w']), P(t['g']), r,
                                   clip, b1, b2, eta, lr, wd, eps)


def adamw_params(multi, count, k0=0):
    if not multi:
        return dict(ADAMW, lr=0.0123, wd=0.021, eta=0.87)
    # a distinct lr, wd and eta for every tensor: a scalar read from the wrong slot changes bits
    return dict(ADAMW, lrs=[0.001 * (1 + (k0 + k) / 37.0) for k in range(count)],
                wds=[0.01 * (1 + (k0 + k) / 53.0) for k in range(count)],
                etas=[1.0 - (k0 + k) / 301.0 for k in range(count)])


@pytest.mark.parametrize("multi", [False, True], ids=["single", "multi"])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", SIZES)
def test_adamw_chunk_edges(mx, n, dtype, multi):
    """_[mp_]adamw_update and _multi_[mp_]adamw_update on one tensor at every chunk edge, two
    steps so the states carry over (the second one clipped), bit for bit"""
    rng = np.random.default_rng(n * 6 + DTYPES.index(dtype) * 2 + multi)
    T = Tensors(mx, rng, [n], dtype)
    for step, extra in enumerate(({}, {'clip_gradient': 0.05})):
        if step:
            T.new_grads(mx, rng)
        params = dict(adamw_params(multi, 1), **extra)
        adamw_gpu(mx, T, multi, 0.37, params)
        adamw_oracle(T, multi, 0.37, params)
        T.check('step %d' % step)


@pytest.mark.parametrize("rescale", [0.0, float('inf'), float('nan')])
@pytest.mark.parametrize("multi", [False, True], ids=["single", "multi"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_adamw_skips_on_zero_or_nonfinite_rescale(mx, dtype, multi, rescale):
    """rescale_grad 0 / inf / nan skips the whole update: no array changes, multi-chunk size"""
    rng = np.random.default_rng(11)
    T = Tensors(mx, rng, [MULTI] if not multi else [MULTI, 5], dtype)
    adamw_gpu(mx, T, multi, rescale, adamw_params(multi, len(T.h)))
    T.check('rescale_grad=%r' % rescale)


def _group_sizes(rng, count):
    """sizes 1..3000 with empty tensors at 1 and 66, one-chunk edges at 5 and 6, and multi-chunk
    tensors on both sides of every 64-tensor group boundary"""
    sizes = [int(s) for s in rng.integers(1, 3000, count)]
    for k, n in ((1, 0), (66, 0), (5, CHUNK), (6, CHUNK - 1), (0, MULTI), (62, 2 * CHUNK + 4099),
                 (63, MULTI), (64, 2 * CHUNK + 4099), (100, MULTI), (127, CHUNK + 1), (128, MULTI)):
        if k < count:
            sizes[k] = n
    return sizes


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("count", [64, 65, 129])
def test_multi_adamw_launch_groups(mx, count, dtype):
    """_multi_[mp_]adamw_update over 1, 2 and 3 launch groups: each tensor takes its own lr / wd /
    eta in every group; two steps, bit for bit"""
    rng = np.random.default_rng(count * 3 + DTYPES.index(dtype))
    T = Tensors(mx, rng, _group_sizes(rng, count), dtype)
    for step in range(2):
        if step:
            T.new_grads(mx, rng)
        params = adamw_params(True, count, k0=step)
        adamw_gpu(mx, T, True, 0.37, params)
        adamw_oracle(T, True, 0.37, params)
        T.check('step %d' % step)


# ------------------------------------------------------------------------------- multi_sum_sq
def _check_sum_sq(got, arrays, dtype):
    for k, a in enumerate(arrays):
        x = wide(a, dtype).astype(np.float64)
        exact = float(np.dot(x, x))   # the GPU squares the widened value in float, as the
        # reference's GPU kernel does (multi_sum_sq.cu): 16-bit squares are exact in float
        bound = sum_sq_rel_bound(a.size, dtype != 'float32') * exact
        assert abs(float(got[k]) - exact) <= bound, (k, a.size, float(got[k]), exact)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("count", [65, 129])
def test_multi_sum_sq_launch_groups(mx, count, dtype):
    """multi_sum_sq over 2 and 3 launch groups, empty arrays at 63 and 64 (the last of the first
    group and the first of the second): every sum lands in its own slot"""
    rng = np.random.default_rng(count + DTYPES.index(dtype))
    sizes = _group_sizes(rng, count)
    sizes[63] = sizes[64] = 0
    # a distinct scale per array, so that a sum written to another slot is wrong
    arrays = [rand(rng, n, dtype, 0.1 * (1 + k % 17), 0.2 * (1 + k % 17)) for k, n in enumerate(sizes)]
    got = mx.nd.multi_sum_sq(*[up(mx, a, dtype) for a in arrays], num_arrays=count).asnumpy()
    assert got.shape == (count,)
    assert got[63] == 0 and got[64] == 0
    _check_sum_sq(got, arrays, dtype)


# ------------------------------------------------------------------------------------ LAMB phases
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", SIZES)
def test_lamb_phases_chunk_edges(mx, n, dtype):
    """[mp_]lamb_update_phase1 (with and without bias correction and clipping) and
    [mp_]lamb_update_phase2 (bounds off and binding) at every chunk edge, bit for bit. r1 and r2
    are inputs, so nothing depends on a sum's association. rescale_grad 0.37 makes the 16-bit
    product of phase 1 round in float16 and bfloat16 alike."""
    rng = np.random.default_rng(n * 3 + DTYPES.index(dtype))
    mp = dtype != 'float32'
    T = Tensors(mx, rng, [n], dtype, master_skew=1e-3)
    t, d = T.h[0], T.d[0]
    L, kind = lib(), KIND[dtype]
    master = t['w32'] if mp else t['w']
    p1s = [dict(t=3, wd=0.01, rescale_grad=0.37, clip_gradient=0.4, beta1=0.9, beta2=0.98, epsilon=1e-6),
           dict(t=4, wd=0.02, rescale_grad=0.37, beta1=0.9, beta2=0.98, epsilon=1e-6, bias_correction=False)]
    for p1 in p1s:
        gout = mx.nd.zeros((n,), mx.gpu(0))
        op1 = 'mp_lamb_update_phase1' if mp else 'lamb_update_phase1'
        mx.nd._invoke(op1, [d[k] for k in T.names()], out=[gout], **p1)
        want = np.empty(n, np.float32)
        b1, b2 = sp(p1['beta1']), sp(p1['beta2'])
        L.kvo_lamb_phase1(n, P(want), P(t['mean']), P(t['var']), P(master),
                          None if mp else P(t['g']), P(t['g']) if mp else None, kind,
                          sp(p1.get('clip_gradient', -1.0)), sp(p1['rescale_grad']), b1,
                          K.Oracle.beta_pow(b1, p1['t']), b2, K.Oracle.beta_pow(b2, p1['t']),
                          sp(p1['wd']), sp(p1['epsilon']), int(p1.get('bias_correction', True)))
        T.check(op1, ('mean', 'var'))
        g = gout.asnumpy()
        assert same(g, want), op1
    r1 = np.float32(np.sqrt(np.dot(wide(t['w'], dtype).astype(np.float64), wide(t['w'], dtype))))
    r2 = np.float32(np.sqrt(np.dot(g.astype(np.float64), g)))
    op2 = 'mp_lamb_update_phase2' if mp else 'lamb_update_phase2'
    for bounds in ({}, dict(lower_bound=float(r1) * 2 + 0.5, upper_bound=float(r1) * 4 + 1),
                   dict(upper_bound=float(r1) / 2)):
        p2 = dict(lr=0.0031, **bounds)
        out = mx.nd.zeros((n,), mx.gpu(0), 'bfloat16' if dtype == 'bfloat16' else dtype)
        ins = [d['w'], mx.nd.array(g, mx.gpu(0)), mx.nd.array([r1], mx.gpu(0)),
               mx.nd.array([r2], mx.gpu(0))] + ([d['w32']] if mp else [])
        mx.nd._invoke(op2, ins, out=[out], **p2)
        want = np.empty(n, np.uint16 if mp else np.float32)
        L.kvo_lamb_phase2(n, None if mp else P(want), P(want) if mp else None, kind, P(master), P(g),
                          float(r1), float(r2), sp(p2['lr']), sp(bounds.get('lower_bound', -1.0)),
                          sp(bounds.get('upper_bound', -1.0)))
        assert same(down(out, dtype), want), (op2, bounds)
    # phase 2 writes only its output: the weight and (mp) the master copy stay as they were
    T.check('phase 2 inputs', ('w', 'w32') if mp else ('w',))


# ------------------------------------------------------------------------------------ multi LAMB
LAMB = dict(beta1=0.9, beta2=0.98, epsilon=1e-6, rescale_grad=0.37, clip_gradient=1.5)


def multi_lamb_check(mx, rng, sizes, dtype, bounds, zero=(), lrs=None, twice=False):
    """one _multi_[mp_]lamb_update call against the restatement: means and vars bit for bit; the
    weights within the bound of the trust ratio's two sums of squares. The expected weight is
    w - lr * (r1 / r2) * temp_g with temp_g from the restated step 1 and r1, r2 from float64
    norms; r1 is the norm of the weight INPUT (the 16-bit weights in the mp form, which is why
    the masters are skewed by 1e-3 from them). Returns the GPU results."""
    mp = dtype != 'float32'
    count = len(sizes)
    T = Tensors(mx, rng, sizes, dtype, master_skew=1e-3)
    for k in zero:
        T.h[k]['w'][...] = 0
        if mp:
            T.h[k]['w32'][...] = 0
        T.d[k] = {key: up(mx, v, T.dt(key)) for key, v in T.h[k].items()}
    norms = [float(np.sqrt(np.dot(wide(t['w'], dtype).astype(np.float64), wide(t['w'], dtype))))
             for t in T.h]
    if bounds == 'binding':
        nz = [x for x in norms if x > 0]
        bounds = dict(lower_bound=2 * min(nz), upper_bound=0.5 * max(nz))
        assert sum(x < bounds['lower_bound'] for x in nz) >= 1 and sum(x > bounds['upper_bound'] for x in nz) >= 1
    else:
        bounds = {}
    params = dict(LAMB, num_tensors=count, step_count=[k + 1 for k in range(count)],
                  learning_rates=lrs or [0.02 * (1 + k / 45.0) for k in range(count)],
                  wds=[0.001 * (1 + k) for k in range(count)], **bounds)
    op = '_multi_mp_lamb_update' if mp else '_multi_lamb_update'
    inputs = T.inputs()
    host_in = [{k: v.copy() for k, v in t.items()} for t in T.h] if twice else None
    mx.nd._invoke(op, inputs, out=[d['w'] for d in T.d], **params)
    got = [{k: down(d[k], T.dt(k)) for k in T.names()} for d in T.d]

    L, kind = lib(), KIND[dtype]
    lb, ub = sp(bounds.get('lower_bound', -1.0)), sp(bounds.get('upper_bound', -1.0))
    for k, t in enumerate(T.h):
        n = t['w'].size
        master = t['w32'] if mp else t['w']
        temp_g = np.empty(n, np.float32)
        L.kvo_multi_lamb_step1(n, P(temp_g), P(t['mean']), P(t['var']), P(master),
                               None if mp else P(t['g']), P(t['g']) if mp else None, kind,
                               sp(LAMB['clip_gradient']), sp(LAMB['rescale_grad']), sp(LAMB['beta1']),
                               sp(LAMB['beta2']), sp(LAMB['epsilon']), K.f32(params['wds'][k]),
                               params['step_count'][k], 1)
        assert same(got[k]['mean'], t['mean']), (k, n, 'mean')
        assert same(got[k]['var'], t['var']), (k, n, 'var')
        # trust ratio as multi_lamb.cc:79-118 computes it, from float64 sums
        r1 = np.float32(norms[k])
        r1 = max(r1, lb) if lb >= 0 else r1
        r1 = min(r1, ub) if ub >= 0 else r1
        r2 = math.sqrt(float(np.dot(temp_g.astype(np.float64), temp_g)))
        r = 1.0 if (r1 == 0 or r2 == 0) else float(r1) / r2
        step = K.f32(params['learning_rates'][k]) * r * temp_g.astype(np.float64)
        want = master.astype(np.float64) - step
        # two sums, two square roots, the division, lr * r and (lr * r) * temp_g; the final
        # subtraction rounds once more (the ulp term)
        eps_r = (sum_sq_rel_bound(n, mp) + sum_sq_rel_bound(n, False)) / 2 + 5 * U
        w_got = got[k]['w32'] if mp else got[k]['w']
        tol = np.abs(step) * eps_r + np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
        bad = np.abs(w_got.astype(np.float64) - want) > tol
        assert not bad.any(), (k, n, int(np.argmax(bad)), r)
        if mp:
            assert same(got[k]['w'], narrow(got[k]['w32'], dtype)), (k, n, '16-bit weight')
    if twice:
        # the same call on equal inputs gives the same bits: the sums are deterministic
        for t, src in zip(T.h, host_in):
            t.update(src)
        T.d = [{k: up(mx, v, T.dt(k)) for k, v in t.items()} for t in T.h]
        mx.nd._invoke(op, T.inputs(), out=[d['w'] for d in T.d], **params)
        for k, d in enumerate(T.d):
            for key in T.names():
                assert same(down(d[key], T.dt(key)), got[k][key]), ('second call', k, key)
    return got


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", SIZES)
def test_multi_lamb_chunk_edges(mx, n, dtype):
    rng = np.random.default_rng(n + 7 * DTYPES.index(dtype))
    multi_lamb_check(mx, rng, [n, 4, n], dtype, None)


@pytest.mark.parametrize("bounds", ["off", "binding"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_multi_lamb_45_tensors(mx, dtype, bounds):
    """_multi_[mp_]lamb_update at its limit of 45 tensors: three of over 20 chunks, one all-zero
    weight (trust ratio 1 without bounds), one empty tensor, a distinct step count, lr and wd per
    tensor; the same call twice gives the same bits"""
    rng = np.random.default_rng(45 + DTYPES.index(dtype) + (bounds == 'binding'))
    sizes = [int(s) for s in rng.integers(1, 30000, 45)]
    sizes[3], sizes[20], sizes[44] = 21 * CHUNK + 5, 25 * CHUNK + 4099, 40 * CHUNK
    sizes[7], sizes[9], sizes[10], sizes[11] = 0, 1, CHUNK, CHUNK + 1
    multi_lamb_check(mx, rng, sizes, dtype, bounds, zero=(12,), twice=True)


def test_multi_lamb_bert_sized(mx):
    """a BERT-base-like float16 parameter set (word embedding, one encoder layer, pooler: 31 M
    elements) through _multi_mp_lamb_update in one call"""
    h = 768
    sizes = [30522 * h, 512 * h, 2 * h, h, h] + [h * h, h] * 4 + [h, h, h * 4 * h, 4 * h, 4 * h * h, h, h, h] + \
        [h * h, h]
    assert len(sizes) <= 45 and sum(sizes) > 30e6
    multi_lamb_check(mx, np.random.default_rng(12), sizes, 'float16', None, lrs=[0.01] * len(sizes))


def test_multi_tensor_count_limits(mx):
    """46 LAMB tensors and 0 LAMB tensors / AdamW weights are refused with an MXNetError"""
    w = [mx.nd.zeros((3,), mx.gpu(0)) for _ in range(46 * 4)]
    with pytest.raises(mx.MXNetError):
        mx.nd._invoke('_multi_lamb_update', w, out=w[0::4], num_tensors=46, learning_rates=[0.1] * 46,
                      wds=[0.0] * 46, step_count=[1] * 46)
    with pytest.raises(mx.MXNetError):
        mx.nd._invoke('_multi_lamb_update', [], num_tensors=0, learning_rates=[], wds=[], step_count=[])
    with pytest.raises(mx.MXNetError):
        mx.nd._invoke('_multi_mp_lamb_update', [], num_tensors=0, learning_rates=[], wds=[],
                      step_count=[])
    rescale = mx.nd.array([1.0], mx.gpu(0))
    for op in ('_multi_adamw_update', '_multi_mp_adamw_update'):
        with pytest.raises(mx.MXNetError):
            mx.nd._invoke(op, [rescale], num_weights=0, lrs=[], wds=[], etas=[])


# --------------------------------------------------------------------------------- alignment
@pytest.mark.parametrize("which", ["all", "var"])
@pytest.mark.parametrize("offset", [1, 2, 4])
@pytest.mark.parametrize("dtype", DTYPES)
def test_misaligned_views(mx, dtype, offset, which):
    """operands that are views starting `offset` elements into a padded base (every operand, or
    only var): float32 at 1 or 2 elements and 16-bit at 1 or 2 are not vector-aligned, so the
    tensor takes the scalar path; 16-bit at 4 (8 bytes) and float32 at 4 (16 bytes) keep the
    vector path. The results are those of aligned operands, and the padding stays untouched."""
    n, pad = 2 * CHUNK + 4099, 3
    rng = np.random.default_rng(offset * 2 + (which == 'var') + 10 * DTYPES.index(dtype))
    T = Tensors(mx, rng, [n], dtype)
    t = T.h[0]
    bases = {}
    for k in T.names():
        off = offset if (which == 'all' or k == 'var') else 0
        head, tail = rand(rng, off, T.dt(k)), rand(rng, pad, T.dt(k))
        bases[k] = (head, tail, up(mx, np.concatenate([head, t[k], tail]), T.dt(k)))
        T.d[0][k] = bases[k][2][off:off + n]
    params = adamw_params(True, 1)
    adamw_gpu(mx, T, True, 0.37, params)
    adamw_oracle(T, True, 0.37, params)
    T.check('views')
    for k, (head, tail, base) in bases.items():
        b = down(base, T.dt(k))
        assert same(b[:head.size], head) and same(b[b.size - pad:], tail), (k, 'padding written')
    # the reducing kernel on a misaligned view
    x = T.h[0]['w']
    got = mx.nd.multi_sum_sq(T.d[0]['w'], num_arrays=1).asnumpy()
    _check_sum_sq(got, [x], dtype)


# -------------------------------------------------------------------------------- plan cache
def test_plan_cache_keeps_dtypes_apart(mx):
    """one buffer viewed as float16, then as float32, at the same 8-byte (not 16-byte) aligned
    address and element count: the float16 tensor is vectorised, the float32 one must not be, so
    the two calls must not share a cached table"""
    import torch
    n = MULTI
    rng = np.random.default_rng(3)
    buf = torch.zeros(4 * n + 64, dtype=torch.uint8, device='cuda')
    off = 8 + (-buf.data_ptr()) % 16
    assert (buf.data_ptr() + off) % 16 == 8
    h16 = rand(rng, n, 'float16')
    v16 = buf[off:off + 2 * n].view(torch.float16)
    v16.copy_(torch.from_numpy(h16.view(np.float16)).cuda())
    torch.cuda.synchronize()
    got16 = mx.nd.multi_sum_sq(mx.nd.from_torch(v16), num_arrays=1).asnumpy()
    _check_sum_sq(got16, [h16], 'float16')
    h32 = rand(rng, n, 'float32')
    v32 = buf[off:off + 4 * n].view(torch.float32)
    v32.copy_(torch.from_numpy(h32).cuda())
    torch.cuda.synchronize()
    got32 = mx.nd.multi_sum_sq(mx.nd.from_torch(v32), num_arrays=1).asnumpy()
    _check_sum_sq(got32, [h32], 'float32')


def test_plan_cache_eviction_in_flight(mx):
    """600 distinct plans with no synchronisation in between (the cache is cleared after 512
    while earlier launches may still be queued), then an early signature again"""
    m, count = MULTI, 600
    rng = np.random.default_rng(5)
    x = rng.uniform(-1, 1, m + count).astype(np.float32)
    base = up(mx, x)
    outs = [mx.nd.multi_sum_sq(base[k:k + m], num_arrays=1) for k in range(count)]
    again = [mx.nd.multi_sum_sq(base[k:k + m], num_arrays=1) for k in (0, 1)]
    x64 = x.astype(np.float64)
    bound = sum_sq_rel_bound(m, False)
    for k, o in list(enumerate(outs)) + list(zip((0, 1), again)):
        exact = float(np.dot(x64[k:k + m], x64[k:k + m]))
        assert abs(float(o.asnumpy()[0]) - exact) <= bound * exact, k
    assert same(again[0].asnumpy(), outs[0].asnumpy()) and same(again[1].asnumpy(), outs[1].asnumpy())


# --------------------------------------------------------------------------------- multi_lars
def test_multi_lars_1000(mx):
    """multi_lars over 1000 tensors (8 blocks of 128 threads), zero weight norms and zero
    gradient norms interleaved, eps = 0, bit for bit"""
    n = 1000
    rng = np.random.default_rng(1000)
    lrs = rng.uniform(0.01, 1, n).astype(np.float32)
    wsq = rng.uniform(0, 50, n).astype(np.float32)
    gsq = rng.uniform(0, 50, n).astype(np.float32)
    wds = rng.uniform(0, 0.01, n).astype(np.float32)
    wsq[0::3] = 0
    gsq[1::4] = 0
    wds[2::5] = 0
    params = dict(eta=0.0013, eps=0.0, rescale_grad=0.37)
    out = mx.nd.zeros((n,), mx.gpu(0))
    mx.nd._invoke('multi_lars', [up(mx, a) for a in (lrs, wsq, gsq, wds)], out=[out], **params)
    want = K.get_oracle().multi_lars(lrs, wsq, gsq, wds, sp(params['eta']), sp(params['eps']),
                                     sp(params['rescale_grad']))
    assert same(out.asnumpy(), want)


# ------------------------------------------------------------------------------ the 2^32 edge
@pytest.mark.parametrize("n", [2 ** 32 - 1, 2 ** 32 - CHUNK])
def test_sum_sq_near_2_pow_32_elements(mx, n):
    """multi_sum_sq on one float16 array of just under 2^32 elements: ones, and 64 in the last
    chunk. Every partial and every fold is then a multiple of 4096 below 2^33, which float32
    holds exactly whatever the association, so the sum is exact."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 12 * 2 ** 30:
        pytest.skip("needs 12 GiB of free device memory, %.1f GiB free" % (free / 2 ** 30))
    last = n - (n - 1) // CHUNK * CHUNK   # elements in the last chunk
    x = torch.ones(n, dtype=torch.float16, device='cuda')
    x[n - last:] = 64.0
    torch.cuda.synchronize()
    try:
        got = mx.nd.multi_sum_sq(mx.nd.from_torch(x), num_arrays=1).asnumpy()[0]
    finally:
        del x
        torch.cuda.empty_cache()
    assert float(got) == float((n - last) + last * 4096)
