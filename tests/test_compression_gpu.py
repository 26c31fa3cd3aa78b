"""2-bit gradient compression with residual on the device store (SURVEY.md 8f-f2): reference
semantics from src/kvstore/comm.h:552-596 + gradient_compression-inl.h:40-132, pinned by the
reference's own kernels through tests/golden/twobit.npz; the nightly test
(tests/nightly/test_kvstore.py:100-212) is the model for the multi-step residual checks.

Every merged gradient is compared bit for bit with the oracle's quantize_2bit / dequantize_2bit and
its 'device' left fold (ElementwiseSum order), at the threshold the store really uses: str(t)
through dmlc::stof. Thresholds 0.1 and 1/3 make the sum of the decoded sources depend on its order
(tests/test_compression_host.py shows that for every case below), 0.25 does not."""
import numpy as np
import pytest

import kvoracle as K

pytestmark = pytest.mark.gpu

# both kernels cap their grid at 132 SMs x 8 CTAs of 256 threads (compress_kernels.cu, GridFor):
# the decode runs one thread per element, the quantize one thread per 16-element word
GRID_THREADS = 132 * 8 * 256
DECODE_GRID_ELEMS = GRID_THREADS            # 270 336
QUANTIZE_GRID_ELEMS = GRID_THREADS * 16     # 4 325 376


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def store_threshold(t):
    """the float the store compresses with: set_gradient_compression passes str(t) to dmlc::stof"""
    return K.dmlc_stof(str(t))


def merge(o, grads, res, thr):
    """quantise every source with its residual (res[i] moves), decode, sum in the store's order"""
    n = grads[0].size
    deq = [o.dequantize_2bit(o.quantize_2bit(g.ravel(), r, thr), n, thr) for g, r in zip(grads, res)]
    return o.reduce(deq, 'device'), deq


def compressed_store(mx, t):
    kv = mx.kv.create('device')
    kv.set_gradient_compression({'type': '2bit', 'threshold': t})
    return kv


def test_twobit_golden_through_store(mx, golden):
    g = golden("twobit")
    grad = g["grad"]
    kv = mx.kv.create('device')
    kv.set_gradient_compression({'type': '2bit', 'threshold': 0.5})
    kv.init(0, mx.nd.zeros(grad.shape, mx.gpu(0)))
    out = mx.nd.empty(grad.shape, mx.gpu(0))
    kv.push(0, mx.nd.array(grad, mx.gpu(0)))
    kv.pull(0, out=out)
    assert eq(out.asnumpy(), g["deq1"])                      # decode of the reference's comp1


def test_twobit_with_optimizer_and_errors(mx, oracle):
    rng = np.random.default_rng(60)
    n = 4099
    kv = mx.kv.create('device')
    kv.set_gradient_compression({'type': '2bit', 'threshold': 0.5})
    w = rng.uniform(-1, 1, n).astype(np.float32)
    kv.init(0, mx.nd.array(w, mx.gpu(0)))
    kv.set_optimizer(mx.optimizer.Test(rescale_grad=1.0))
    res = np.zeros(n, np.float32)
    out = mx.nd.empty((n,), mx.gpu(0))
    for step in range(3):
        g = rng.uniform(-1, 1, n).astype(np.float32)
        kv.pushpull(0, mx.nd.array(g, mx.gpu(0)), out=out)
        comp = oracle.quantize_2bit(g, res, 0.5)
        w = w + oracle.dequantize_2bit(comp, n, 0.5)          # Test optimizer: w += 1.0 * merged
        assert eq(out.asnumpy(), w), step
    with pytest.raises(mx.MXNetError, match="Unknown type"):
        kv.set_gradient_compression({'type': '1bit'})
    with pytest.raises(Exception, match="not supported"):
        mx.kv.create('local').set_gradient_compression({'type': '2bit'})


# ------------------------------------------------------------------ order-sensitive sums
ORDER_THRESHOLDS = [0.25, 0.1, 1 / 3]
ORDER_NSRC = [1, 2, 3, 4, 5, 8, 9, 16]
ORDER_SHAPES = [(1,), (15,), (16,), (17,), (4099,), (1003,), (64, 33), (5,)]
ORDER_STEPS = 4


def order_grads(t, nsrc, step):
    """the gradients of one step of test_twobit_residual_over_steps: [key][source]"""
    rng = np.random.default_rng([50, nsrc, step, ORDER_THRESHOLDS.index(t)])
    a = np.float32(1.6 * t)
    return [[rng.uniform(-a, a, s).astype(np.float32) for _ in range(nsrc)] for s in ORDER_SHAPES]


def order_trajectory(o, t, nsrc):
    """per step: (gradients [key][source], decoded sources [key][source]) of the oracle, with each
    source's residual carried from step to step"""
    thr = store_threshold(t)
    res = [[np.zeros(int(np.prod(s)), np.float32) for _ in range(nsrc)] for s in ORDER_SHAPES]
    for step in range(ORDER_STEPS):
        grads = order_grads(t, nsrc, step)
        yield grads, [merge(o, grads[k], res[k], thr)[1] for k in range(len(ORDER_SHAPES))]


@pytest.mark.parametrize("t", ORDER_THRESHOLDS, ids=["t0.25", "t0.1", "t1_3"])
@pytest.mark.parametrize("nsrc", ORDER_NSRC)
def test_twobit_residual_over_steps(mx, oracle, nsrc, t):
    kv = compressed_store(mx, t)
    keys = list(range(len(ORDER_SHAPES)))
    kv.init(keys, [mx.nd.zeros(s, mx.gpu(0)) for s in ORDER_SHAPES])
    outs = [mx.nd.empty(s, mx.gpu(0)) for s in ORDER_SHAPES]
    for step, (grads, deq) in enumerate(order_trajectory(oracle, t, nsrc)):
        kv.push(keys, [[mx.nd.array(a, mx.gpu(0)) for a in gs] for gs in grads])
        kv.pull(keys, out=outs)
        for k in keys:
            assert eq(outs[k].asnumpy().ravel(), oracle.reduce(deq[k], 'device')), (step, k)


# ------------------------------------------------------------------ past one grid
@pytest.mark.parametrize("n,nsrc", [(QUANTIZE_GRID_ELEMS + 4099, 2), (DECODE_GRID_ELEMS + 5, 16)])
def test_twobit_past_one_grid(mx, oracle, n, nsrc):
    """both grid-stride loops take a second trip (the first case), the decode with 16 sources"""
    t = 0.1
    thr = store_threshold(t)
    rng = np.random.default_rng(n + nsrc)
    kv = compressed_store(mx, t)
    kv.init(0, mx.nd.zeros((n,), mx.gpu(0)))
    out = mx.nd.empty((n,), mx.gpu(0))
    res = [np.zeros(n, np.float32) for _ in range(nsrc)]
    for step in range(2):
        grads = [rng.uniform(-0.16, 0.16, n).astype(np.float32) for _ in range(nsrc)]
        kv.pushpull(0, [mx.nd.array(g, mx.gpu(0)) for g in grads], out=out)
        want, _ = merge(oracle, grads, res, thr)
        got = out.asnumpy()
        assert eq(got, want), (step, int(np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))[0]))


# ------------------------------------------------------------------ edge values
def edge_values(thr):
    """16 values of gradient + residual: on, inside and outside +-t, half of +-t (carried onto the
    threshold by the next step), signed zeros, infinities, NaN and subnormals"""
    f = np.float32
    t = f(thr)
    sub = np.finfo(f).smallest_subnormal
    return np.array([t, -t, np.nextafter(t, f(0)), np.nextafter(t, f(np.inf)),
                     np.nextafter(-t, f(0)), np.nextafter(-t, f(-np.inf)), t / f(2), -t / f(2),
                     f(0.0), f(-0.0), f(np.inf), f(-np.inf), f(np.nan),
                     sub, -sub, np.nextafter(np.finfo(f).tiny, f(0))], f)


@pytest.mark.parametrize("t", [0.1, 1 / 3, 0.5, 1.2345e-05], ids=["t0.1", "t1_3", "t0.5", "t1.2345e-05"])
def test_twobit_edge_values(mx, oracle, t):
    """the edge values fill the first and a middle 16-element word and 15 of them the last,
    partial, word (each source rotated differently); step 2 pushes them again, step 3 random
    values, so the residuals carry them. What NaN and inf do is what the oracle's C code does.
    dmlc::stof parses 1.2345e-05 one float above its nearest float32: a store that compressed with
    the nearest float would fire on the value one ulp below the threshold."""
    thr = store_threshold(t)
    nsrc, words = 3, 41
    n = 16 * (words - 1) + 15
    edges = edge_values(thr)
    rng = np.random.default_rng(77)
    base = [rng.uniform(-1.5 * thr, 1.5 * thr, n).astype(np.float32) for _ in range(nsrc)]
    for s in range(nsrc):
        base[s][0:16] = np.roll(edges, s)
        base[s][16 * 20:16 * 21] = np.roll(edges, s + 5)
        base[s][16 * (words - 1):] = np.roll(edges, s + 9)[:15]
    steps = [base, base, [rng.uniform(-1.5 * thr, 1.5 * thr, n).astype(np.float32) for _ in range(nsrc)]]
    kv = compressed_store(mx, t)
    kv.init(0, mx.nd.zeros((n,), mx.gpu(0)))
    out = mx.nd.empty((n,), mx.gpu(0))
    res = [np.zeros(n, np.float32) for _ in range(nsrc)]
    for step, grads in enumerate(steps):
        kv.pushpull(0, [mx.nd.array(g, mx.gpu(0)) for g in grads], out=out)
        want, _ = merge(oracle, grads, res, thr)
        assert eq(out.asnumpy(), want), step


# ------------------------------------------------------------------ the merged gradient downstream
DOWN_SHAPES = [(4099,), (64, 33), (17,)]


def _optimizer(mx, route):
    if route == 'sgd':
        return mx.optimizer.SGD(learning_rate=0.1, wd=1e-4, rescale_grad=0.25), \
            dict(kind='sgd', lr=0.1, wd=1e-4, rescale_grad=0.25)
    if route == 'sgd_mom':
        return mx.optimizer.SGD(learning_rate=0.1, momentum=0.9, wd=1e-4, rescale_grad=0.25), \
            dict(kind='sgd', lr=0.1, momentum=0.9, wd=1e-4, rescale_grad=0.25)
    if route == 'adam':
        return mx.optimizer.Adam(learning_rate=1e-3, wd=0.01, rescale_grad=0.25), \
            dict(kind='adam', lr=1e-3, wd=0.01, rescale_grad=0.25)
    raise ValueError(route)


@pytest.mark.parametrize("route", ['sgd', 'sgd_mom', 'adam', 'nag_callback', 'local_update'])
def test_twobit_merged_gradient_downstream(mx, oracle, route):
    """the fused SGD / SGD-momentum / Adam steps and the per-key updater callback (the NAG mirror)
    run on the decoded sum; with update_on_kvstore=False the pull returns that sum itself"""
    import golden_update_ops as GU
    t, nsrc = 1 / 3, 4
    thr = store_threshold(t)
    rng = np.random.default_rng(61)
    kv = compressed_store(mx, t)
    keys = list(range(len(DOWN_SHAPES)))
    w = [rng.uniform(-1, 1, s).astype(np.float32) for s in DOWN_SHAPES]
    kv.init(keys, [mx.nd.array(x, mx.gpu(0)) for x in w])
    model = K.LocalKVStoreModel('device')
    for k in keys:
        model.init(k, w[k])
    nag = dict(lr=0.05, momentum=0.9, wd=1e-3, rescale_grad=0.5)
    mom = [np.zeros(s, np.float32) for s in DOWN_SHAPES]
    if route == 'nag_callback':
        from compat import mxnet_optimizer_update as mxopt
        kv.set_optimizer(mxopt.NAG(learning_rate=nag['lr'], momentum=nag['momentum'], wd=nag['wd'],
                                   rescale_grad=nag['rescale_grad']))
        assert kv._fused is None
    elif route != 'local_update':
        opt, kw = _optimizer(mx, route)
        kv.set_optimizer(opt)
        model.set_optimizer(**kw)
    res = [[np.zeros(int(np.prod(s)), np.float32) for _ in range(nsrc)] for s in DOWN_SHAPES]
    outs = [mx.nd.empty(s, mx.gpu(0)) for s in DOWN_SHAPES]
    for step in range(3):
        grads = [[rng.uniform(-0.5, 0.5, s).astype(np.float32) for _ in range(nsrc)] for s in DOWN_SHAPES]
        kv.pushpull(keys, [[mx.nd.array(g, mx.gpu(0)) for g in gs] for gs in grads], out=outs)
        for k, s in enumerate(DOWN_SHAPES):
            merged = merge(oracle, grads[k], res[k], thr)[0].reshape(s)
            if route == 'nag_callback':
                w[k], (mom[k],) = GU.restate('nag_mom_update', [w[k], merged, mom[k]], nag)
                want = w[k]
            else:
                model.push(k, [merged])
                want = model.pull(k)
            assert eq(outs[k].asnumpy(), want), (step, k)


# ------------------------------------------------------------------ host values and call patterns
@pytest.mark.parametrize("placement", ['cpu', 'cpu_gpu_cpu'])
def test_twobit_host_values(mx, oracle, placement):
    """values in host memory are staged to the key's GPU before they are quantised"""
    t = 1 / 3
    thr = store_threshold(t)
    rng = np.random.default_rng(62)
    ctxs = [mx.cpu(0), mx.cpu(1), mx.cpu(2)] if placement == 'cpu' else [mx.cpu(0), mx.gpu(0), mx.cpu(1)]
    kv = compressed_store(mx, t)
    keys = list(range(len(DOWN_SHAPES)))
    kv.init(keys, [mx.nd.zeros(s, mx.gpu(0)) for s in DOWN_SHAPES])
    res = [[np.zeros(int(np.prod(s)), np.float32) for _ in ctxs] for s in DOWN_SHAPES]
    outs = [mx.nd.empty(s, mx.gpu(0)) for s in DOWN_SHAPES]
    for step in range(3):
        grads = [[rng.uniform(-0.5, 0.5, s).astype(np.float32) for _ in ctxs] for s in DOWN_SHAPES]
        kv.pushpull(keys, [[mx.nd.array(g, c) for g, c in zip(gs, ctxs)] for gs in grads], out=outs)
        for k in keys:
            want = merge(oracle, grads[k], res[k], thr)[0]
            assert eq(outs[k].asnumpy().ravel(), want), (step, k)


def test_twobit_source_count_changes(mx, oracle):
    """one key pushed with 4, then 2, then 4 values: residual i belongs to value position i, and
    the residuals the first call allocated carry through the shorter call"""
    t = 0.1
    thr = store_threshold(t)
    rng = np.random.default_rng(63)
    kv = compressed_store(mx, t)
    keys = [0, 1]
    shapes = [(4099,), (17,)]
    kv.init(keys, [mx.nd.zeros(s, mx.gpu(0)) for s in shapes])
    res = [[np.zeros(int(np.prod(s)), np.float32) for _ in range(4)] for s in shapes]
    outs = [mx.nd.empty(s, mx.gpu(0)) for s in shapes]
    for step, nsrc in enumerate([4, 2, 4, 2]):
        grads = [[rng.uniform(-0.16, 0.16, s).astype(np.float32) for _ in range(nsrc)] for s in shapes]
        kv.pushpull(keys, [[mx.nd.array(g, mx.gpu(0)) for g in gs] for gs in grads], out=outs)
        for k in keys:
            want = merge(oracle, grads[k], res[k][:nsrc], thr)[0]
            assert eq(outs[k].asnumpy().ravel(), want), (step, k)


def test_twobit_per_key_calls_equal_one_call(mx, oracle):
    """the per-parameter pattern of gluon.Trainer (one pushpull per key, bucketing queue enabled)
    gives the bits of one call that carries every key, and both those of the oracle"""
    import ctypes
    t = 1 / 3
    thr = store_threshold(t)
    rng = np.random.default_rng(64)
    shapes = DOWN_SHAPES + [(16,), (1,)]
    keys = list(range(len(shapes)))
    w0 = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]
    stores = []
    for _ in range(2):
        kv = compressed_store(mx, t)
        kv.init(keys, [mx.nd.array(x, mx.gpu(0)) for x in w0])
        kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9, wd=1e-4, rescale_grad=0.25))
        stores.append(kv)
    mx.base.check_call(mx.base._LIB.B200KVStoreSetBucketBytes(stores[0].handle, ctypes.c_size_t(1 << 30)))
    model = K.LocalKVStoreModel('device')
    for k in keys:
        model.init(k, w0[k])
    model.set_optimizer('sgd', lr=0.1, momentum=0.9, wd=1e-4, rescale_grad=0.25)
    res = [[np.zeros(int(np.prod(s)), np.float32) for _ in range(3)] for s in shapes]
    outs = [[mx.nd.empty(s, mx.gpu(0)) for s in shapes] for _ in stores]
    for step in range(3):
        grads = [[rng.uniform(-0.5, 0.5, s).astype(np.float32) for _ in range(3)] for s in shapes]
        vals = [[mx.nd.array(g, mx.gpu(0)) for g in gs] for gs in grads]
        for k in keys:
            stores[0].pushpull(k, vals[k], out=outs[0][k], priority=-k)
        stores[1].pushpull(keys, vals, out=outs[1])
        for k in keys:
            model.push(k, [merge(oracle, grads[k], res[k], thr)[0].reshape(shapes[k])])
            want = model.pull(k)
            assert eq(outs[0][k].asnumpy(), want) and eq(outs[1][k].asnumpy(), want), (step, k)


# ------------------------------------------------------------------ refused calls change nothing
REF_SHAPES = [(4099,), (17,)]
REF_NSRC = 4


def _refused_call(mx, kv, case, good):
    """one call the store must refuse; `good` are this step's valid values [key][source]"""
    ctx = mx.gpu(0)
    dev = [[mx.nd.array(g, ctx) for g in gs] for gs in good]

    def swap_last(k, arr):
        vals = [list(v) for v in dev]
        vals[k][-1] = arr
        return vals
    if case == 'seventeen_values':
        kv.push(0, [mx.nd.array(good[0][i % REF_NSRC], ctx) for i in range(17)])
    elif case in ('float16_value', 'float64_value'):
        dt = case.split('_')[0]
        kv.push([0, 1], swap_last(1, mx.nd.array(good[1][-1].astype(dt), ctx, dt)))
    elif case == 'size_first_key':
        kv.push([0, 1], swap_last(0, mx.nd.array(good[0][-1][:-1], ctx)))
    elif case == 'size_second_key':
        kv.push([0, 1], swap_last(1, mx.nd.array(good[1][-1][:-1], ctx)))
    elif case == 'float16_key':
        kv.push([0, 2], [dev[0], [mx.nd.zeros((33,), ctx, 'float16') for _ in range(REF_NSRC)]])
    else:
        raise ValueError(case)


REFUSALS = {
    'seventeen_values': "at most 16 values per key and push",
    'float16_value': "push: dtype mismatch for key 1",
    'float64_value': "push: dtype mismatch for key 1",
    'size_first_key': "push: shape mismatch for key 0",
    'size_second_key': "push: shape mismatch for key 1",
    'float16_key': "2-bit gradient compression needs float32 gradients",
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
@pytest.mark.parametrize("store", ['assign', 'sgd_mom'])
def test_twobit_refused_call_changes_nothing(mx, oracle, case, store):
    """a valid step, one refused call, a valid step: the second step's merged gradient (pulled
    back with no optimizer) and weights (SGD-momentum) are those of the oracle trajectory that
    never saw the refused call -- no residual moved"""
    t = 1 / 3
    thr = store_threshold(t)
    rng = np.random.default_rng(65)
    ctx = mx.gpu(0)
    kv = compressed_store(mx, t)
    w0 = [rng.uniform(-1, 1, s).astype(np.float32) for s in REF_SHAPES]
    kv.init([0, 1], [mx.nd.array(x, ctx) for x in w0])
    kv.init(2, mx.nd.zeros((33,), ctx, 'float16'))
    model = K.LocalKVStoreModel('device')
    for k in (0, 1):
        model.init(k, w0[k])
    if store == 'sgd_mom':
        kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9, wd=1e-4, rescale_grad=0.25))
        model.set_optimizer('sgd', lr=0.1, momentum=0.9, wd=1e-4, rescale_grad=0.25)
    res = [[np.zeros(int(np.prod(s)), np.float32) for _ in range(REF_NSRC)] for s in REF_SHAPES]
    outs = [mx.nd.empty(s, ctx) for s in REF_SHAPES]
    for step in range(2):
        grads = [[rng.uniform(-0.5, 0.5, s).astype(np.float32) for _ in range(REF_NSRC)] for s in REF_SHAPES]
        if step == 1:
            with pytest.raises(mx.MXNetError) as err:
                _refused_call(mx, kv, case, grads)
        kv.pushpull([0, 1], [[mx.nd.array(g, ctx) for g in gs] for gs in grads], out=outs)
        for k in (0, 1):
            model.push(k, [merge(oracle, grads[k], res[k], thr)[0].reshape(REF_SHAPES[k])])
            assert eq(outs[k].asnumpy(), model.pull(k)), (step, k)
    assert REFUSALS[case] in str(err.value)
