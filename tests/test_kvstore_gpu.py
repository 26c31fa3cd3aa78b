"""GPU parity tests of the dense KVStore path, through the C ABI (ctypes front-end).

Structure follows the reference's own tests: tests/python/unittest/test_kvstore.py (init / push /
pull / aggregation over several values of a key / str keys / updater / error cases),
tests/python/gpu/test_device.py (ones over n values == n, 7 shapes) and
tests/nightly/test_kvstore.py (random data, 'test' optimizer). The checker is the CPU oracle
(oracle/kvoracle.c, pinned to the reference); comparisons are BIT-EXACT, which is stronger than the
1e-6 relative bound the reference's nightly test and north_star ask for.
"""
import numpy as np
import pytest

import kvoracle as K

pytestmark = pytest.mark.gpu

SHAPES = [(4, 4), (100, 100), (3,), (1027,), (4099, 3), (2000, 2000)]


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def rnd(rng, shape):
    return rng.uniform(-1, 1, shape).astype(np.float32)


# ------------------------------------------------------------------ plumbing (test_kvstore.py)
def test_single_kv_pair(mx):
    for name in ('local', 'device'):
        kv = mx.kv.create(name)
        assert kv.type == name and kv.rank == 0 and kv.num_workers == 1
        kv.init(3, mx.nd.zeros((4, 4), mx.gpu(0)))
        kv.push(3, mx.nd.ones((4, 4), mx.gpu(0)))
        val = mx.nd.empty((4, 4), mx.gpu(0))
        kv.pull(3, out=val)
        assert np.all(val.asnumpy() == 1)


def test_init_pull_keeps_value(mx):
    kv = mx.kv.create('device')
    v = np.arange(12, dtype=np.float32).reshape(3, 4)
    kv.init('w', mx.nd.array(v, mx.cpu()))          # host-resident init value
    out = [mx.nd.empty((3, 4), mx.gpu(0)) for _ in range(3)]
    kv.pull('w', out=out)
    for o in out:
        assert eq(o.asnumpy(), v)


def test_list_kv_pair_and_str_keys(mx):
    for keys in ([5, 7, 9], ['b', 'c', 'd']):
        kv = mx.kv.create('local')
        kv.init(keys, [mx.nd.zeros((4, 4), mx.gpu(0))] * len(keys))
        kv.push(keys, [mx.nd.ones((4, 4), mx.gpu(0)) * 4] * len(keys))
        val = [mx.nd.empty((4, 4), mx.gpu(0))] * len(keys)
        kv.pull(keys, out=val)
        for v in val:
            assert np.all(v.asnumpy() == 4)


@pytest.mark.parametrize("kvtype", ['local', 'device'])
def test_aggregator_ones(mx, kvtype):
    # test_device.py:38-71 / test_kvstore.py:129-176: n values of a key -> n
    kv = mx.kv.create(kvtype)
    shapes = [(10,), (100, 50), (2, 3, 4, 5, 6, 7, 8)]
    for k, s in enumerate(shapes):
        kv.init(k, mx.nd.zeros(s, mx.gpu(0)))
    for n in (1, 2, 3, 4, 8):
        for k, s in enumerate(shapes):
            vals = [mx.nd.ones(s, mx.gpu(0)) for _ in range(n)]
            outs = [mx.nd.empty(s, mx.gpu(0)) for _ in range(n)]
            kv.push(k, vals)
            kv.pull(k, out=outs)
            for o in outs:
                assert np.all(o.asnumpy() == n)


def test_updater_callback(mx):
    # test_kvstore.py:227-279: updater `local += recv`, four pushes over four values
    def updater(key, recv, local):
        local += recv
    for keys in ([3], ['a', 'b']):
        kv = mx.kv.create('local')
        kv._set_updater(updater)
        kv.init(keys, [mx.nd.ones((4, 4), mx.gpu(0))] * len(keys))
        for _ in range(4):
            kv.push(keys, [[mx.nd.ones((4, 4), mx.gpu(0))] * 4] * len(keys))
        outs = [mx.nd.empty((4, 4), mx.gpu(0)) for _ in keys]
        kv.pull(keys, out=outs)
        for o in outs:
            assert np.all(o.asnumpy() == 17)


def test_error_cases(mx):
    # test_kvstore.py:288-345
    kv = mx.kv.create('local')
    kv.init(1, mx.nd.zeros((2, 2), mx.gpu(0)))
    with pytest.raises(mx.MXNetError, match="duplicate init"):
        kv.init(1, mx.nd.zeros((2, 2), mx.gpu(0)))
    with pytest.raises(mx.MXNetError, match="has not been inited"):
        kv.push(2, mx.nd.zeros((2, 2), mx.gpu(0)))
    with pytest.raises(mx.MXNetError, match="has not been inited"):
        kv.pull(2, out=mx.nd.zeros((2, 2), mx.gpu(0)))
    with pytest.raises(mx.MXNetError, match="Mixed key types"):
        kv.init('a', mx.nd.zeros((2, 2), mx.gpu(0)))
    with pytest.raises(mx.MXNetError, match="shape mismatch"):
        kv.push(1, mx.nd.zeros((3, 2), mx.gpu(0)))
    with pytest.raises(mx.MXNetError):
        mx.kv.create('dist_sync')


# ------------------------------------------------------------------ reduce parity vs oracle
@pytest.mark.parametrize("kvtype,order", [('local', 'local'), ('device', 'device')])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 8, 9, 16])
def test_reduce_bit_exact(mx, oracle, kvtype, order, n):
    rng = np.random.default_rng(100 + n)
    kv = mx.kv.create(kvtype)
    for k, s in enumerate(SHAPES):
        kv.init(k, mx.nd.zeros(s, mx.gpu(0)))
    srcs = {k: [rnd(rng, s) for _ in range(n)] for k, s in enumerate(SHAPES)}
    keys = list(range(len(SHAPES)))
    vals = [[mx.nd.array(a, mx.gpu(0)) for a in srcs[k]] for k in keys]
    outs = [mx.nd.empty(s, mx.gpu(0)) for s in SHAPES]
    kv.pushpull(keys, vals, out=outs)        # grouped call: ONE fused launch
    for k in keys:
        assert eq(outs[k].asnumpy().ravel(), oracle.reduce(srcs[k], order)), (k, n)
    # per-key push then pull (tools/bandwidth/measure.py:112-122 call pattern)
    for k in keys:
        kv.push(k, vals[k], priority=-k)
        o = mx.nd.empty(SHAPES[k], mx.gpu(0))
        kv.pull(k, out=o, priority=-k)
        assert eq(o.asnumpy().ravel(), oracle.reduce(srcs[k], order))


def test_reduce_golden_fixture(mx, golden):
    g = golden("reduce_local")
    kv = mx.kv.create('local')
    for n in range(1, 10):
        src = g["n%d_src" % n]
        kv.init(n, mx.nd.zeros(src[0].shape, mx.gpu(0)))
        out = mx.nd.empty(src[0].shape, mx.gpu(0))
        kv.pushpull(n, [mx.nd.array(s, mx.gpu(0)) for s in src], out=out)
        assert eq(out.asnumpy(), g["n%d_out" % n]), n


def test_unaligned_external_memory(mx):
    # views of torch memory at odd element offsets take the scalar path
    import torch
    rng = np.random.default_rng(5)
    n = 5000
    a = rnd(rng, n + 3)
    t = torch.from_numpy(a).cuda()
    view = t[1:1 + n]                       # 4-byte aligned only
    out_t = torch.zeros(n + 5, device='cuda')
    out_view = out_t[3:3 + n]
    mx.base.set_stream(0, torch.cuda.current_stream().cuda_stream)
    try:
        kv = mx.kv.create('device')
        kv.init(0, mx.nd.zeros((n,), mx.gpu(0)))
        kv.pushpull(0, [mx.nd.from_torch(view), mx.nd.from_torch(view)], out=mx.nd.from_torch(out_view))
        torch.cuda.synchronize()
        assert eq(out_view.cpu().numpy(), a[1:1 + n] + a[1:1 + n])
        assert out_t[:3].abs().sum().item() == 0 and out_t[3 + n:].abs().sum().item() == 0
    finally:
        mx.base.set_stream(0, None)


def test_host_buffers_end_to_end(mx, oracle):
    # kvstore('local') with CPU-context values: staged through the GPU, result back on the host
    rng = np.random.default_rng(6)
    kv = mx.kv.create('local')
    shape = (1024, 1024)                    # BASELINE.json configs[0]
    kv.init(0, mx.nd.zeros(shape, mx.cpu()))
    srcs = [rnd(rng, shape) for _ in range(4)]
    out = mx.nd.empty(shape, mx.cpu())
    kv.push(0, [mx.nd.array(s, mx.cpu(i)) for i, s in enumerate(srcs)])
    kv.pull(0, out=out)
    assert eq(out.asnumpy().ravel(), oracle.reduce(srcs, 'local'))


# ------------------------------------------------------------------ fused optimizers vs oracle
def _run_fused(mx, kvtype, opt, model_kw, steps, n, shapes, rng, lr_mult=None, wd_mult=None):
    kv = mx.kv.create(kvtype)
    model = K.LocalKVStoreModel('local' if kvtype == 'local' else 'device')
    keys = list(range(len(shapes)))
    w0 = [rnd(rng, s) for s in shapes]
    for k in keys:
        kv.init(k, mx.nd.array(w0[k], mx.gpu(0)))
        model.init(k, w0[k])
    if lr_mult:
        opt.set_lr_mult(lr_mult)
    if wd_mult:
        opt.set_wd_mult(wd_mult)
    kv.set_optimizer(opt)
    model.set_optimizer(lr_mult=lr_mult, wd_mult=wd_mult, **model_kw)
    outs = [[mx.nd.empty(s, mx.gpu(0)) for _ in range(n)] for s in shapes]
    for step in range(steps):
        grads = [[rnd(rng, s) for _ in range(n)] for s in shapes]
        vals = [[mx.nd.array(g, mx.gpu(0)) for g in grads[k]] for k in keys]
        kv.pushpull(keys, vals, out=outs)
        for k in keys:
            model.push(k, grads[k])
            ref = model.pull(k)
            for o in outs[k]:
                assert eq(o.asnumpy(), ref), (step, k)
    return kv, model


@pytest.mark.parametrize("kvtype", ['local', 'device'])
@pytest.mark.parametrize("momentum,clip", [(0.9, None), (0.0, None), (0.9, 0.02), (0.0, 0.02)])
def test_fused_sgd_bit_exact(mx, kvtype, momentum, clip):
    rng = np.random.default_rng(7)
    opt = mx.optimizer.SGD(learning_rate=0.1, momentum=momentum, wd=1e-4, rescale_grad=1.0 / 256,
                           clip_gradient=clip)
    _run_fused(mx, kvtype, opt, dict(kind='sgd', lr=0.1, momentum=momentum, wd=1e-4,
                                     rescale_grad=1.0 / 256, clip_gradient=clip),
               steps=3, n=4, shapes=SHAPES[:5], rng=rng, lr_mult={1: 0.5, 3: 2.0}, wd_mult={0: 0.0})


@pytest.mark.parametrize("clip", [None, 0.5])
def test_fused_adam_bit_exact(mx, clip):
    rng = np.random.default_rng(8)
    opt = mx.optimizer.Adam(learning_rate=1e-3, wd=0.01, clip_gradient=clip)
    _run_fused(mx, 'device', opt, dict(kind='adam', lr=1e-3, wd=0.01, clip_gradient=clip),
               steps=5, n=2, shapes=SHAPES[:5], rng=rng, lr_mult={2: 0.1})


def test_fused_test_optimizer(mx):
    # tests/nightly/test_kvstore.py: 'test' optimizer w += rescale*g over 4 values, 10 repeats
    rng = np.random.default_rng(9)
    opt = mx.optimizer.Test(rescale_grad=2.0)
    _run_fused(mx, 'local', opt, dict(kind='test', rescale_grad=2.0), steps=10, n=4,
               shapes=[(4, 4), (100, 100), (2000, 2000)], rng=rng)


@pytest.mark.parametrize("optname,dtype", [
    pytest.param('sgd', np.float32, id='sgd'), pytest.param('adam', np.float32, id='adam'),
    pytest.param('test', np.float32, id='test'), pytest.param('sgd', np.float16, id='sgd-float16'),
    pytest.param('adam', np.float16, id='adam-float16')])
def test_callback_route_equals_fused_route(mx, optname, dtype, monkeypatch):
    """The reference's route (store -> Python Updater -> optimizer operators) and the fused route
    must agree bit-for-bit, including update counts and Adam's bias-corrected lr. On float16 keys
    both keep float32 master weights (multi_precision=True)."""
    results = []
    mp = dtype != np.float32
    for fused in ('1', '0'):
        monkeypatch.setenv('B200KV_FUSED_OPTIMIZER', fused)
        rng = np.random.default_rng(10)
        kv = mx.kv.create('device')
        shapes = SHAPES[:4]
        for k, s in enumerate(shapes):
            kv.init(k, mx.nd.array(rnd(rng, s), mx.gpu(0), dtype))
        # objects of the reference's optimizer classes (tests/compat mirror): the store fuses SGD /
        # Adam natively, or -- B200KV_FUSED_OPTIMIZER=0 -- calls their own update() back per key
        from compat import mxnet_optimizer as mxopt
        if optname == 'sgd':
            opt = mxopt.SGD(learning_rate=0.05, momentum=0.9, wd=1e-3, rescale_grad=0.5, multi_precision=mp)
        elif optname == 'adam':
            opt = mxopt.Adam(learning_rate=2e-3, wd=0.02, rescale_grad=0.25, multi_precision=mp)
        else:   # dmlc::stof and std::stod-then-float parse this rescale_grad differently
            opt = mxopt.Test(rescale_grad=1.2345e-05)
        kv.set_optimizer(opt)
        assert (kv._fused is not None) == (fused == '1')
        outs = [mx.nd.empty(s, mx.gpu(0), dtype) for s in shapes]
        for _ in range(3):
            for k, s in enumerate(shapes):
                kv.push(k, [mx.nd.array(rnd(rng, s), mx.gpu(0), dtype) for _ in range(3)])
                kv.pull(k, out=outs[k])
        results.append([o.asnumpy() for o in outs])
    for a, b in zip(*results):
        assert eq(a, b)


# ------------------------------------------------------------------ optimizer operators vs golden
@pytest.mark.parametrize("tag,clip", [("noclip", None), ("clip", 0.002)])
def test_optimizer_ops_golden(mx, golden, tag, clip):
    """MXImperativeInvokeEx(sgd_update, ...) etc. against outputs of the reference's own kernels."""
    g = golden("optimizers")
    lr, wd, rescale, momentum = [float(x) for x in g["hp"]]
    kw = dict(rescale_grad=rescale)
    if clip:
        kw['clip_gradient'] = clip
    dev = mx.gpu(0)
    w, gr = g["sgd_%s_in" % tag]
    wn = mx.nd.array(w, dev)
    mx.nd.sgd_update(wn, mx.nd.array(gr, dev), out=wn, lr=lr, wd=wd, **kw)
    assert eq(wn.asnumpy(), g["sgd_%s_out" % tag])
    w, gr, m = g["sgdmom_%s_in" % tag]
    wn, mn = mx.nd.array(w, dev), mx.nd.array(m, dev)
    mx.nd.sgd_mom_update(wn, mx.nd.array(gr, dev), mn, out=wn, lr=lr, wd=wd, momentum=momentum, **kw)
    assert eq(np.stack([wn.asnumpy(), mn.asnumpy()]), g["sgdmom_%s_out" % tag])
    wn, mn = mx.nd.array(w, dev), mx.nd.array(m, dev)
    mx.nd.multi_sgd_mom_update(wn, mx.nd.array(gr, dev), mn, out=[wn], num_weights=1, lrs=(lr,),
                               wds=(wd,), momentum=momentum, **kw)
    assert eq(np.stack([wn.asnumpy(), mn.asnumpy()]), g["multisgdmom_%s_out" % tag])
    wn = mx.nd.array(w, dev)
    mx.nd.multi_sgd_update(wn, mx.nd.array(gr, dev), out=[wn], num_weights=1, lrs=(lr,), wds=(wd,), **kw)
    assert eq(wn.asnumpy(), g["multisgd_%s_out" % tag])
    # fp16 weights + fp32 master
    w16, g16 = g["mp_%s_in16" % tag]
    w32, m = g["mp_%s_in32" % tag]
    a16 = mx.nd.array(w16.view(np.float16), dev, np.float16)
    ag = mx.nd.array(g16.view(np.float16), dev, np.float16)
    a32, am = mx.nd.array(w32, dev), mx.nd.array(m, dev)
    mx.nd.multi_mp_sgd_mom_update(a16, ag, am, a32, out=[a16], num_weights=1, lrs=(lr,), wds=(wd,),
                                  momentum=momentum, **kw)
    assert eq(a16.asnumpy().view(np.uint16), g["mpmom_%s_out16" % tag])
    assert eq(np.stack([a32.asnumpy(), am.asnumpy()]), g["mpmom_%s_out32" % tag])
    a16 = mx.nd.array(w16.view(np.float16), dev, np.float16)
    a32 = mx.nd.array(w32, dev)
    mx.nd.mp_sgd_update(a16, ag, a32, out=a16, lr=lr, wd=wd, **kw)
    assert eq(a16.asnumpy().view(np.uint16), g["mpsgd_%s_out16" % tag])
    assert eq(a32.asnumpy(), g["mpsgd_%s_out32" % tag])


@pytest.mark.parametrize("tag,clip", [("noclip", None), ("clip", 0.5)])
def test_adam_op_golden(mx, golden, tag, clip):
    g = golden("optimizers")
    dev = mx.gpu(0)
    w, gr, m, v = [mx.nd.array(x, dev) for x in g["adam_%s_in" % tag]]
    kw = dict(clip_gradient=clip) if clip else {}
    for t in range(1, 6):
        lr_t = K.adam_lr(1e-3, 0.9, 0.999, t)   # python double, formatted by str() like the reference
        mx.nd.adam_update(w, gr, m, v, out=w, lr=lr_t, beta1=0.9, beta2=0.999, epsilon=1e-8, wd=0.01,
                          rescale_grad=1.0, **kw)
        got = np.stack([w.asnumpy(), m.asnumpy(), v.asnumpy()])
        # the fixture's scalars went through the reference's own dmlc::stof(repr(x)); so do ours
        assert eq(got, g["adam_%s_out" % tag][t - 1]), t


# ------------------------------------------------------------------ mixed precision through the store
@pytest.mark.parametrize("dtype,kind", [(np.float16, 0), ('bfloat16', 1)])
def test_fused_mixed_precision(mx, oracle, dtype, kind):
    rng = np.random.default_rng(11)
    n, size = 2, 10007
    w32 = rnd(rng, size)
    w16 = oracle.to_half(w32, kind)
    kv = mx.kv.create('device')
    if kind == 0:
        init = mx.nd.array(w16.view(np.float16), mx.gpu(0), np.float16)
    else:
        init = mx.nd.array(oracle.from_half(w16, 1), mx.gpu(0), 'bfloat16')
    kv.init(0, init)
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9, wd=1e-4, rescale_grad=1 / 64,
                                      multi_precision=True))
    master = oracle.from_half(w16, kind).copy()     # weight.astype(float32)
    mom = np.zeros(size, np.float32)
    out = mx.nd.empty((size,), mx.gpu(0), dtype)
    for step in range(3):
        g16 = [oracle.to_half(rnd(rng, size), kind) for _ in range(n)]
        if kind == 0:
            vals = [mx.nd.array(g.view(np.float16), mx.gpu(0), np.float16) for g in g16]
        else:
            vals = [mx.nd.array(oracle.from_half(g, 1), mx.gpu(0), 'bfloat16') for g in g16]
        kv.pushpull(0, vals, out=out)
        # reference: 16-bit ElementwiseSum (rounds after each add) then multi_mp_sgd_mom_update
        merged = oracle.to_half(oracle.from_half(g16[0], kind) + oracle.from_half(g16[1], kind), kind)
        ref16 = np.zeros(size, np.uint16)
        oracle.multi_mp_sgd_update(ref16, master, merged, mom, kind, K.f32(0.1), K.f32(0.9),
                                   K.f32(1e-4), K.f32(1 / 64))
        got = out.asnumpy()
        got16 = got.view(np.uint16) if kind == 0 else oracle.to_half(got, 1)
        assert eq(got16, ref16), step


# ------------------------------------------------------------------ full-size properties (BASELINE configs[1])
def test_resnet50_sized_properties(mx):
    """ResNet-50 gradient set (157 tensors / 25.5M elements) through ONE grouped pushpull:
    linearity (sum of ones == n), idempotent pull, and a checksum against float64 numpy."""
    from bench import resnet50_shapes
    import torch
    shapes = resnet50_shapes()
    assert len(shapes) == 157 and sum(int(np.prod(s)) for s in shapes) == 25549486
    kv = mx.kv.create('device')
    keys = list(range(len(shapes)))
    kv.init(keys, [mx.nd.zeros(s, mx.gpu(0)) for s in shapes])
    n = 2
    torch.manual_seed(0)
    gt = [[torch.rand(s, device='cuda') * 2 - 1 for _ in range(n)] for s in shapes]
    outs_t = [torch.empty(s, device='cuda') for s in shapes]
    torch.cuda.synchronize()
    vals = [[mx.nd.from_torch(t) for t in g] for g in gt]
    outs = [mx.nd.from_torch(t) for t in outs_t]
    kv.pushpull(keys, vals, out=outs)
    mx.nd.waitall()
    tot = 0.0
    ref = 0.0
    for k in keys:
        assert torch.equal(outs_t[k], gt[k][0] + gt[k][1])      # 2-input sum is order-free: exact
        tot += outs_t[k].double().sum().item()
        ref += gt[k][0].double().sum().item() + gt[k][1].double().sum().item()
    assert abs(tot - ref) <= 1e-6 * max(1.0, abs(ref))
    outs2_t = [torch.empty(s, device='cuda') for s in shapes]
    kv.pull(keys, out=[mx.nd.from_torch(t) for t in outs2_t])
    mx.nd.waitall()
    for a, b in zip(outs_t, outs2_t):
        assert torch.equal(a, b)


# ------------------------------------------------------------------ the other mshadow dtypes
@pytest.mark.parametrize("dtype", [np.float64, np.int32, np.int64, np.uint8, np.int8])
@pytest.mark.parametrize("kvtype", ['local', 'device'])
def test_reduce_other_dtypes(mx, dtype, kvtype):
    """the reference's reducers exist for every mshadow dtype (MSHADOW_TYPE_SWITCH, comm.h:273,
    ndarray_function-inl.h:399): push of n values / pull, in both association orders"""
    rng = np.random.default_rng(77)
    shape = (1027, 5)
    kv = mx.kv.create(kvtype)
    kv.init(0, mx.nd.array(np.zeros(shape, dtype), mx.gpu(0), dtype))
    for n in (1, 3, 6):
        if np.issubdtype(dtype, np.floating):
            vals = [rng.uniform(-1, 1, shape).astype(dtype) for _ in range(n)]
        else:
            info = np.iinfo(dtype)
            vals = [rng.integers(info.min // 8, info.max // 8, shape).astype(dtype) for _ in range(n)]
        kv.push(0, [mx.nd.array(v, mx.gpu(0), dtype) for v in vals])
        out = mx.nd.empty(shape, mx.gpu(0), dtype)
        kv.pull(0, out=out)
        # the association of the store type, in the dtype's own arithmetic
        if kvtype == 'device':
            want = vals[0].copy()
            for v in vals[1:]:
                want = (want + v).astype(dtype)
        else:
            want = vals[0].copy()
            for i in range(1, n, 4):
                t = vals[i].copy()
                for q in range(1, 4):
                    if i + q < n:
                        t = (t + vals[i + q]).astype(dtype)
                want = (want + t).astype(dtype)
        got = out.asnumpy()
        assert got.dtype == np.dtype(dtype) and eq(got, want), (dtype, n)
    with pytest.raises(mx.MXNetError, match="optimizers on the store run on float32"):
        kv.set_optimizer(mx.optimizer.Test(rescale_grad=1.0))
        kv.push(0, mx.nd.array(np.ones(shape, dtype), mx.gpu(0), dtype))
        mx.nd.waitall()


# ------------------------------------------------------------------ TMA pack kernel
def test_pack_bulk_copy(mx):
    """Many arrays (3 elements .. 4 MB, fp32 and 16-bit, aligned and ragged byte sizes) copied by
    ONE TMA bulk-copy launch: device->device, pinned host->device and device->pinned host."""
    import ctypes
    rng = np.random.default_rng(12)
    shapes = [(3,), (1,), (4099,), (16384,), (1000, 1000), (7, 11, 13), (4096 * 4 + 4,)]
    lib = mx.base._LIB
    for src_ctx, dst_ctx in ((mx.gpu(0), mx.gpu(0)), (mx.cpu(), mx.gpu(0)), (mx.gpu(0), mx.cpu())):
        srcs, dsts, want = [], [], []
        for i, s in enumerate(shapes):
            dt = np.float16 if i % 3 == 2 else np.float32
            a = rng.uniform(-1, 1, s).astype(dt)
            want.append(a)
            srcs.append(mx.nd.array(a, src_ctx, dt))
            dsts.append(mx.nd.array(np.zeros(s, dt), dst_ctx, dt))
        n = len(shapes)
        sa = (ctypes.c_void_p * n)(*[x._hv for x in srcs])
        da = (ctypes.c_void_p * n)(*[x._hv for x in dsts])
        packed = ctypes.c_int()
        mx.base.check_call(lib.B200KVTestPackCopy(n, sa, da, ctypes.byref(packed)))
        assert packed.value == n
        assert mx.base.last_kernel_info()[0].startswith("pack_bulk")
        for d, w in zip(dsts, want):
            assert eq(d.asnumpy(), w)
