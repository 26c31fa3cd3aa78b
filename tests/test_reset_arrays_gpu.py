"""reset_arrays and zeros_like on row_sparse arrays, on the GPU. The oracle is numpy zeros, and every
byte around each zeroed array -- a sentinel frame of the buffer it was sliced from -- unchanged:
every accepted dtype alone and mixed, patterns with -0.0, NaN, inf and denormals, every head and tail
misalignment of float16 / float32 / float64 slices on both sides of the 16 KB tile, a huge array
beside tiny and empty ones, 157 / 200 / 201 / 450 arrays and their launch counts, row_sparse inputs,
the engine ordering against a queued push, a pull anchor and DLPack-imported torch tensors on the
caller's stream, the accumulate / pushpull / zero_grad loop against the oracle model, and every
refusal."""
import numpy as np
import pytest

import bench
import kvoracle as K

pytestmark = pytest.mark.gpu
TILE = 16384            # kRATileBytes (kernels.h)
DTYPES = ['float16', 'bfloat16', 'float32', 'float64']
ITEM = {'float16': 2, 'bfloat16': 2, 'float32': 4, 'float64': 8}


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def raw(a):
    """the array's bytes in its own dtype (bfloat16 comes back widened to float32)"""
    h = a.asnumpy()
    if a.dtype == 'bfloat16':
        h = (h.view(np.uint32) >> 16).astype(np.uint16)
    return np.ascontiguousarray(h).reshape(-1).view(np.uint8)


def upload(mx, bits, dtype):
    """raw bits (uint8) -> a GPU array of dtype holding exactly those bits"""
    if dtype == 'bfloat16':
        host = (bits.view(np.uint16).astype(np.uint32) << 16).view(np.float32)
    else:
        host = bits.view({'float16': np.float16, 'float32': np.float32, 'float64': np.float64}[dtype])
    return mx.nd.array(host, mx.gpu(0), dtype)


SPECIAL = {   # -0.0, +-inf, quiet and signalling NaN, smallest and largest denormal, 1.0
    'float16': [0x8000, 0x7C00, 0xFC00, 0x7E00, 0x7C01, 0x0001, 0x03FF, 0x3C00],
    'bfloat16': [0x8000, 0x7F80, 0xFF80, 0x7FC0, 0x7F81, 0x0001, 0x007F, 0x3F80],
    'float32': [0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001, 0x00000001, 0x007FFFFF, 0x3F800000],
    'float64': [0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000,
                0x7FF0000000000001, 0x0000000000000001, 0x000FFFFFFFFFFFFF, 0x3FF0000000000000],
}
UINT = {2: np.uint16, 4: np.uint32, 8: np.uint64}


def pattern(rng, dtype, n):
    """n elements: the special values of the dtype repeated, then random bits with no zero byte"""
    it = ITEM[dtype]
    el = rng.integers(1, 256, n * it, dtype=np.uint8)
    sp = np.array(SPECIAL[dtype], UINT[it]).view(np.uint8)
    k = min(len(sp), len(el))
    el[:k] = sp[:k]
    return el


class Framed(object):
    """a view of n elements, `head` elements into a buffer filled with a sentinel pattern that
    runs `tail` elements past the view's end"""

    def __init__(self, mx, rng, dtype, n, head=0, tail=0):
        self.dtype, self.head, self.n = dtype, head, n
        self.bits = pattern(rng, dtype, head + n + tail)
        self.whole = upload(mx, self.bits, dtype)
        self.view = self.whole[head:head + n] if (head or tail) else self.whole

    def check_zeroed(self):
        got, want = raw(self.whole), self.bits.copy()
        it = ITEM[self.dtype]
        want[self.head * it:(self.head + self.n) * it] = 0
        assert np.array_equal(got, want), (self.dtype, self.head, self.n)

    def check_unchanged(self):
        assert np.array_equal(raw(self.whole), self.bits), (self.dtype, self.head, self.n)


def reset(mx, arrays):
    """reset_arrays over `arrays`; returns the launches it spent (queued store calls are issued
    first, so that their launches are not counted)"""
    mx.base.flush_all()
    before = mx.base.kernel_launch_count()
    res = mx.nd.reset_arrays(*arrays, num_arrays=len(arrays))
    assert not res
    return mx.base.kernel_launch_count() - before


# ------------------------------------------------------------------------------ dtypes and values
@pytest.mark.parametrize("dtype", DTYPES)
def test_each_dtype_alone(mx, dtype):
    rng = np.random.default_rng(1)
    for n in (1, 7, 1000, TILE // ITEM[dtype] + 3, 300001):
        f = Framed(mx, rng, dtype, n, head=8, tail=8)
        assert reset(mx, [f.view]) == 1
        f.check_zeroed()
    f = Framed(mx, rng, dtype, 4097)      # the whole buffer, 256-byte aligned by the allocator
    assert reset(mx, [f.view]) == 1
    f.check_zeroed()
    assert not raw(f.whole).any()


def test_mixed_dtypes_in_one_call(mx):
    rng = np.random.default_rng(2)
    frames = [Framed(mx, rng, DTYPES[i % 4], int(n), head=int(h), tail=3)
              for i, (n, h) in enumerate(zip(rng.integers(1, 20000, 40), rng.integers(0, 9, 40)))]
    assert reset(mx, [f.view for f in frames]) == 1
    for f in frames:
        f.check_zeroed()


# ------------------------------------------------------------------------------ slices
@pytest.mark.parametrize("dtype", ['float16', 'float32', 'float64'])
def test_every_head_and_tail_misalignment(mx, dtype):
    """slices of a buffer whose base is 256-byte aligned: the slice starts at every byte offset
    0..15 (mod 16) its element size allows and ends at every one, within one 16-byte word, within
    one tile and across two tile boundaries"""
    it = ITEM[dtype]
    per = 16 // it
    rng = np.random.default_rng(3)
    n_max = 2 * TILE // it + 4 * per
    f = Framed(mx, rng, dtype, 0, head=0, tail=n_max + 2 * per)
    keep = f.whole.copy()
    seen = set()
    for h in range(per):
        for t in range(per):
            for q in (0, 1, 2 * TILE // 16 + 1):
                n = q * per + t
                if n == 0:
                    continue
                view = f.whole[h:h + n]
                assert reset(mx, [view]) == 1
                got, want = raw(f.whole), f.bits.copy()
                want[h * it:(h + n) * it] = 0
                assert np.array_equal(got, want), (dtype, h, n)
                seen.add(((h * it) % 16, ((h + n) * it) % 16))
                keep.copyto(f.whole)
    assert len(seen) == per * per


# ------------------------------------------------------------------------------ sizes
def test_huge_array_beside_tiny_and_empty_ones(mx):
    rng = np.random.default_rng(4)
    huge = Framed(mx, rng, 'float32', 100_000_003, head=1, tail=5)
    tiny = [Framed(mx, rng, DTYPES[i % 4], 1, head=i % 3, tail=1) for i in range(60)]
    empty = [mx.nd.array(np.zeros(0, np.float32), mx.gpu(0)), mx.nd.array(np.zeros((0, 5), np.float16), mx.gpu(0), np.float16)]
    arrays = [t.view for t in tiny[:30]] + [empty[0], huge.view, empty[1]] + [t.view for t in tiny[30:]]
    assert reset(mx, arrays) == 1
    huge.check_zeroed()
    for t in tiny:
        t.check_zeroed()


def test_only_empty_arrays_launch_nothing(mx):
    e = [mx.nd.array(np.zeros(0, np.float32), mx.gpu(0)), mx.nd.array(np.zeros((3, 0), np.float64), mx.gpu(0), np.float64)]
    assert reset(mx, e) == 0
    assert reset(mx, e[:1]) == 0


# ------------------------------------------------------------------------------ grouping
@pytest.mark.parametrize("count,launches", [('r50', 1), (200, 1), (201, 2), (450, 3)])
def test_grouping_and_launch_counts(mx, count, launches):
    rng = np.random.default_rng(5)
    if count == 'r50':
        shapes = bench.resnet50_shapes()
        assert len(shapes) == 157
        frames = [Framed(mx, rng, 'float32', int(np.prod(s)), head=0, tail=1) for s in shapes]
    else:
        frames = [Framed(mx, rng, DTYPES[i % 4], int(n), head=int(h), tail=2)
                  for i, (n, h) in enumerate(zip(rng.integers(1, 3000, count), rng.integers(0, 5, count)))]
    assert reset(mx, [f.view for f in frames]) == launches
    for f in frames:
        f.check_zeroed()


def test_empty_arrays_do_not_count_toward_a_group(mx):
    """200 non-empty arrays with empty ones between them still take one launch"""
    rng = np.random.default_rng(6)
    frames = [Framed(mx, rng, 'float32', 5, tail=1) for _ in range(200)]
    e = mx.nd.array(np.zeros(0, np.float32), mx.gpu(0))
    arrays = []
    for f in frames:
        arrays += [f.view, e]
    assert reset(mx, arrays) == 1
    for f in frames:
        f.check_zeroed()


def test_duplicated_and_overlapping_arrays(mx):
    rng = np.random.default_rng(7)
    f = Framed(mx, rng, 'float32', 9000, head=2, tail=2)
    inner = f.whole[100:5000]
    assert reset(mx, [f.view, inner, f.view, f.whole[3:4]]) == 1
    f.check_zeroed()


# ------------------------------------------------------------------------------ row_sparse
def rsp(mx, shape, ids, dtype=np.float32, seed=0):
    rows = np.random.default_rng(seed).uniform(1, 2, (len(ids),) + tuple(shape[1:])).astype(dtype)
    return mx.nd.sparse.row_sparse_array((rows, np.array(ids, np.int64)), shape=shape, ctx=mx.gpu(0), dtype=dtype), rows


def test_row_sparse_inputs_mixed_with_dense(mx):
    rng = np.random.default_rng(8)
    a, rows_a = rsp(mx, (50, 8), [2, 17, 49], seed=1)
    b, rows_b = rsp(mx, (1000, 3), list(range(0, 1000, 7)), seed=2)
    never = mx.nd.sparse.zeros('row_sparse', (20, 4), mx.gpu(0))
    data_a, data_b = a.data, b.data                  # views of the stored rows, taken before
    dense = [Framed(mx, rng, DTYPES[i % 4], 3000 + i, head=i % 3, tail=1) for i in range(5)]
    arrays = [a, dense[0].view, never, dense[1].view, b] + [d.view for d in dense[2:]]
    assert reset(mx, arrays) == 1
    for d in dense:
        d.check_zeroed()
    for r in (a, b, never):
        assert r.stype == 'row_sparse' and r.indices.shape == (0,) and r.data.shape[0] == 0
        assert not r.asnumpy().any()
    assert a.shape == (50, 8) and b.shape == (1000, 3)
    # the storage is kept as it was: the rows are still there, just not stored rows any more
    assert np.array_equal(data_a.asnumpy(), rows_a) and np.array_equal(data_b.asnumpy(), rows_b)
    assert reset(mx, [a, never, b]) == 0


def test_row_sparse_push_and_pull_after_reset(mx):
    shape = (64, 16)
    w = np.random.default_rng(9).uniform(-1, 1, shape).astype(np.float32)
    kv = mx.kv.create('device')
    kv.init('e', mx.nd.array(w, mx.gpu(0)).tostype('row_sparse'))
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1))
    g, _ = rsp(mx, shape, [1, 5, 63], seed=3)
    assert reset(mx, [g]) == 0
    kv.push('e', g)                                  # a gradient with no rows: the weights stay
    ids = np.array([0, 5, 17, 63], np.int64)
    kv.row_sparse_pull('e', out=g, row_ids=mx.nd.array(ids, mx.gpu(0), np.int64))
    assert np.array_equal(g.indices.asnumpy(), ids)
    assert np.array_equal(g.data.asnumpy(), w[ids])
    assert reset(mx, [g]) == 0
    assert g.indices.shape == (0,)
    kv.row_sparse_pull('e', out=g, row_ids=mx.nd.array(ids[:2], mx.gpu(0), np.int64))
    assert np.array_equal(g.asnumpy()[ids[:2]], w[ids[:2]])


# ------------------------------------------------------------------------------ zeros_like
def test_zeros_like_row_sparse(mx):
    for dtype in (np.float32, np.float16):
        a, rows = rsp(mx, (30, 5), [0, 4, 29], dtype=dtype, seed=4)
        data = a.data
        for fn in (mx.nd.zeros_like, mx.nd.sparse.zeros_like):
            z = fn(a)
            assert isinstance(z, mx.nd.RowSparseNDArray) and z.stype == 'row_sparse'
            assert z.shape == (30, 5) and z.dtype == dtype and z.context == mx.gpu(0)
            assert z.indices.shape == (0,) and not z.asnumpy().any()
            assert a.indices.shape == (3,)           # the input is not touched
        assert np.array_equal(a.asnumpy()[[0, 4, 29]], rows)
        out = mx.nd.zeros_like(a, out=a)
        assert out is a and a.indices.shape == (0,) and not a.asnumpy().any()
        assert np.array_equal(data.asnumpy(), rows)  # storage kept
        b, _ = rsp(mx, (30, 5), [3], dtype=dtype, seed=5)
        mx.nd.sparse.zeros_like(mx.nd.array(np.ones((30, 5)), mx.gpu(0), dtype), out=b)
        assert b.indices.shape == (0,)
    # dense zeros_like is as it was: a dense array of zeros, or zeros written into a dense out
    d = mx.nd.array(np.ones((4, 3)), mx.gpu(0))
    z = mx.nd.zeros_like(d)
    assert z.stype == 'default' and z.shape == (4, 3) and not z.asnumpy().any()
    a, _ = rsp(mx, (4, 3), [1], seed=6)
    mx.nd.zeros_like(a, out=d)
    assert not d.asnumpy().any()


# ------------------------------------------------------------------------------ ordering
def test_order_after_a_queued_single_key_push(mx):
    """a single-key push is bucketed (issued later); the zeroing must not overtake its read"""
    shape = (2048, 1024)
    rng = np.random.default_rng(10)
    w, gh = rng.uniform(-1, 1, shape).astype(np.float32), rng.uniform(-1, 1, shape).astype(np.float32)
    kv = mx.kv.create('device')
    kv.init(3, mx.nd.array(w, mx.gpu(0)))
    g = mx.nd.array(gh, mx.gpu(0))
    kv.push(3, g)
    mx.nd.reset_arrays(g, num_arrays=1)
    out = mx.nd.empty(shape, mx.gpu(0))
    kv.pull(3, out=out)
    assert np.array_equal(out.asnumpy(), gh)         # no optimizer: the stored value is the push
    assert not g.asnumpy().any()


def test_order_with_an_anchored_pull_target(mx):
    """reset_arrays on a pushpull's pull target (the key's value lives there): the target reads
    zeros, the store keeps the value, and the next pushpull continues from it"""
    shapes = [(64, 3, 7, 7), (1000, 512), (3,)]
    rng = np.random.default_rng(11)
    keys = list(range(len(shapes)))
    kv, model = mx.kv.create('device'), K.LocalKVStoreModel('device')
    for k, s in enumerate(shapes):
        w = rng.uniform(-1, 1, s).astype(np.float32)
        kv.init(k, mx.nd.array(w, mx.gpu(0)))
        model.init(k, w)
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9, wd=1e-4))
    model.set_optimizer('sgd', lr=0.1, momentum=0.9, wd=1e-4)
    outs = [mx.nd.empty(s, mx.gpu(0)) for s in shapes]

    def step():
        g = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]
        kv.pushpull(keys, [mx.nd.array(a, mx.gpu(0)) for a in g], out=outs)
        for k in keys:
            model.push(k, g[k])
    for _ in range(2):
        step()
    assert reset(mx, outs) == 1
    for o in outs:
        assert not o.asnumpy().any()
    fresh = [mx.nd.empty(s, mx.gpu(0)) for s in shapes]
    kv.pull(keys, out=fresh)
    for k in keys:
        assert np.array_equal(fresh[k].asnumpy(), model.pull(k)), k
    step()
    for k in keys:
        assert np.array_equal(outs[k].asnumpy(), model.pull(k)), k


def test_order_on_the_callers_stream_with_torch_tensors(mx):
    """DLPack-imported torch gradients, the library on torch's stream: torch's pending writes come
    before the zeroing, torch's later reads after it, with no synchronisation in between"""
    import torch
    s = torch.cuda.Stream(device=0)
    sizes = [1 << 24, 1000, 3, 1 << 20]
    with torch.cuda.stream(s):
        ts = [torch.ones(n, device='cuda:0', dtype=torch.float32 if i % 2 == 0 else torch.float16)
              for i, n in enumerate(sizes)]
        mx.base.set_stream(0, s.cuda_stream)
        try:
            arrays = [mx.nd.from_torch(t) for t in ts]
            for t in ts:
                for _ in range(4):
                    t.mul_(3)                           # queued on s ahead of the zeroing
            assert reset(mx, arrays) == 1
            after = [t.abs().sum() for t in ts]          # queued on s behind it
            for t in ts:
                t.add_(2)
            totals = [t.float().sum() for t in ts]
        finally:
            mx.base.set_stream(0, None)
    s.synchronize()
    assert [float(a) for a in after] == [0.0] * len(ts)
    assert [float(x) for x in totals] == [2.0 * n for n in sizes]


# ------------------------------------------------------------------------------ accumulation loop
class Param(object):
    def __init__(self, grad_req, grads):
        self.grad_req, self._grad = grad_req, grads

    def list_grad(self):
        return list(self._grad)


def test_accumulate_pushpull_zero_grad_loop(mx):
    """grad_req='add' training: k micro-batches summed into the gradients with _plus, pushpull with
    the fused SGD-momentum step, then the zero_grad mirror -- three rounds, on two GPUs when there
    are two. The weights equal the oracle model's, fed the summed gradients, bit for bit."""
    import torch
    from compat import mxnet_gluon_parameter as P
    ndev = 2 if torch.cuda.device_count() >= 2 else 1
    shapes = [(64, 3, 7, 7), (64,), (256, 64, 1, 1), (1000, 2048), (1000,), (3,)]
    rng = np.random.default_rng(12)
    keys = list(range(len(shapes)))
    kv, model = mx.kv.create('device'), K.LocalKVStoreModel('device')
    weights = []
    for k, s in enumerate(shapes):
        w = rng.uniform(-1, 1, s).astype(np.float32)
        kv.init(k, mx.nd.array(w, mx.gpu(0)))
        model.init(k, w)
        weights.append([mx.nd.array(w, mx.gpu(d)) for d in range(ndev)])
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.05, momentum=0.9, wd=1e-4, rescale_grad=1.0 / 64))
    model.set_optimizer('sgd', lr=0.05, momentum=0.9, wd=1e-4, rescale_grad=1.0 / 64)
    grads = [[mx.nd.zeros(s, mx.gpu(d)) for d in range(ndev)] for s in shapes]
    params = {'p%d' % k: Param('add', grads[k]) for k in keys}
    params['frozen'] = Param('null', [mx.nd.array(np.ones(5), mx.gpu(d)) for d in range(ndev)])
    for _ in range(3):
        sums = [[np.zeros(s, np.float32) for _ in range(ndev)] for s in shapes]
        for _ in range(3):                            # micro-batches
            for k, s in enumerate(shapes):
                for d in range(ndev):
                    m = rng.uniform(-1, 1, s).astype(np.float32)
                    grads[k][d] += mx.nd.array(m, mx.gpu(d))
                    sums[k][d] += m
        for k in keys:
            for d in range(ndev):
                assert np.array_equal(grads[k][d].asnumpy(), sums[k][d]), (k, d)
        kv.pushpull(keys, grads, out=weights)
        for k in keys:
            model.push(k, sums[k])
        mx.base.flush_all()
        before = mx.base.kernel_launch_count()
        P.zero_grad(params)
        assert mx.base.kernel_launch_count() - before == ndev
        for k in keys:
            for d in range(ndev):
                assert not grads[k][d].asnumpy().any(), (k, d)
                assert np.array_equal(weights[k][d].asnumpy(), model.pull(k)), (k, d)
        assert params['frozen']._grad[0].asnumpy().all()


# ------------------------------------------------------------------------------ refusals
def test_refusals_leave_every_operand_unchanged(mx):
    import torch
    rng = np.random.default_rng(13)
    Err = mx.base.MXNetError
    f32 = Framed(mx, rng, 'float32', 100, tail=1)
    f16 = Framed(mx, rng, 'float16', 100, tail=1)
    ints = {dt: mx.nd.array(np.arange(1, 9).astype(dt), mx.gpu(0), dt) for dt in ('uint8', 'int8', 'int32', 'int64')}
    cpu = mx.nd.array(np.ones(10, np.float32), mx.cpu())
    a, rows = rsp(mx, (10, 4), [1, 7], seed=7)
    ok = [f32.view, f16.view, a]
    cases = [
        ([f32.view], {}, None, 'Required parameter num_arrays of reset_arrays is missing'),
        (ok, dict(num_arrays=2), None, 'expected num_arrays inputs'),
        ([], dict(num_arrays=0), None, 'num_arrays must be at least 1'),
        (ok, dict(num_arrays=3, wd=0.1), None, r"Cannot find argument 'wd', Possible Arguments: num_arrays$"),
        (ok, dict(num_arrays=3), f32.view, 'has no output'),
        (ok + [ints['uint8']], dict(num_arrays=4), None, 'This operation only support floating point types not uint8$'),
        (ok + [ints['int8']], dict(num_arrays=4), None, 'This operation only support floating point types not int8$'),
        (ok + [ints['int32']], dict(num_arrays=4), None, 'This operation only support floating point types, not int32$'),
        (ok + [ints['int64']], dict(num_arrays=4), None, 'This operation only support floating point types, not int64$'),
        (ok + [cpu], dict(num_arrays=4), None, 'no CPU fallback'),
        ([cpu] + ok, dict(num_arrays=4), None, 'no CPU fallback'),
    ]
    if torch.cuda.device_count() >= 2:
        cases.append((ok + [mx.nd.array(np.ones(4), mx.gpu(1))], dict(num_arrays=4), None, "not on array_0's GPU"))
    for arrays, params, out, msg in cases:
        with pytest.raises(Err, match=msg):
            mx.nd.reset_arrays(*arrays, out=out, **params)
        f32.check_unchanged()
        f16.check_unchanged()
        assert a.indices.shape == (2,) and np.array_equal(a.data.asnumpy(), rows), msg
    for dt, x in ints.items():
        assert np.array_equal(x.asnumpy(), np.arange(1, 9).astype(dt))
    assert cpu.asnumpy().all()

    # elementwise operators take dense arrays only: a row_sparse operand or out is refused
    d = f32.view
    like = mx.nd.array(np.ones((10, 4), np.float32), mx.gpu(0))
    refused = [
        lambda: a.__setitem__(slice(None), 1.0),                                   # _full
        lambda: like + a, lambda: a + like, lambda: a + 2.0, lambda: a * 3.0,      # _plus, _plus_scalar, _mul_scalar
        lambda: mx.nd._invoke('_plus', [like, like], out=a),
        lambda: mx.nd._invoke('_mul_scalar', [like], out=a, scalar=2.0),
        lambda: mx.nd._invoke('elemwise_mul', [a, a]),
        lambda: mx.nd.sqrt(a),
    ]
    for fn in refused:
        with pytest.raises(Err, match='elementwise operators take dense arrays only'):
            fn()
        assert a.indices.shape == (2,) and np.array_equal(a.data.asnumpy(), rows)
        assert like.asnumpy().all()
    # zeros_like into a row_sparse out: shape, dtype and placement are checked first
    b16, _ = rsp(mx, (10, 4), [2], dtype=np.float16, seed=8)
    for args, kw, msg in [((like[0:5],), dict(out=a), 'out shape mismatch'),
                          ((like,), dict(out=b16), 'out dtype mismatch'),
                          ((mx.nd.array(np.ones((10, 4)), mx.cpu()),), dict(out=a), 'no CPU fallback')]:
        with pytest.raises(Err, match=msg):
            mx.nd.zeros_like(*args, **kw)
        assert a.indices.shape == (2,) and b16.indices.shape == (1,)
    assert np.array_equal(raw(d), f32.bits[:400])
