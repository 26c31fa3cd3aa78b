"""gluon.utils.clip_global_norm and contrib.multi_scale on the GPU, through the C ABI and the Python
surface: the reference's own test (test_gluon.py:1131-1149), every fixture case of
tests/golden/clip_global_norm.npz, seeded gradient sets on both sides of every size the kernels
branch on (one tile, the 16-byte vector, the per-thread load count, the 200-array group), unaligned
bases, empty and row_sparse members, the not-clipped / inf / nan cases that must not write, the
launch counts, issue order without host waits, and every refusal."""
import warnings

import numpy as np
import pytest

import golden_clip_global_norm as G

pytestmark = pytest.mark.gpu
F = np.float32


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def dev(mx, a):
    return mx.nd.array(np.asarray(a, F), mx.gpu(0))


def clip(mx, arrays, max_norm):
    """one operator call; the norm as the (1,) float32 numpy array the GPU wrote"""
    out = mx.nd._invoke('_b200kv_clip_global_norm', list(arrays), num_arrays=len(arrays), max_norm=max_norm)
    return out.asnumpy()


def check_set(mx, xs, max_norm, make=None):
    """clip the host arrays `xs` on the GPU: the norm within 1e-5 of a float64 sum, bit-equal on a
    second call over restored inputs (`make` builds the device arrays, at the same alignment each
    time: the 16-byte and the element-wise path associate a tile's sum differently), and every
    output bit-equal to the restatement on that norm"""
    make = make or (lambda: [dev(mx, x) for x in xs])
    arrays = make()
    norm = clip(mx, arrays, max_norm)[0]
    exact = np.sqrt(sum(float(np.sum(np.asarray(x, np.float64) ** 2)) for x in xs))
    if np.isfinite(exact) and exact < 3e38:
        assert abs(float(norm) - exact) <= 1e-5 * exact, (norm, exact)
    got = [a.asnumpy() for a in arrays]
    for i, (x, g) in enumerate(zip(xs, got)):
        assert eq(g.reshape(-1), G.restate(norm, max_norm, np.asarray(x, F).reshape(-1))), i
    again = make()
    assert eq(clip(mx, again, max_norm), np.array([norm], F))
    for g, a in zip(got, again):
        assert eq(g, a.asnumpy())
    return norm, got, arrays


# ------------------------------------------------------------------ the reference's own test
@pytest.mark.parametrize("stype", ['default', 'row_sparse'])
@pytest.mark.parametrize("check_isfinite", [True, False])
def test_global_norm_clip_as_the_reference_tests_it(mx, stype, check_isfinite):
    x1 = dev(mx, np.ones((3, 3))).tostype(stype)
    x2 = dev(mx, np.ones((4, 4))).tostype(stype)
    norm = mx.gluon.utils.clip_global_norm([x1, x2], 1.0, check_isfinite=check_isfinite)
    if check_isfinite:
        assert isinstance(norm, float)
    else:
        assert norm.shape == (1,) and norm.dtype == np.float32 and norm.context == mx.gpu(0)
        norm = norm.asscalar()
    assert norm == 5.0
    np.testing.assert_allclose(x1.asnumpy(), np.ones((3, 3)) / 5, rtol=1e-6)
    np.testing.assert_allclose(x2.asnumpy(), np.ones((4, 4)) / 5, rtol=1e-6)
    x3 = dev(mx, np.array([1.0, 2.0, float('nan')])).tostype(stype)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        mx.gluon.utils.clip_global_norm([x1, x3], 2.0, check_isfinite=check_isfinite)
        assert len(w) == check_isfinite


# ------------------------------------------------------------------------------ fixture cases
@pytest.mark.parametrize("name", sorted(G.SETS))
def test_fixture_set(mx, golden, name):
    case, g = G.SETS[name], golden("clip_global_norm")
    xs = G.inputs(case, name)
    norm, got, _ = check_set(mx, xs, case['max_norm'])
    want_norm = g[name + '_norm'].view(F)[0]
    if case['kind'] != 'float':      # sums of small integers are exact in every association
        assert eq(np.array([norm], F), np.array([want_norm], F))
        for i, o in enumerate(got):
            assert eq(o.view(np.uint32), g['%s_out%d' % (name, i)]), (name, i)
    elif np.isfinite(want_norm):
        assert abs(float(norm) - float(want_norm)) <= 1e-5 * float(want_norm)
    else:                            # inf and nan norms: the value comes back, nothing is written
        assert np.isnan(norm) if np.isnan(want_norm) else norm == want_norm
        for x, o in zip(xs, got):
            assert eq(x, o)


def test_not_clipped_inf_and_nan_leave_every_byte(mx):
    rng = np.random.default_rng(5)
    xs = [rng.standard_normal(n).astype(F) for n in (5, G.TILE + 9, 70000)]
    for poke, max_norm in ((None, '1e6'), (np.inf, '1.0'), (-np.inf, '1.0'), (np.nan, '1.0')):
        ys = [x.copy() for x in xs]
        if poke is not None:
            ys[1][G.TILE + 8] = poke
        arrays = [dev(mx, y) for y in ys]
        norm = clip(mx, arrays, max_norm)[0]
        if poke is None:
            assert np.isfinite(norm) and norm < 1e6
        elif np.isnan(poke):
            assert np.isnan(norm)
        else:
            assert norm == np.inf
        for y, a in zip(ys, arrays):
            assert eq(y, a.asnumpy())


# -------------------------------------------------------------------------------- seeded sets
def _shapes_resnet50():
    """the 157 dense gradient arrays of a ResNet-50 (conv / bn / fc), 25.5 M elements"""
    s = [(64, 3, 7, 7), (64,), (64,)]
    cin = 64
    for width, blocks in ((64, 3), (128, 4), (256, 6), (512, 3)):
        for b in range(blocks):
            s += [(width, cin, 1, 1), (width,), (width,), (width, width, 3, 3), (width,), (width,),
                  (4 * width, width, 1, 1), (4 * width,), (4 * width,)]
            if b == 0:
                s += [(4 * width, cin, 1, 1), (4 * width,), (4 * width,)]
            cin = 4 * width
    s += [(1000, 2048), (1000,)]
    return s[:157]


def _sizes(shapes):
    return [int(np.prod(s)) for s in shapes]


def _seeded(sizes, seed, scale=1e-2):
    rng = np.random.default_rng(seed)
    return [(rng.standard_normal(n) * scale).astype(F) for n in sizes]


@pytest.mark.parametrize("max_norm", ['1.0', '1e4'])
def test_resnet50_set(mx, max_norm):
    sizes = _sizes(_shapes_resnet50())
    assert len(sizes) == 157
    check_set(mx, _seeded(sizes, 50), max_norm)


def test_bert_base_sized_set(mx):
    """199 arrays shaped like BERT-base's (embeddings, 12 layers of 16 arrays, pooler), at a reduced
    hidden size so that the float64 check stays quick"""
    h = 192
    sizes = [30522 * h, 512 * h, 2 * h, h, h]
    for _ in range(12):
        sizes += [h * h, h] * 4 + [h, h, 4 * h * h, 4 * h, 4 * h * h, h, h, h]
    sizes += [h * h, h]
    assert len(sizes) == 199
    check_set(mx, _seeded(sizes, 199), '1.0')


@pytest.mark.parametrize("n", [1, 200, 201, 450])
def test_group_boundaries_and_launch_counts(mx, n):
    """at most 2 * ceil(n / 200) + 1 launches: a partial and a scale launch per group, one fold"""
    rng = np.random.default_rng(n)
    sizes = [int(s) for s in rng.integers(1, 3000, n)]
    xs = _seeded(sizes, n, 1.0)
    arrays = [dev(mx, x) for x in xs]
    mx.nd.waitall()
    before = mx.base.kernel_launch_count()
    out = mx.nd._invoke('_b200kv_clip_global_norm', arrays, num_arrays=n, max_norm='0.5')
    assert mx.base.kernel_launch_count() - before == 2 * ((n + 199) // 200) + 1
    norm = out.asnumpy()[0]
    for x, a in zip(xs, arrays):
        assert eq(a.asnumpy(), G.restate(norm, '0.5', x))
    before = mx.base.kernel_launch_count()
    mx.nd.contrib.multi_scale(*arrays, scalar=0.25)
    assert mx.base.kernel_launch_count() - before == (n + 199) // 200
    for x, a in zip(xs, arrays):
        assert eq(a.asnumpy(), G.multi_scale(G.restate(norm, '0.5', x), '0.25'))


def test_sizes_around_vector_tile_and_load_count(mx):
    t = G.TILE
    sizes = [1, 2, 3, 4, 5, 7, 8, 15, 16, 17, 255 * 4, 256 * 4, 256 * 4 + 1, 256 * 16 - 1, t - 4, t - 1, t, t + 1,
             t + 4, 2 * t - 1, 2 * t, 2 * t + 1, 3 * t + 1023, 3 * t + 1025]
    check_set(mx, _seeded(sizes, 3, 1.0), '0.75')
    for n in sizes:                     # and each alone
        check_set(mx, _seeded([n], n, 1.0), '0.01')


@pytest.mark.parametrize("shift", [1, 2, 3])
def test_bases_offset_by_4_8_12_bytes(mx, shift):
    """slices of larger arrays: the element-wise path; the elements outside the slice keep their bytes"""
    rng = np.random.default_rng(shift)
    ns = [G.TILE + 7, 5, 2 * G.TILE]
    wholes_h = [rng.standard_normal(n + shift + 2).astype(F) for n in ns]
    aligned_h = rng.standard_normal(1000).astype(F)
    made = []

    def make():
        wholes = [dev(mx, w) for w in wholes_h]
        made.append(wholes)
        return [w[shift:shift + n] for w, n in zip(wholes, ns)] + [dev(mx, aligned_h)]
    xs = [w[shift:shift + n] for w, n in zip(wholes_h, ns)] + [aligned_h]
    check_set(mx, xs, '0.5', make)
    for w, wh, n in zip(made[0], wholes_h, ns):
        got = w.asnumpy()
        assert eq(got[:shift], wh[:shift]) and eq(got[shift + n:], wh[shift + n:])


def test_empty_and_row_sparse_members(mx):
    rng = np.random.default_rng(11)
    shape = (50, 24)
    rows = rng.standard_normal((3, 24)).astype(F)
    ids = np.array([2, 17, 49], np.int64)
    rsp = mx.nd.sparse.row_sparse_array((rows, ids), shape=shape, ctx=mx.gpu(0))
    empty_rsp = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
    empty = dev(mx, np.zeros(0, F))
    d = rng.standard_normal(77).astype(F)
    dense = dev(mx, d)
    norm = clip(mx, [empty, rsp, empty_rsp, dense, empty], '0.3')[0]
    exact = np.sqrt(float(np.sum(rows.astype(np.float64) ** 2) + np.sum(d.astype(np.float64) ** 2)))
    assert abs(norm - exact) <= 1e-5 * exact
    assert eq(rsp.data.asnumpy(), G.restate(norm, '0.3', rows))
    assert eq(rsp.indices.asnumpy(), ids)
    assert eq(dense.asnumpy(), G.restate(norm, '0.3', d))
    assert empty_rsp.indices.shape[0] == 0
    dn = rsp.asnumpy()
    assert not dn[[0, 1, 3, 48]].any()
    # only empty members: norm 0, nothing to launch but the fold
    before = mx.base.kernel_launch_count()
    assert clip(mx, [empty, empty_rsp], '1.0')[0] == 0.0
    assert mx.base.kernel_launch_count() - before == 1
    mx.nd.contrib.multi_scale(rsp, empty, empty_rsp, scalar='3.0')
    assert eq(rsp.data.asnumpy(), G.multi_scale(G.restate(norm, '0.3', rows), '3.0'))
    assert eq(rsp.indices.asnumpy(), ids)


def test_total_norm_given_as_out(mx):
    a = dev(mx, np.full(16, 3.0))
    out = mx.nd.full((1,), 7.0, mx.gpu(0))
    mx.nd._invoke('_b200kv_clip_global_norm', [a], out=out, num_arrays=1, max_norm=6)
    assert out.asnumpy()[0] == 12.0
    assert eq(a.asnumpy(), G.restate(F(12.0), '6', np.full(16, 3.0, F)))


# -------------------------------------------------------------------------------- multi_scale
@pytest.mark.parametrize("name", sorted(G.SCALE_SETS))
def test_multi_scale_fixture(mx, golden, name):
    case, g = G.SCALE_SETS[name], golden("clip_global_norm")
    xs = G.scale_inputs(case, name)
    arrays = [dev(mx, x) for x in xs]
    mx.nd.contrib.multi_scale(*arrays, scalar=case['scalar'])
    for i, a in enumerate(arrays):
        # a nan result is a nan in the same place: the GPU writes its canonical nan (0x7FFFFFFF)
        # where the CPU keeps the operand's payload or gives the default nan
        got, want = a.asnumpy(), g['mscale_%s_out%d' % (name, i)].view(F)
        assert np.array_equal(np.isnan(got), np.isnan(want)), (name, i)
        assert eq(np.where(np.isnan(want), F(0), got), np.where(np.isnan(want), F(0), want)), (name, i)


def test_multi_scale_by_one_writes_nothing(mx):
    x = np.array([1.0, np.nan, np.inf, -0.0, 1e-45], F)
    x.view(np.uint32)[1] = 0x7FA00001          # a signalling nan keeps its payload
    a = dev(mx, x)
    mx.nd.contrib.multi_scale(a, scalar=1)
    assert eq(a.asnumpy(), x)
    mx.nd.contrib.multi_scale(a, scalar='1.00000001')   # rounds to 1.0f
    assert eq(a.asnumpy(), x)


# ----------------------------------------------------------------------------------- ordering
def test_back_to_back_without_waits_equals_step_by_step(mx):
    """overflow check, unscale, clip and a multi-tensor SGD-momentum update over the same gradients,
    issued back to back with no host wait, against the same calls with a wait after each"""
    rng = np.random.default_rng(77)
    sizes = [int(s) for s in rng.integers(1, 9000, 230)]
    w0 = _seeded(sizes, 1, 1.0)
    g0 = _seeded(sizes, 2, 65536.0)

    def run(wait):
        ws, gs = [dev(mx, w) for w in w0], [dev(mx, g) for g in g0]
        ms = [dev(mx, np.zeros(n)) for n in sizes]
        flag = mx.nd.full((1,), 1.0, mx.gpu(0))
        for _ in range(3):
            steps = [
                lambda: [mx.nd.multi_all_finite(*gs[i:i + 200], num_arrays=len(gs[i:i + 200]),
                                                init_output=False, out=flag) for i in (0, 200)],
                lambda: mx.nd.contrib.multi_scale(*gs, scalar=1.0 / 256),
                lambda: mx.gluon.utils.clip_global_norm(gs, 10.0, check_isfinite=False),
            ]
            for i in range(0, len(ws), 40):
                sl = slice(i, i + 40)
                flat = [a for t in zip(ws[sl], gs[sl], ms[sl]) for a in t]
                k = len(ws[sl])
                steps.append(lambda flat=flat, k=k, sl=sl: mx.nd.multi_sgd_mom_update(
                    *flat, out=ws[sl], num_weights=k, lrs=(0.1,) * k, wds=(1e-4,) * k, momentum=0.9))
            for s in steps:
                s()
                if wait:
                    mx.nd.waitall()
        return [w.asnumpy() for w in ws], [m.asnumpy() for m in ms], [g.asnumpy() for g in gs], flag.asnumpy()

    a, b = run(False), run(True)
    for xs, ys in zip(a[:3], b[:3]):
        for x, y in zip(xs, ys):
            assert eq(x, y)
    assert eq(a[3], b[3]) and a[3][0] == 1.0


# ----------------------------------------------------------------------------------- refusals
def test_refusals_leave_operands_unchanged(mx):
    x = np.arange(1, 11, dtype=F)
    g32, other = dev(mx, x), dev(mx, x)
    g16 = mx.nd.array(x.astype(np.float16), mx.gpu(0), np.float16)
    cpu = mx.nd.array(x, mx.cpu())
    op, ms = '_b200kv_clip_global_norm', '_b200kv_multi_scale'
    bad_out = [mx.nd.full((2,), 7.0, mx.gpu(0)), mx.nd.full((1,), 7.0, mx.cpu()),
               mx.nd.array(np.full(1, 7.0, np.float16), mx.gpu(0), np.float16)]
    cases = [
        (op, [g32], dict(max_norm=1.0), None, 'Required parameter num_arrays'),
        (op, [g32], dict(num_arrays=0, max_norm=1.0), None, 'num_arrays must be at least 1'),
        (op, [g32, other], dict(num_arrays=1, max_norm=1.0), None, 'expected num_arrays inputs'),
        (op, [g32, g16], dict(num_arrays=2, max_norm=1.0), None, 'array_1 is float16.*16-bit gradients are not served'),
        (op, [g32, cpu], dict(num_arrays=2, max_norm=1.0), None, 'no CPU fallback'),
        (op, [cpu], dict(num_arrays=1, max_norm=1.0), None, 'no CPU fallback'),
        (op, [g32], dict(num_arrays=1), None, 'Required parameter max_norm'),
        (op, [g32], dict(num_arrays=1, max_norm='nan'), None, 'max_norm must be positive'),
        (op, [g32], dict(num_arrays=1, max_norm=0), None, 'max_norm must be positive'),
        (op, [g32], dict(num_arrays=1, max_norm=-2.0), None, 'max_norm must be positive'),
        (op, [g32], dict(num_arrays=1, max_norm='abc'), None, 'cannot parse max_norm'),
        (op, [g32], dict(num_arrays=1, max_norm=1.0, wd=0.1), None, "Cannot find argument 'wd'"),
        (op, [g32, other, g32], dict(num_arrays=3, max_norm=1.0), None, 'same storage listed twice'),
        (op, [g32, g32[2:5]], dict(num_arrays=2, max_norm=1.0), None, 'same storage listed twice'),
        (ms, [g32], dict(scalar=0.5), None, 'Required parameter num_arrays'),
        (ms, [g32], dict(num_arrays=1), None, 'Required parameter scalar'),
        (ms, [g32], dict(num_arrays=1, scalar=0.5, max_norm=1), None, "Cannot find argument 'max_norm'"),
        (ms, [g16], dict(num_arrays=1, scalar=0.5), None, '16-bit gradients are not served'),
        (ms, [g32, g32], dict(num_arrays=2, scalar=0.5), None, 'same storage listed twice'),
        (ms, [g32, cpu], dict(num_arrays=2, scalar=0.5), None, 'no CPU fallback'),
        (ms, [g32], dict(num_arrays=1, scalar=0.5), other, 'has no output'),
    ] + [(op, [g32], dict(num_arrays=1, max_norm=1.0), o, r'total_norm must be a dense \(1,\) float32') for o in bad_out]
    for name, arrays, params, out, msg in cases:
        outs = [] if out is None else [out]
        before = [o.asnumpy().copy() for o in outs]
        with pytest.raises(mx.base.MXNetError, match=msg):
            mx.nd._invoke(name, arrays, out=out, **params)
        for a in (g32, other, cpu):
            assert eq(a.asnumpy(), x), (name, msg)
        assert eq(g16.asnumpy(), x.astype(np.float16))
        for o, b in zip(outs, before):
            assert eq(o.asnumpy(), b), (name, msg)
    # disjoint slices of one array are two operands, not one storage twice
    clip(mx, [g32[0:5], g32[5:10]], '1.0')
    assert eq(g32.asnumpy(), G.restate(np.sqrt(F(385.0)), '1.0', x))
