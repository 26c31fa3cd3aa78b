"""add_n / ElementWiseSum on the GPU, bit for bit against tests/golden/add_n.npz (the reference's own
outputs; NaNs by position): every dtype at n = 1, 2, 3, 4, 5, 9, 200 and 201 with signed zeros, inf,
NaN and integer wrap-around, 16-byte aligned and unaligned operands, out = input 0, the
all-row_sparse, > 4 dense-containing and <= 4 fallback forms, a 1 M x 512 row_sparse sum and a
64 M-element dense sum against the restatement, the launch counts, and every refusal with nothing
launched and out unchanged."""
import numpy as np
import pytest

import golden_add_n as GAN

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def host(bits, dtype):
    """raw bits -> what mx.nd.array uploads bit for bit (bfloat16 travels as its float32 widening)"""
    if dtype == 'bfloat16':
        return GAN.widen_bf16(bits)
    return GAN.values(bits, dtype)


def bits_of(a, dtype):
    x = a.asnumpy()
    if dtype == 'bfloat16':
        return (x.view(np.uint32) >> 16).astype(np.uint16)
    return x.view(GAN.RAW[dtype])


def upload(mx, bits, dtype, shift=0):
    """a dense GPU array of the raw bits, starting `shift` elements into a larger allocation"""
    flat = np.asarray(bits).reshape(-1)
    if shift == 0:
        return mx.nd.array(host(bits, dtype), mx.gpu(0), dtype)
    assert len(np.shape(bits)) == 1
    pad = np.concatenate([flat[:shift], flat])
    return mx.nd.array(host(pad, dtype), mx.gpu(0), dtype)[shift:shift + len(flat)]


def operands(mx, case, ins, shift=0):
    out = []
    for s, a in zip(case['stypes'], ins):
        if s == 'row_sparse':
            ids, rows = a
            out.append(mx.nd.sparse.row_sparse_array((rows, ids), shape=case['shape'], ctx=mx.gpu(0)))
        else:
            out.append(upload(mx, a, case['dtype'], shift))
    return out


def check(case, name, got, g):
    if all(s == 'row_sparse' for s in case['stypes']):
        assert got.stype == 'row_sparse', name
        assert np.array_equal(got.indices.asnumpy(), g[name + '_idx']), name
        assert GAN.same_bits(got.data.asnumpy().reshape(g[name + '_val'].shape), g[name + '_val']), name
    else:
        assert got.stype == 'default', name
        assert GAN.same_bits(bits_of(got, case['dtype']), g[name], case['dtype']), name


@pytest.mark.parametrize("name", sorted(GAN.CASES))
def test_fixture_case(mx, golden, name):
    """default out, then a given out"""
    case = GAN.CASES[name]
    ins = GAN.inputs(case, name)
    arrays = operands(mx, case, ins)
    check(case, name, mx.nd.add_n(*arrays), golden("add_n"))
    if all(s == 'row_sparse' for s in case['stypes']):
        out = mx.nd.sparse.zeros('row_sparse', case['shape'], mx.gpu(0))
        mx.nd.sparse.add_n(*arrays, out=out)
    else:
        out = mx.nd.empty(case['shape'], mx.gpu(0), case['dtype'])
        mx.nd.ElementWiseSum(*arrays, out=out)
    check(case, name, out, golden("add_n"))


DENSE = sorted(n for n, c in GAN.CASES.items() if set(c['stypes']) == {'default'} and len(c['stypes']) in (2, 5, 201))


@pytest.mark.parametrize("name", DENSE)
def test_unaligned_slices(mx, golden, name):
    """inputs starting one element into their allocation (the scalar path), with an aligned out and
    then an unaligned one; one aligned input among unaligned ones"""
    case = GAN.CASES[name]
    ins = GAN.inputs(case, name)
    arrays = operands(mx, case, ins, shift=1)
    check(case, name, mx.nd.add_n(*arrays), golden("add_n"))
    out = upload(mx, np.zeros(GAN.SIZE, GAN.RAW[case['dtype']]), case['dtype'], shift=1)
    mx.nd.add_n(*arrays, out=out)
    check(case, name, out, golden("add_n"))
    mixed = operands(mx, case, ins[:1]) + arrays[1:]
    check(case, name, mx.nd.add_n(*mixed), golden("add_n"))


@pytest.mark.parametrize("name", ['float32_n3', 'float16_n4', 'int8_n9', 'float64_n201', 'bfloat16_n2',
                                  'mix_gt4_dense_first', 'mix_le4_drd', 'rsp_overlap', 'rsp_n20'])
def test_out_is_input0(mx, golden, name):
    case = GAN.CASES[name]
    arrays = operands(mx, case, GAN.inputs(case, name))
    got = mx.nd.add_n(*arrays, out=arrays[0])
    assert got is arrays[0]
    check(case, name, arrays[0], golden("add_n"))


def test_neg_zero_in_an_absent_row(mx):
    """> 4 inputs with a dense one: a -0.0 where no row_sparse input holds the row stays -0.0 when
    input 0 is dense; a row_sparse input 0 starts out at +0.0, and the <= 4 fallback adds +0.0"""
    for name, want in (('mix_gt4_dense_first', 0x80000000), ('mix_gt4_one_dense', 0),
                       ('mix_gt4_rsp_first', 0), ('mix_le4_dr', 0), ('mix_le4_rrdr', 0)):
        case = GAN.CASES[name]
        got = mx.nd.add_n(*operands(mx, case, GAN.inputs(case, name)))
        assert got.asnumpy().view(np.uint32)[6, 3] == want, name


def test_launch_counts(mx):
    """all dense: one launch up to 200 inputs, two at 201; nothing for an empty out or all-empty
    row_sparse inputs"""
    arrays = [mx.nd.array(np.full(1000, k, np.float32), mx.gpu(0)) for k in range(201)]
    out = mx.nd.empty((1000,), mx.gpu(0))
    for n, want in ((1, 1), (2, 1), (4, 1), (5, 1), (200, 1), (201, 2)):
        out.wait_to_read()
        before = mx.base.kernel_launch_count()
        mx.nd.add_n(*arrays[:n], out=out)
        assert mx.base.kernel_launch_count() - before == want, n
        assert np.array_equal(out.asnumpy(), np.full(1000, sum(range(n)), np.float32)), n
    empty = mx.nd.array(np.zeros(0, np.float32), mx.gpu(0))
    before = mx.base.kernel_launch_count()
    assert mx.nd.add_n(empty, empty).shape == (0,)
    z = [mx.nd.sparse.zeros('row_sparse', (50, 8), mx.gpu(0)) for _ in range(3)]
    r = mx.nd.sparse.add_n(*z)
    assert r.stype == 'row_sparse' and r.indices.shape == (0,)
    assert mx.base.kernel_launch_count() - before == 0


def test_refusals_launch_nothing_and_keep_out(mx):
    g = mx.gpu(0)
    a = mx.nd.array(np.arange(12, dtype=np.float32), g)
    b = mx.nd.array(np.ones(12, np.float32), g)
    h = mx.nd.array(np.ones(12, np.float16), g, np.float16)
    c = mx.nd.array(np.ones(13, np.float32), g)
    cpu = mx.nd.array(np.ones(12, np.float32), mx.cpu())
    big = mx.nd.array(np.arange(24, dtype=np.float32), g)
    rsp = mx.nd.sparse.row_sparse_array((np.ones((2, 4), np.float32), np.array([0, 2])), shape=(3, 4), ctx=g)
    d34 = mx.nd.array(np.ones((3, 4), np.float32), g)
    rsp16 = mx.nd.sparse.zeros('row_sparse', (3, 4), g, np.float16)
    cases = [
        ([a, b], dict(num_args=3), None, 'expected num_args inputs'),
        ([a, b], dict(num_args=1), None, 'expected num_args inputs'),
        ([a], dict(num_args=0), None, 'num_args must be at least 1'),
        ([a, b], dict(num_args=2, axis=0), None, "Cannot find argument 'axis'"),
        ([a, c], {}, None, 'shape differs from input 0'),
        ([a, h], {}, None, 'dtype differs from input 0'),
        ([a, cpu], {}, None, 'no CPU fallback'),
        ([cpu, cpu], {}, None, 'no CPU fallback'),
        ([a, b], {}, mx.nd.empty((12,), mx.cpu()), 'no CPU fallback'),
        ([rsp16, rsp16], {}, None, 'row_sparse inputs are float32'),
        ([d34, rsp], {}, mx.nd.sparse.zeros('row_sparse', (3, 4), g), 'out must be default'),
        ([rsp, rsp], {}, mx.nd.empty((3, 4), g), 'out must be row_sparse'),
        ([a, b], {}, mx.nd.empty((13,), g), 'out has the wrong shape'),
        ([a, b], {}, mx.nd.empty((12,), g, np.float16), 'out dtype differs'),
        ([a, b, a], {}, a, 'out overlaps input 2'),
        ([a, b], {}, b, 'out overlaps input 1'),
        ([big[12:24], big[6:18]], {}, big[0:12], 'out overlaps input 1'),
        ([big[0:12], b], {}, big[1:13], 'out overlaps input 0'),
        ([rsp, rsp], {}, rsp, 'out overlaps input 1'),
    ]
    for arrays, params, out, msg in cases:
        watched = [x for x in arrays + ([out] if out is not None else []) if x.stype == 'default']
        before = [x.asnumpy().copy() for x in watched]
        rsp_before = rsp.indices.asnumpy().copy(), rsp.data.asnumpy().copy()
        mx.nd.waitall()
        n0 = mx.base.kernel_launch_count()
        with pytest.raises(mx.base.MXNetError, match=msg):
            mx.nd.add_n(*arrays, out=out, **params)
        assert mx.base.kernel_launch_count() == n0, msg
        for x, want in zip(watched, before):
            assert np.array_equal(x.asnumpy().view(np.uint8), want.view(np.uint8)), msg
        assert np.array_equal(rsp.indices.asnumpy(), rsp_before[0]) and np.array_equal(rsp.data.asnumpy(), rsp_before[1])


def test_large_row_sparse(mx):
    """8 row_sparse inputs of 10 000 random rows each of a 1 M x 512 table, against the restatement"""
    rng = np.random.default_rng(5)
    shape = (1_000_000, 512)
    ins = [(np.sort(rng.choice(shape[0], 10_000, replace=False)).astype(np.int64),
            rng.standard_normal((10_000, 512)).astype(np.float32)) for _ in range(8)]
    case = dict(dtype='float32', stypes=['row_sparse'] * 8, shape=shape)
    got = mx.nd.sparse.add_n(*operands(mx, case, ins))
    ids, rows = GAN.restate(case, ins)
    assert np.array_equal(got.indices.asnumpy(), ids)
    assert np.array_equal(got.data.asnumpy().view(np.uint32), rows.view(np.uint32))


def test_large_dense(mx):
    """64 M float32 elements, 3 and 5 inputs, against the restatement"""
    rng = np.random.default_rng(6)
    n = 64 * 1024 * 1024
    ins = [rng.standard_normal(n, dtype=np.float32).view(np.uint32) for _ in range(5)]
    arrays = [mx.nd.array(x.view(np.float32), mx.gpu(0)) for x in ins]
    for k in (3, 5):
        got = mx.nd.add_n(*arrays[:k]).asnumpy().view(np.uint32)
        assert np.array_equal(got, GAN.fold(ins[:k], 'float32')), k
