"""The NDArray arithmetic, fill and cast operators on the GPU, bit for bit against the reference's
own code (tests/golden/ndarray_ops.npz, written by oracle/golden_ndarray_ops.py) and its numpy
restatement, on float16, bfloat16, float32, float64, int32 and int64:

- `+`, `-`, `*` with an array and with a scalar, `+=`, `-=`, `*=`, `sqrt`, `a[:] = v` and `astype`
  over the 6 x 6 dtype matrix;
- sizes 1, 7, 4099 and 2^20 + 3, the last past the kernels' grid-stride cap of 540,672 elements;
- a new result, `out` = the input, a distinct `out`, `a += a`, and slice views `a[1:]` whose
  preceding element must stay as it was;
- scalars whose dmlc::stof and std::stod parses differ, scalars half or bfloat16 cannot represent,
  negative and fractional scalars on integers; assigned values 2^24 + 1, 2^53 - 1, 0.1 and -0.0;
  cast edges: the int32 range ends, 2^53 +- 1, subnormals, half overflow, rounding ties, and NaN
  and inf between float types.

NaN compares as NaN (the GPU writes its canonical NaN). What the reference leaves undefined is not
tested: signed integer overflow, float-to-int conversion of NaN, inf or out-of-range values, and
integer sqrt of negatives. uint8 and int8 arithmetic, and casts to them, are refused cleanly."""
import numpy as np
import pytest

import golden_ndarray_ops as G

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


@pytest.fixture(scope="module")
def fixture():
    d = np.load(G.os.path.join(G.GOLD, "ndarray_ops.npz"))
    return {str(n): (s, h) for n, s, h in zip(d['names'], d['sha256'], d['head'])}


def up(mx, x, dt):
    """a GPU array holding exactly x's bits"""
    if dt == 'bfloat16':
        return mx.nd.array(G.bf16_to_f32(x), mx.gpu(0), dtype='bfloat16')
    return mx.nd.array(np.ascontiguousarray(x, G.STORE[dt]), mx.gpu(0), dtype=G.STORE[dt])


def down(nd, dt):
    x = nd.asnumpy()
    if dt == 'bfloat16':
        return (x.view(np.uint32) >> 16).astype(np.uint16)
    return x


def check(got, want, dt, what):
    """bit equality, NaN as NaN, with the first differences named"""
    if G.same(got, want, dt):
        return
    a, b = G.canon(got, dt), G.canon(want, dt)
    u = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.itemsize]
    bad = np.nonzero(a.view(u) != b.view(u))[0] if a.shape == b.shape else []
    lines = ['%s: %d of %d elements differ' % (what, len(bad), b.size)]
    for i in bad[:6]:
        lines.append('  [%d] got %r want %r' % (i, a[i], b[i]))
    pytest.fail('\n'.join(lines))


def check_fixture(fixture, name, got, dt):
    sha, head = fixture[name]
    assert np.array_equal(G.head_bytes(got, dt), head), name + ': head differs from the reference'
    assert np.array_equal(G.sha256(got, dt), sha), name + ': differs from the reference'


def fill(mx, n, dt, seed):
    """an out array holding seeded values, to see that every element is written"""
    x = G.operands('out|%d' % seed, n, dt, 'plus')[0]
    return up(mx, x, dt), x


# --------------------------------------------------------------------------------- array ops
IOP = {'plus': '__iadd__', 'minus': '__isub__', 'mul': '__imul__'}
NAME = {'plus': '_plus', 'minus': '_minus', 'mul': '_mul'}
ALIAS = {'plus': 'elemwise_add', 'minus': 'elemwise_sub', 'mul': 'elemwise_mul'}


@pytest.mark.parametrize("case", G.array_cases(), ids=lambda c: c[0])
def test_array_operator(mx, fixture, case):
    name, op, dt, n = case
    a, b = G.inputs('array', case)
    want = G.restate('array', case)
    A, B = up(mx, a, dt), up(mx, b, dt)
    if op == 'sqrt':
        got = down(mx.nd.sqrt(A), dt)
        check(got, want, dt, name)
        check_fixture(fixture, name, got, dt)
        O, _ = fill(mx, n, dt, 1)
        mx.nd.sqrt(A, out=O)                                   # a distinct out
        check(down(O, dt), want, dt, name + ' out=')
        check(down(A, dt), a, dt, name + ' input kept')
        mx.nd.sqrt(A, out=A)                                   # out = the input
        check(down(A, dt), want, dt, name + ' in place')
        return
    got = down({'plus': A + B, 'minus': A - B, 'mul': A * B}[op], dt)
    check(got, want, dt, name)
    check_fixture(fixture, name, got, dt)
    for opname in (NAME[op], ALIAS[op]):
        O, _ = fill(mx, n, dt, 2)
        mx.nd._invoke(opname, [A, B], out=O)
        check(down(O, dt), want, dt, '%s %s out=' % (name, opname))
        check_fixture(fixture, name, down(O, dt), dt)
    check(down(A, dt), a, dt, name + ' input kept')
    R = getattr(A, IOP[op])(B)                                  # a op= b
    assert R is A
    check(down(A, dt), want, dt, name + ' in place')
    check(down(B, dt), b, dt, name + ' other operand kept')


@pytest.mark.parametrize("dt", G.DTYPES)
@pytest.mark.parametrize("n", [7, (1 << 20) + 3])
def test_self_aliasing(mx, dt, n):
    """a += a, a *= a and a - a read and write the same memory"""
    for op in ('plus', 'mul', 'minus'):
        a = G.operands('alias|%s|%s|%d' % (op, dt, n), n, dt, 'mul' if op == 'mul' else 'plus')[0]
        A = up(mx, a, dt)
        mx.nd._invoke(NAME[op], [A, A], out=A)
        check(down(A, dt), G.binary(op, a, a, dt), dt, '%s a,a %s %d' % (op, dt, n))


@pytest.mark.parametrize("dt", G.DTYPES)
@pytest.mark.parametrize("n", [1, 4099, (1 << 20) + 3])
def test_slice_views(mx, dt, n):
    """operators on a[1:] write the view and leave the element before it as it was"""
    base = G.operands('view|%s|%d' % (dt, n), n + 1, dt, 'plus')[0]
    b = G.operands('view-b|%s|%d' % (dt, n), n, dt, 'plus')[0]
    s = '0.30000000000000004'
    for what, run, want in [
            ('+=', lambda V, B: V.__iadd__(B), lambda v: G.binary('plus', v, b, dt)),
            ('*= s', lambda V, B: V.__imul__(float(s)), lambda v: G.binary_scalar('mul', v, s, dt)),
            ('sqrt', lambda V, B: mx.nd.sqrt(V, out=V), lambda v: G.sqrt(v, dt)),
            ('[:] =', lambda V, B: V.__setitem__(slice(None), 0.1), lambda v: G.full(0.1, n, dt))]:
        if what == 'sqrt' and dt not in G.FLOATS:
            base = np.abs(base)
        Base = up(mx, base, dt)
        V = Base[1:]
        run(V, up(mx, b, dt))
        got = down(Base, dt)
        check(got[:1], base[:1], dt, '%s %s %d: element before the view' % (what, dt, n))
        check(got[1:], want(base[1:]), dt, '%s %s %d' % (what, dt, n))


# -------------------------------------------------------------------------------- scalar ops
@pytest.mark.parametrize("dt", G.DTYPES)
def test_scalar_operators(mx, fixture, dt):
    """`a + s`, `a - s`, `a * s` and their in-place forms for every scalar of the fixture"""
    for case in G.scalar_cases():
        name, op, _, s = case
        if case[2] != dt:
            continue
        a = G.inputs('scalar', case)[0]
        want = G.restate('scalar', case)
        A = up(mx, a, dt)
        got = down({'plus': A + float(s), 'minus': A - float(s), 'mul': A * float(s)}[op], dt)
        check(got, want, dt, '%s (scalar %s)' % (name, s))
        check_fixture(fixture, name, got, dt)
        getattr(A, IOP[op])(float(s))
        check(down(A, dt), want, dt, '%s in place (scalar %s)' % (name, s))


@pytest.mark.parametrize("dt", G.DTYPES)
def test_assignment(mx, fixture, dt):
    """a[:] = v is the reference's _full: dmlc::stod of repr(float(v)), then static_cast<DType>"""
    for case in G.full_cases():
        name, cdt, v, n = case
        if cdt != dt:
            continue
        A, _ = fill(mx, n, dt, 3)
        A[:] = v
        got = down(A, dt)
        check(got, G.full(v, n, dt), dt, '%s (value %r)' % (name, v))
        check_fixture(fixture, name, got, dt)
    if dt == 'float32':
        # _set_value: a fill from its float src, with a value float32 holds exactly
        A, _ = fill(mx, 4099, dt, 3)
        mx.nd._invoke('_set_value', [], out=A, src=0.375)
        check(down(A, dt), G.full(0.375, 4099, dt), dt, '_set_value')


# ---------------------------------------------------------------------------------------- casts
@pytest.mark.parametrize("dst", G.DTYPES)
@pytest.mark.parametrize("src", G.DTYPES)
def test_cast(mx, fixture, src, dst):
    for n in G.SIZES:
        case = ('cast|%s|%s|%d' % (src, dst, n), src, dst, n)
        x = G.inputs('cast', case)[0]
        want = G.restate('cast', case)
        X = up(mx, x, src)
        for result in (X.astype(dst), mx.nd._invoke('Cast', [X], dtype=dst)):
            got = down(result, dst)
            check(got, want, dst, case[0])
            check_fixture(fixture, case[0], got, dst)
        if n <= 4099:
            O, _ = fill(mx, n, dst, 4)
            mx.nd.cast(X, dtype=dst, out=O)
            check(down(O, dst), want, dst, case[0] + ' out=')
        check(down(X, src), x, src, case[0] + ' input kept')


# ------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("dt", [np.uint8, np.int8])
def test_8bit_arithmetic_is_refused_cleanly(mx, dt):
    x = np.arange(1, 8).astype(dt)
    A = mx.nd.array(x, mx.gpu(0), dtype=dt)
    F = mx.nd.array(np.arange(7, dtype=np.float32), mx.gpu(0))
    for fn in [lambda: A + A, lambda: A - A, lambda: A * A, lambda: A + 1, lambda: A * 2.5,
               lambda: A.__iadd__(A), lambda: A.__imul__(3), lambda: mx.nd.sqrt(A),
               lambda: mx.nd.sqrt(A, out=A), lambda: A.__setitem__(slice(None), 3)]:
        with pytest.raises(mx.base.MXNetError, match='elementwise operators take float16'):
            fn()
        assert np.array_equal(A.asnumpy(), x)
    for target in ('uint8', 'int8'):
        with pytest.raises(mx.base.MXNetError, match='cast: unsupported dtype'):
            F.astype(target)
    O = mx.nd.array(x, mx.gpu(0), dtype=dt)
    with pytest.raises(mx.base.MXNetError, match='out dtype differs'):
        mx.nd.cast(F, dtype='float32', out=O)
    assert np.array_equal(O.asnumpy(), x)
    assert np.array_equal(F.asnumpy(), np.arange(7, dtype=np.float32))
