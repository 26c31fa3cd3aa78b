"""TEST INFRASTRUCTURE ONLY -- the operators the dense-gradient branches of the reference's AdaGrad and
GroupAdaGrad add to the Adamax / Nadam / AdaDelta arithmetic (square; mean over the last axis;
broadcast_add / _sub / _mul / _div / _maximum with an rhs of one value per row): numpy restatements
per dtype, the reference's own code (`ref()` over oracle/_ref/libmxref_dense_adagrad.so, built from
oracle/ref_dense_adagrad.cc by oracle/dense_adagrad.mk), the seeded cases, and the writer of
tests/golden/dense_adagrad_ops.npz:

    make -f oracle/dense_adagrad.mk && python oracle/golden_dense_adagrad.py

Arrays, dtypes, the fixture format (a sha256 and the first bytes of each output, NaN payloads
canonical) and the helpers are those of oracle/golden_ndarray_ops.py. What is restated, per dtype:

- square is math::sqr: float(a) * float(a) for every dtype but float64, then DType(...): the 16-bit
  types round to nearest even, integers truncate (so an integer above 2^12 squares through float and
  can lose bits). float64 squares in double. An integer square outside the integer range is
  undefined in the reference and is not among the cases.
- mean folds each row left to right with red::sum's Kahan step in the dtype, every operation rounded
  to it (float16 / bfloat16: computed in float32, rounded once):
      y = x - r;  t = s + y;  r = 0 if isinf(t) else (t - s) - y;  s = t
  from s = r = 0, then divides s by DType(C), the row length converted to the dtype (float16 and
  bfloat16 round it from float32). bfloat16 is not in the reference; it is restated the same way.
- the row broadcasts are golden_arith_ops' per-dtype functors with rhs[i // C].
"""
import ctypes
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import golden_arith_ops as GA  # noqa: E402
import golden_ndarray_ops as GN  # noqa: E402

GOLD = GN.GOLD
DTYPES, FLOATS, SIXTEEN, STORE, F32 = GN.DTYPES, GN.FLOATS, GN.SIXTEEN, GN.STORE, GN.F32
BINARY = ('broadcast_add', 'broadcast_sub', 'broadcast_mul', 'broadcast_div', 'broadcast_maximum')
# the row-mean kernel's tile (reduce_kernels.cu): 32 rows per CTA, 32 columns per tile, and its
# grid cap of 132 SMs x 32 CTAs; WAVE rows fill one pass of the grid-stride loop
TILE = 32
WAVE = 132 * 32 * 32


def build():
    """oracle/_ref/libmxref_dense_adagrad.so, where the reference's sources exist"""
    if os.path.isfile("/root/reference/src/operator/tensor/broadcast_reduce_op.h"):
        import subprocess
        subprocess.run(["make", "-s", "-f", os.path.join(HERE, "dense_adagrad.mk")], check=True)


# ------------------------------------------------------------------------------- restatement
def square(a, dt):
    a = np.asarray(a, STORE[dt])
    with np.errstate(all='ignore'):
        if dt in SIXTEEN:
            f = GN.to_f32(a, dt)
            return GN.from_f32(f * f, dt)
        if dt in FLOATS:
            return (a * a).astype(STORE[dt])
        f = a.astype(F32)
        return np.trunc(f * f).astype(STORE[dt])


def _rounder(dt):
    """the value an operation leaves in a DType variable, in the arithmetic type"""
    if dt in SIXTEEN:
        return lambda x: GN.to_f32(GN.from_f32(x, dt), dt)
    return lambda x: x


def _arith(x, dt):
    """the array in its arithmetic type: float32 for the 16-bit types"""
    return GN.to_f32(x, dt) if dt in SIXTEEN else np.asarray(x, STORE[dt])


def _finish(s, cols, dt):
    """s / DType(cols), in the dtype's storage"""
    R = _rounder(dt)
    ctype = np.float64 if dt == 'float64' else F32
    with np.errstate(all='ignore'):
        q = R(s / R(np.full(s.shape, cols, ctype)))
    return GN.from_f32(q, dt) if dt in SIXTEEN else q.astype(STORE[dt])


def row_fold_kahan(x2, dt):
    """the reference's fold of each row of a (rows, cols) array, in the arithmetic type"""
    R = _rounder(dt)
    v = _arith(x2, dt)
    s = np.zeros(v.shape[0], v.dtype)
    r = np.zeros(v.shape[0], v.dtype)
    with np.errstate(all='ignore'):
        for k in range(v.shape[1]):
            y = R(v[:, k] - r)
            t = R(s + y)
            r = np.where(np.isinf(t), v.dtype.type(0), R(R(t - s) - y))
            s = t
    return s


def mean_rows(x, dt, fold=row_fold_kahan):
    """mean over the last axis, keepdims=False, through `fold` (rows, cols) -> (rows,)"""
    x = np.asarray(x, STORE[dt])
    cols = x.shape[-1]
    s = fold(x.reshape(int(np.prod(x.shape[:-1])), cols), dt)
    return _finish(s, cols, dt).reshape(x.shape[:-1])


def row_broadcast(op, a, b, dt):
    """op(lhs, rhs) with rhs of shape lhs.shape[:-1] + (1,)"""
    return GA.restate_array(op, a, np.broadcast_to(b, a.shape), dt).reshape(a.shape)


# folds that order or group a row differently; each gives other bits than the reference's on the
# fixture's mixed-magnitude rows (tests/test_dense_adagrad_host.py)
def row_fold_naive(x2, dt):
    R = _rounder(dt)
    v = _arith(x2, dt)
    s = np.zeros(v.shape[0], v.dtype)
    with np.errstate(all='ignore'):
        for k in range(v.shape[1]):
            s = R(s + v[:, k])
    return s


def row_fold_pairwise(x2, dt):
    R = _rounder(dt)
    v = _arith(x2, dt)
    with np.errstate(all='ignore'):
        while v.shape[1] > 1:
            if v.shape[1] % 2:
                v = np.concatenate([v, np.zeros((v.shape[0], 1), v.dtype)], axis=1)
            v = R(v[:, 0::2] + v[:, 1::2])
    return v[:, 0] if v.shape[1] else np.zeros(v.shape[0], v.dtype)


def row_fold_warp_tree(x2, dt):
    """32 lanes: lane l folds elements l, l + 32, ... with the Kahan step, then a shuffle tree of
    the 32 partial sums"""
    v = _arith(x2, dt)
    lanes = []
    for lane in range(32):
        part = v[:, lane::32]
        lanes.append(row_fold_kahan(part, dt) if part.shape[1] else np.zeros(v.shape[0], v.dtype))
    R = _rounder(dt)
    p = np.stack(lanes, axis=1)
    with np.errstate(all='ignore'):
        while p.shape[1] > 1:
            h = p.shape[1] // 2
            p = R(p[:, :h] + p[:, h:])
    return p[:, 0]


FOLDS = {'naive': row_fold_naive, 'pairwise': row_fold_pairwise, 'warp_tree': row_fold_warp_tree}


# ------------------------------------------------------------------------------------- cases
def _rng(name):
    return GN._rng('dense_adagrad|' + name)


def square_cases():
    """(name, dtype, n)"""
    return [('square|%s|%d' % (dt, n), dt, n) for dt in DTYPES for n in (1, 7, 4099, (1 << 20) + 3)]


SQUARE_EDGES = [0.0, -0.0, 1.0, -1.0, 0.1, 2.5, 255.0, 256.0, 257.0, 300.0, -300.0, 65504.0, 1e19,
                1.9e19, 1e20, 1e154, 1e155, 2 ** -13, 2 ** -24, 1e-23, 1e-160, 1 + 2 ** -11,
                math.inf, -math.inf, math.nan]
# int32 squares stay below 2^31 (|a| <= 46340); int64 below 2^62
SQUARE_INT_EDGES = {'int32': [0, 1, -1, 4095, 4096, 4097, -4097, 8191, 46340, -46340, 46339],
                    'int64': [0, 1, -1, 4097, 46341, 16777217, 2 ** 31 - 1, -(2 ** 31 - 1), 3037000, 67108865]}


def square_operand(name, dt, n):
    rng = _rng(name)
    if dt in FLOATS:
        x = GN._floats(rng, n, dt, -20, 20)
        e = np.array(SQUARE_EDGES, np.float64)
        with np.errstate(over='ignore'):
            e = GN.from_f32(e.astype(F32), dt) if dt in SIXTEEN else e.astype(STORE[dt])
    else:
        lim = 46340 if dt == 'int32' else 2 ** 31 - 1
        x = rng.integers(-lim, lim, n, dtype=STORE[dt], endpoint=True)
        e = np.array(SQUARE_INT_EDGES[dt], STORE[dt])
    k = min(n, len(e))
    x[:k] = e[:k]
    return x


# (rows, cols) and the ways of spelling the last axis; `mixed` rows put 1e3 beside 0.1
MEAN_COLS = (1, 2, 31, 32, 33, 63, 64, 65, 97, 4099)
MEAN_ROWS = (1, 7, 100)


def mean_cases():
    """(name, dtype, shape, axis string, keepdims string, values)"""
    out = []
    for dt in FLOATS:
        for c in MEAN_COLS:
            for r in MEAN_ROWS:
                if r * c > 200000:
                    continue
                out.append(('mean|%s|%dx%d|mixed' % (dt, r, c), dt, (r, c), '1', 'True', 'mixed'))
        out.append(('mean|%s|wave|mixed' % dt, dt, (WAVE + 37, 3), '-1', 'True', 'mixed'))
        out.append(('mean|%s|2wave|signed' % dt, dt, (2 * WAVE + 5, 2), '1', 'False', 'signed'))
        out.append(('mean|%s|300x517|signed' % dt, dt, (300, 517), '(1,)', 'False', 'signed'))
        out.append(('mean|%s|9x70|neg1tuple' % dt, dt, (9, 70), '(-1,)', 'True', 'mixed'))
        out.append(('mean|%s|3x5x33|mixed' % dt, dt, (3, 5, 33), '2', 'True', 'mixed'))
        out.append(('mean|%s|4x3x40|nokeep' % dt, dt, (4, 3, 40), '-1', 'False', 'signed'))
        out.append(('mean|%s|40x77|inf' % dt, dt, (40, 77), '1', 'True', 'inf'))
        out.append(('mean|%s|40x77|nan' % dt, dt, (40, 77), '-1', 'False', 'nan'))
    return out


def _big(dt):
    """a finite value of the dtype whose doubling overflows"""
    return {'float16': 40000.0, 'bfloat16': 2e38, 'float32': 2e38, 'float64': 1e308}[dt]


def mean_operand(name, dt, shape, values):
    rng = _rng(name)
    n = int(np.prod(shape))
    mag = np.where(rng.random(n) < 0.5, 1e3, 0.1) * rng.uniform(0.5, 1.5, n)
    if values == 'signed':
        mag = mag * np.where(rng.random(n) < 0.5, -1.0, 1.0)
    x = mag.reshape(shape)
    if values in ('inf', 'nan'):
        x = x.reshape(int(np.prod(shape[:-1])), shape[-1]).copy()
        rows = x.shape[0]
        for i in range(0, rows, 3):                 # every third row reaches inf part way along
            j = int(rng.integers(1, shape[-1] - 2))
            x[i, j] = x[i, j + 1] = _big(dt)
        for i in range(1, rows, 5):                 # and some cross back: +inf then -inf gives NaN
            j = int(rng.integers(1, shape[-1] - 3))
            x[i, j] = x[i, j + 1] = _big(dt)
            x[i, j + 2] = -math.inf
        if values == 'nan':
            for i in range(2, rows, 4):
                x[i, int(rng.integers(0, shape[-1]))] = math.nan
        x = x.reshape(shape)
    with np.errstate(over='ignore'):
        return GN.from_f32(x.astype(F32), dt) if dt in SIXTEEN else x.astype(STORE[dt])


def mean_restate(case):
    name, dt, shape, axis, keepdims, values = case
    x = mean_operand(name, dt, shape, values)
    m = mean_rows(x, dt)
    return m.reshape(shape[:-1] + (1,)) if keepdims == 'True' else m


ROW_SHAPES = [(7, 5), (4, 2), (1, 9), (3, 4, 33), (1000, 513)]


def broadcast_cases():
    """(name, op, dtype, lhs shape); rhs is lhs.shape[:-1] + (1,)"""
    return [('%s|rows|%s|%s' % (op, dt, 'x'.join(map(str, s))), op, dt, s)
            for op in BINARY for dt in DTYPES for s in ROW_SHAPES
            if not (op == 'broadcast_div' and dt not in FLOATS)]


def broadcast_operands(name, op, dt, shape):
    n = int(np.prod(shape))
    rn = n // shape[-1]
    a, b = GA.operands(name, op, dt, n)
    # b: rn values (the row operand), its first ones edge values as GA.operands places them
    b = b[:rn].copy()
    if op == 'broadcast_mul' and dt not in FLOATS:
        a = (a % (1 << 15)).astype(STORE[dt])
        b = (b % (1 << 15)).astype(STORE[dt])
    return a.reshape(shape), b.reshape(shape[:-1] + (1,))


def inputs(kind, case):
    if kind == 'square':
        return (square_operand(*case),)
    if kind == 'mean':
        return (mean_operand(case[0], case[1], case[2], case[5]),)
    return broadcast_operands(*case)


def restate(kind, case):
    if kind == 'square':
        return square(inputs(kind, case)[0], case[1])
    if kind == 'mean':
        return mean_restate(case)
    a, b = inputs(kind, case)
    return row_broadcast(case[1], a, b, case[2])


def all_cases():
    return ([('square', c) for c in square_cases()] + [('mean', c) for c in mean_cases()] +
            [('broadcast', c) for c in broadcast_cases()])


def out_dtype(kind, case):
    return case[2] if kind == 'broadcast' else case[1]


# ------------------------------------------------------------------------------- the library
class RefDenseAdaGrad(GN.RefND):
    """the entry points of oracle/_ref/libmxref_dense_adagrad.so (its mxref_nd_* are
    golden_ndarray_ops')"""

    def square(self, a, dt):
        a = np.ascontiguousarray(a, STORE[dt])
        out = np.empty_like(a)
        self._call(self.lib.mxref_da_square, ctypes.c_int(GN.MX_FLAG[dt]), self._p(a), self._p(out),
                   ctypes.c_int64(a.size))
        return out

    def mean(self, x, dt, axis=None, keepdims=None, exclude=None):
        """mean(x, axis=..., keepdims=..., exclude=...) with the attribute strings given (None: not
        passed): the result, in the shape ReduceAxesShapeImpl gives"""
        x = np.ascontiguousarray(x, STORE[dt])
        shape = np.array(x.shape, np.int64)
        out = np.empty(max(1, x.size, int(np.prod(x.shape[:-1]))), STORE[dt])
        ondim = ctypes.c_int()
        oshape = np.zeros(8, np.int64)
        enc = lambda s: None if s is None else str(s).encode()  # noqa: E731
        self._call(self.lib.mxref_da_mean, ctypes.c_int(GN.MX_FLAG[dt]), self._p(x), ctypes.c_int(x.ndim),
                   self._p(shape), enc(axis), enc(keepdims), enc(exclude), self._p(out),
                   ctypes.byref(ondim), self._p(oshape))
        osh = tuple(int(v) for v in oshape[:ondim.value])
        return out[:int(np.prod(osh))].reshape(osh)

    def broadcast(self, op, a, b, dt):
        a, b = np.ascontiguousarray(a, STORE[dt]), np.ascontiguousarray(b, STORE[dt])
        out = np.empty_like(a)
        ls, rs = np.array(a.shape, np.int64), np.array(b.shape, np.int64)
        self._call(self.lib.mxref_da_broadcast, ctypes.c_int(BINARY.index(op)), ctypes.c_int(GN.MX_FLAG[dt]),
                   self._p(a), self._p(b), self._p(out), ctypes.c_int(a.ndim), self._p(ls), self._p(rs))
        return out


_ref = False


def ref():
    """The reference's code, or None when oracle/_ref/libmxref_dense_adagrad.so has not been built."""
    global _ref
    if _ref is False:
        path = os.path.join(HERE, "_ref", "libmxref_dense_adagrad.so")
        _ref = RefDenseAdaGrad(path) if os.path.exists(path) else None
    return _ref


def live(kind, case):
    """the output the reference's code gives for a case; None for bfloat16, which it lacks"""
    r = ref()
    dt = out_dtype(kind, case)
    if dt == 'bfloat16':
        return None
    ins = inputs(kind, case)
    if kind == 'square':
        return r.square(ins[0], dt)
    if kind == 'mean':
        return r.mean(ins[0], dt, axis=case[3], keepdims=case[4])
    return r.broadcast(case[1], ins[0], ins[1], dt)


def gen_dense_adagrad_ops():
    """tests/golden/dense_adagrad_ops.npz: every case's output from the reference's code (from the
    restatement for bfloat16), asserted against the restatement on the way, shapes included. One
    row per case: `names`, `sha256` (32 bytes) and `head` (the first HEAD_BYTES canonical bytes,
    zero padded) of the flattened output."""
    names, shas, heads = [], [], []
    for kind, case in all_cases():
        dt = out_dtype(kind, case)
        want = restate(kind, case)
        got = live(kind, case)
        if got is None:
            got = want
        assert GN.same(got, want, dt), case[0]
        names.append(case[0])
        shas.append(GN.sha256(np.ravel(got), dt))
        heads.append(GN.head_bytes(np.ravel(got), dt))
    d = dict(names=np.array(names), sha256=np.stack(shas), head=np.stack(heads))
    np.savez_compressed(os.path.join(GOLD, "dense_adagrad_ops.npz"), **d)
    return d


if __name__ == "__main__":
    build()
    assert ref() is not None, "build oracle/_ref/libmxref_dense_adagrad.so first"
    d = gen_dense_adagrad_ops()
    print("wrote", len(d['names']), "cases")
