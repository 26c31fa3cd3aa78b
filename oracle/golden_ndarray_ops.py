"""TEST INFRASTRUCTURE ONLY -- the NDArray arithmetic, fill and cast operators that custom updaters
run (`+ - *` with an array or a scalar, `+=`, `*=`, `sqrt`, `a[:] = v`, `astype`): numpy restatements
per dtype, the reference's own code (`ref()` over oracle/_ref/libmxref_ndarith.so, built from
oracle/ref_ndarray_ops.cc by oracle/ndarray_ops.mk), the seeded cases, and the writer of
tests/golden/ndarray_ops.npz:

    make -f oracle/ndarray_ops.mk && python oracle/golden_ndarray_ops.py

Arrays are numpy arrays of their dtype; bfloat16 arrays are their uint16 bit patterns. What is
restated, per dtype:

- float32, float64, int32, int64 compute in their own arithmetic (mshadow_op::plus / minus / mul).
- float16 computes in float32 and rounds once to half (half_t's operators). bfloat16 has no
  counterpart in the reference; it is restated the same way, with one round to nearest even.
- A scalar operator's string goes through std::stod (Python's float() is the same correctly rounded
  conversion) and then DType(alpha): float16 through float32 first (half_t(double)), integers by
  truncation.
- sqrt is taken in float32 for the 16-bit types and float32, in double for float64 and for integers,
  which then truncate (math::sqrt).
- `a[:] = v` is `_full(value=repr(float(v)))`: dmlc::stod, then Fill: zero bytes when the value is
  0 (so -0.0 stores +0.0), else static_cast<DType>(value).
- cast converts directly, except through float32 when either side is 16-bit.

What the reference leaves undefined is not among the cases: signed integer overflow, float-to-int
conversion of NaN, inf or out-of-range values, and integer sqrt of negatives. NaN payloads are not
compared: every comparison maps NaN to one canonical pattern first.

Every case's output is stored as a sha256 of its canonical bytes and its first HEAD_BYTES bytes; the
inputs are regenerated from the case's name by `inputs()`.
"""
import ctypes
import hashlib
import math
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
DTYPES = ('float16', 'bfloat16', 'float32', 'float64', 'int32', 'int64')
FLOATS = ('float16', 'bfloat16', 'float32', 'float64')
SIXTEEN = ('float16', 'bfloat16')
MX_FLAG = {'float32': 0, 'float64': 1, 'float16': 2, 'int32': 4, 'int64': 6}   # mshadow type flags
STORE = {'float16': np.float16, 'bfloat16': np.uint16, 'float32': np.float32, 'float64': np.float64,
         'int32': np.int32, 'int64': np.int64}
# the grid-stride cap of misc_kernels.cu (kNumSMs * 16 CTAs of 256 threads) is 540,672 elements
SIZES = (1, 7, 4099, (1 << 20) + 3)
HEAD_BYTES = 128
F32 = np.float32


def build():
    """oracle/_ref/libmxref_ndarith.so, where the reference's sources exist"""
    if os.path.isfile("/root/reference/src/operator/tensor/init_op.h"):
        import subprocess
        subprocess.run(["make", "-s", "-f", os.path.join(HERE, "ndarray_ops.mk")], check=True)


# ------------------------------------------------------------------------------- bfloat16 bits
def bf16_from_f32(x):
    """float32 -> bfloat16 bits, round to nearest even; NaN -> the canonical 0x7FFF"""
    x = np.ascontiguousarray(x, F32)
    u = x.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(x), np.uint16(0x7FFF), r).astype(np.uint16)


def bf16_to_f32(b):
    return (np.ascontiguousarray(b, np.uint16).astype(np.uint32) << 16).view(F32)


def to_f32(x, dt):
    """the float32 a 16-bit value widens to (exact)"""
    return bf16_to_f32(x) if dt == 'bfloat16' else np.asarray(x).astype(F32)


def from_f32(x, dt):
    """float32 -> a 16-bit dtype, round to nearest even"""
    with np.errstate(over='ignore'):
        return bf16_from_f32(x) if dt == 'bfloat16' else np.asarray(x, F32).astype(np.float16)


def canon(x, dt):
    """the bytes compared: NaN payloads mapped to one pattern"""
    x = np.ascontiguousarray(x, STORE[dt]).copy()
    if dt == 'bfloat16':
        x[(x & 0x7FFF) > 0x7F80] = 0x7FFF
    elif dt in FLOATS:
        x[np.isnan(x)] = np.nan
        bits = x.view({2: np.uint16, 4: np.uint32, 8: np.uint64}[x.itemsize])
        nan_bits = np.array([np.nan], x.dtype).view(bits.dtype)[0]
        bits[np.isnan(x)] = nan_bits
    return x


def same(a, b, dt):
    """bit equality with NaN as NaN"""
    a, b = canon(a, dt), canon(b, dt)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


# ------------------------------------------------------------------------------- restatement
def scalar_of(s, dt):
    """std::stod(s), then DType(alpha), in the array's storage"""
    alpha = float(s)
    with np.errstate(over='ignore'):
        if dt in SIXTEEN:
            return from_f32(np.array([alpha], F32), dt)[0]
        if dt in FLOATS:
            return STORE[dt](alpha)
    return STORE[dt](math.trunc(alpha))


def binary(op, a, b, dt):
    """op: 'plus' | 'minus' | 'mul'"""
    f = {'plus': np.add, 'minus': np.subtract, 'mul': np.multiply}[op]
    with np.errstate(all='ignore'):
        if dt in SIXTEEN:
            return from_f32(f(to_f32(a, dt), to_f32(b, dt)), dt)
        return f(np.asarray(a, STORE[dt]), np.asarray(b, STORE[dt])).astype(STORE[dt])


def binary_scalar(op, a, s, dt):
    """_plus_scalar / _minus_scalar / _mul_scalar with the attribute string s"""
    a = np.asarray(a, STORE[dt])
    return binary(op, a, np.full(a.shape, scalar_of(s, dt), STORE[dt]), dt)


def sqrt(a, dt):
    with np.errstate(invalid='ignore'):
        if dt in SIXTEEN:
            return from_f32(np.sqrt(to_f32(a, dt)), dt)
        if dt in FLOATS:
            return np.sqrt(np.asarray(a, STORE[dt]))
        return np.trunc(np.sqrt(np.asarray(a).astype(np.float64))).astype(STORE[dt])


def dmlc_stod(s):
    """dmlc::stod == ParseFloat<double, true> (dmlc-core strtonum.h:99-254), for the strings Python's
    repr makes: every step in double, the fraction as double(digits) / double(10^k)"""
    s = s.strip()
    sign = -1.0 if s.startswith('-') else 1.0
    s = s.lstrip('+-')
    low = s.lower()
    if low in ('inf', 'infinity'):
        return sign * math.inf
    if low == 'nan':
        return math.nan
    mant, _, exp = low.partition('e')
    ip, _, fp = mant.partition('.')
    value = float(int(ip or '0'))
    if fp:
        fp = fp[:19]
        value += float(int(fp)) / float(10 ** len(fp))
    if exp:
        e = int(exp)
        frac, e = e < 0, abs(e)
        assert e <= 308
        scale = 1.0
        while e >= 8:
            scale *= float(np.float32(1e8))
            e -= 8
        while e > 0:
            scale *= 10.0
            e -= 1
        value = value / scale if frac else value * scale
    return sign * value


def full(value, n, dt):
    """a[:] = value: the array _full leaves"""
    v = dmlc_stod(repr(float(value)))
    if v == 0:
        return np.zeros(n, STORE[dt])
    with np.errstate(over='ignore'):
        if dt in SIXTEEN:
            return from_f32(np.full(n, F32(v), F32), dt)
        if dt in FLOATS:
            return np.full(n, v, STORE[dt])
    return np.full(n, math.trunc(v), STORE[dt])


def cast(x, src, dst):
    """x.astype(dst)"""
    if src == dst:
        return np.array(x, STORE[dst])
    with np.errstate(all='ignore'):
        if src in SIXTEEN or dst in SIXTEEN:
            f = to_f32(x, src) if src in SIXTEEN else np.asarray(x).astype(F32)
            return from_f32(f, dst) if dst in SIXTEEN else f.astype(STORE[dst])
        return np.asarray(x).astype(STORE[dst])


# ------------------------------------------------------------------------------------- cases
def _rng(name):
    return np.random.default_rng(zlib.crc32(('ndops|' + name).encode()))


def _floats(rng, n, dt, lo=-30, hi=30):
    """seeded values spread over many binades, in the dtype's storage"""
    if dt == 'float16':
        lo, hi = max(lo, -26), min(hi, 17)
    v = rng.standard_normal(n) * np.exp2(rng.uniform(lo, hi, n))
    with np.errstate(over='ignore'):
        if dt in SIXTEEN:
            return from_f32(v.astype(F32), dt)
        return v.astype(STORE[dt])


# values that sit where conversions and roundings go wrong, as float64
FLOAT_EDGES = [0.0, -0.0, 1.0, -1.0, 0.1, 1 / 3, 2.5, -2.5, 65504.0, 65519.0, 65520.0, 1e5, -1e5,
               1 + 2 ** -11, 1 + 3 * 2 ** -11, 1 + 2 ** -8, 1 + 3 * 2 ** -8, 1 + 2 ** -24,
               2 ** -24, 2 ** -25, 3 * 2 ** -26, 2 ** -14, 2 ** -149, 2 ** -126, 1e-45, 1e-300,
               2 ** 24 + 1, 2.0 ** 53 + 1, 2.0 ** 53 - 1, 3.4028235e38, 1e300, float(np.finfo(F32).max),
               math.inf, -math.inf, math.nan]


def _float_edges(dt):
    e = np.array(FLOAT_EDGES, np.float64)
    with np.errstate(over='ignore'):
        if dt in SIXTEEN:
            return from_f32(e.astype(F32), dt)
        return e.astype(STORE[dt])


INT_EDGES = {'int32': [0, 1, -1, 7, -7, 16785408, 16777217, 2 ** 24 + 1, 46340, -46341, 2 ** 31 - 1, -2 ** 31],
             'int64': [0, 1, -1, 2 ** 40 + 1, 2 ** 53 + 1, 2 ** 53 - 1, 2 ** 53, 16785408, 4503599761588224,
                       2 ** 62, -2 ** 62, 2 ** 63 - 1, -2 ** 63]}


def operands(name, n, dt, op):
    """(a, b) of size n for `op`; integer values stay where op cannot overflow"""
    rng = _rng(name)
    if dt in FLOATS:
        a, b = _floats(rng, n, dt), _floats(rng, n, dt)
        e = _float_edges(dt)
        k = min(n, len(e))
        a[:k] = e[:k]
        b[:k] = rng.permutation(e)[:k]
        return a, b
    info = np.iinfo(STORE[dt])
    if op == 'sqrt':
        a = rng.integers(0, info.max, n, dtype=STORE[dt], endpoint=True)
        e = np.array([v for v in INT_EDGES[dt] if v >= 0], STORE[dt])
    else:
        lim = (1 << (15 if dt == 'int32' else 31)) if op == 'mul' else info.max // 2
        a = rng.integers(-lim, lim, n, dtype=STORE[dt])
        e = np.array([v for v in INT_EDGES[dt] if abs(v) < lim], STORE[dt])
    b = rng.integers(-(a.max(initial=0) // 4 + 1), a.max(initial=0) // 4 + 1, n, dtype=STORE[dt]) \
        if op != 'mul' else rng.integers(-(1 << 15), 1 << 15, n, dtype=STORE[dt])
    k = min(n, len(e))
    a[:k] = e[:k]
    return a, b


def array_cases():
    """(name, op, dtype, n) for the array operators and sqrt"""
    return [('%s|%s|%d' % (op, dt, n), op, dt, n)
            for op in ('plus', 'minus', 'mul', 'sqrt') for dt in DTYPES for n in SIZES]


def _differing_parses():
    """the strings of tests/golden/scalar_parse.npz whose dmlc::stof and std::stod-to-float differ"""
    d = np.load(os.path.join(GOLD, 'scalar_parse.npz'))
    vals, parsed = d['values'], d['parsed']
    return [repr(float(v)) for v, p in zip(vals, parsed)
            if F32(v).view(np.uint32) != F32(p).view(np.uint32)]


# scalars that cannot be represented in half or bfloat16, that overflow or underflow them, and
# negative and fractional ones, which an integer array truncates
EXTRA_SCALARS = ['0.1', '2.5', '-2.5', '-0.5', '0.9999', '-0.9999', '3.7', '-3.7', '1e-08', '65519.0',
                 '65520.0', '70000.0', '1.00390625', '1.01171875', '1.00048828125', '1.000732421875',
                 '5.960464477539063e-08', '2.9802322387695312e-08', '3.4028235e+38', '1e+39', '1e+300',
                 '0.30000000000000004', '16777217.0', '-1000.25', '123456.789', '-0.0', '0.0', '1.0']


def scalar_cases():
    """(name, op, dtype, scalar string): every scalar on every dtype, integers only where
    DType(alpha) and the result stay in range"""
    out = []
    scalars = _differing_parses() + EXTRA_SCALARS
    for dt in DTYPES:
        for i, s in enumerate(scalars):
            if dt not in FLOATS and abs(float(s)) > 1e6:
                continue
            for op in ('plus', 'minus', 'mul'):
                out.append(('%s_scalar|%s|%03d' % (op, dt, i), op, dt, s))
    return out


def scalar_operand(name, dt):
    """the size-7 array a scalar case runs on"""
    rng = _rng(name)
    if dt in FLOATS:
        a = _floats(rng, 7, dt, -8, 8)
        a[:3] = _float_edges(dt)[[0, 1, 2]]
        return a
    return rng.integers(-1000, 1000, 7, dtype=STORE[dt])


FULL_VALUES = [2 ** 24 + 1, 2 ** 53 - 1, 0.1, -0.0, 0.0, 2.5, -2.5, 1e-8, 65520.0, 1e300, 3.0, 7,
               1.00390625, math.inf, math.nan]


def full_cases():
    """(name, dtype, value, n)"""
    out = []
    for dt in DTYPES:
        for i, v in enumerate(FULL_VALUES):
            if dt not in FLOATS:
                if not math.isfinite(v) or abs(v) >= np.iinfo(STORE[dt]).max:
                    continue
            for n in (1, 7, 4099):
                out.append(('full|%s|%02d|%d' % (dt, i, n), dt, v, n))
    return out


def _defined_cast_values(x, src, dst):
    """x with the values whose cast the reference leaves undefined (or, for integer narrowing,
    implementation-defined) replaced by 0"""
    if dst in FLOATS or src == dst:
        return x
    info = np.iinfo(STORE[dst])
    if src in FLOATS:
        f = to_f32(x, src).astype(np.float64) if src in SIXTEEN else x.astype(np.float64)
        with np.errstate(invalid='ignore'):
            t = np.trunc(f)
            ok = np.isfinite(f) & (t >= info.min) & (t <= info.max)
    else:
        ok = (x >= info.min) & (x <= info.max)
    y = x.copy()
    y[~ok] = 0
    return y


def cast_cases():
    return [('cast|%s|%s|%d' % (src, dst, n), src, dst, n) for src in DTYPES for dst in DTYPES
            for n in SIZES]


def cast_operand(name, src, dst, n):
    rng = _rng(name)
    if src in FLOATS:
        lo, hi = (-30, 40) if dst not in FLOATS else (-160, 160)
        x = _floats(rng, n, src, lo, hi)
        e = _float_edges(src)
        extra = np.array([-2147483648.0, 2147483647.0, 2147483648.0, -2147483904.0, 9.2e18],
                         np.float64)
        with np.errstate(over='ignore'):
            extra = from_f32(extra.astype(F32), src) if src in SIXTEEN else extra.astype(STORE[src])
        e = np.concatenate([e, extra])
    else:
        x = rng.integers(np.iinfo(STORE[src]).min, np.iinfo(STORE[src]).max, n, dtype=STORE[src])
        small = rng.integers(-70000, 70000, n, dtype=STORE[src])
        x = np.where(rng.random(n) < 0.5, x, small).astype(STORE[src])
        e = np.array(INT_EDGES[src] + [2049, 2051, -2049, 65504, 65520, 65535, 257, 259], STORE[src])
    k = min(n, len(e))
    x[:k] = e[:k]
    return _defined_cast_values(x, src, dst)


def inputs(kind, case):
    """the input arrays of a case, regenerated from its name"""
    if kind == 'array':
        name, op, dt, n = case
        return operands(name, n, dt, op)
    if kind == 'scalar':
        return (scalar_operand(case[0], case[2]),)
    if kind == 'cast':
        name, src, dst, n = case
        return (cast_operand(name, src, dst, n),)
    return ()


def restate(kind, case):
    """the output the restatement gives for a case"""
    if kind == 'array':
        name, op, dt, n = case
        a, b = inputs(kind, case)
        return sqrt(a, dt) if op == 'sqrt' else binary(op, a, b, dt)
    if kind == 'scalar':
        name, op, dt, s = case
        return binary_scalar(op, inputs(kind, case)[0], s, dt)
    if kind == 'full':
        name, dt, v, n = case
        return full(v, n, dt)
    name, src, dst, n = case
    return cast(inputs(kind, case)[0], src, dst)


def all_cases():
    return ([('array', c) for c in array_cases()] + [('scalar', c) for c in scalar_cases()] +
            [('full', c) for c in full_cases()] + [('cast', c) for c in cast_cases()])


def out_dtype(kind, case):
    """the dtype of a case's output"""
    return case[1] if kind == 'full' else case[2]


# ------------------------------------------------------------------------------- the library
class RefND(object):
    """the entry points of oracle/_ref/libmxref_ndarith.so (no bfloat16: the reference has none)"""

    def __init__(self, path):
        self.lib = ctypes.CDLL(path)

    def _call(self, fn, *args):
        err = ctypes.create_string_buffer(1024)
        rc = fn(*args, err, ctypes.c_int(len(err)))
        if rc != 0:
            raise RuntimeError(err.value.decode())

    @staticmethod
    def _p(a):
        return a.ctypes.data_as(ctypes.c_void_p)

    def binary(self, op, a, b, dt):
        a, b = np.ascontiguousarray(a, STORE[dt]), np.ascontiguousarray(b, STORE[dt])
        out = np.empty_like(a)
        self._call(self.lib.mxref_nd_binary, ctypes.c_int(['plus', 'minus', 'mul'].index(op)),
                   ctypes.c_int(MX_FLAG[dt]), self._p(a), self._p(b), self._p(out), ctypes.c_int64(a.size))
        return out

    def binary_scalar(self, op, a, s, dt):
        a = np.ascontiguousarray(a, STORE[dt])
        out = np.empty_like(a)
        self._call(self.lib.mxref_nd_scalar, ctypes.c_int(['plus', 'minus', 'mul'].index(op)),
                   ctypes.c_int(MX_FLAG[dt]), self._p(a), str(s).encode(), self._p(out),
                   ctypes.c_int64(a.size))
        return out

    def sqrt(self, a, dt):
        a = np.ascontiguousarray(a, STORE[dt])
        out = np.empty_like(a)
        self._call(self.lib.mxref_nd_sqrt, ctypes.c_int(MX_FLAG[dt]), self._p(a), self._p(out),
                   ctypes.c_int64(a.size))
        return out

    def full(self, value, n, dt):
        """(the parsed double, the array) of _full(value=repr(float(value)))"""
        out = np.empty(n, STORE[dt])
        parsed = ctypes.c_double()
        self._call(self.lib.mxref_nd_full, ctypes.c_int(MX_FLAG[dt]), repr(float(value)).encode(),
                   ctypes.byref(parsed), self._p(out), ctypes.c_int64(n))
        return parsed.value, out

    def cast(self, x, src, dst):
        x = np.ascontiguousarray(x, STORE[src])
        out = np.empty(x.shape, STORE[dst])
        self._call(self.lib.mxref_nd_cast, ctypes.c_int(MX_FLAG[dst]), self._p(x), ctypes.c_int(MX_FLAG[src]),
                   self._p(out), ctypes.c_int64(x.size))
        return out


_ref = False


def ref():
    """The reference's code, or None when oracle/_ref/libmxref_ndarith.so has not been built."""
    global _ref
    if _ref is False:
        path = os.path.join(HERE, "_ref", "libmxref_ndarith.so")
        _ref = RefND(path) if os.path.exists(path) else None
    return _ref


def live(kind, case):
    """the output the reference's code gives for a case; None for bfloat16, which it lacks"""
    r = ref()
    if kind == 'array':
        name, op, dt, n = case
        if dt == 'bfloat16':
            return None
        a, b = inputs(kind, case)
        return r.sqrt(a, dt) if op == 'sqrt' else r.binary(op, a, b, dt)
    if kind == 'scalar':
        name, op, dt, s = case
        return None if dt == 'bfloat16' else r.binary_scalar(op, inputs(kind, case)[0], s, dt)
    if kind == 'full':
        name, dt, v, n = case
        return None if dt == 'bfloat16' else r.full(v, n, dt)[1]
    name, src, dst, n = case
    if 'bfloat16' in (src, dst):
        return None
    return r.cast(inputs(kind, case)[0], src, dst)


def gen_ndarray_ops():
    """tests/golden/ndarray_ops.npz: every case's output from the reference's code (from the
    restatement for bfloat16), asserted against the restatement on the way. One row per case:
    `names`, `sha256` (32 bytes) and `head` (the first HEAD_BYTES canonical bytes, zero padded)."""
    names, shas, heads = [], [], []
    for kind, case in all_cases():
        dt = out_dtype(kind, case)
        want = restate(kind, case)
        got = live(kind, case)
        if got is None:
            got = want
        assert same(got, want, dt), case
        names.append(case[0])
        shas.append(sha256(got, dt))
        heads.append(head_bytes(got, dt))
    d = dict(names=np.array(names), sha256=np.stack(shas), head=np.stack(heads))
    np.savez_compressed(os.path.join(GOLD, "ndarray_ops.npz"), **d)
    return d


def head_bytes(x, dt):
    """the first HEAD_BYTES canonical bytes of an output, zero padded"""
    out = np.zeros(HEAD_BYTES, np.uint8)
    h = canon(x, dt).view(np.uint8)[:HEAD_BYTES]
    out[:h.size] = h
    return out


def sha256(x, dt):
    """the digest the fixture stores for an output"""
    return np.frombuffer(hashlib.sha256(canon(x, dt).tobytes()).digest(), np.uint8)


if __name__ == "__main__":
    build()
    assert ref() is not None, "build oracle/_ref/libmxref_ndarith.so first"
    d = gen_ndarray_ops()
    print("wrote", len(d['names']), "cases")
