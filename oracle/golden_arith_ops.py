"""TEST INFRASTRUCTURE ONLY -- the arithmetic operators that the reference's Adamax, Nadam and AdaDelta
optimizers compose (broadcast_add / _sub / _mul / _div / _maximum on operands of one shape,
_div_scalar, abs, clip): numpy restatements per dtype, the reference's own code (`ref()` over
oracle/_ref/libmxref_arith.so, built from oracle/ref_arith_ops.cc by oracle/arith_ops.mk), the seeded
cases, and the writer of tests/golden/arith_ops.npz:

    make -f oracle/arith_ops.mk && python oracle/golden_arith_ops.py

Arrays, dtypes, the fixture format (a sha256 and the first bytes of each output, NaN payloads
canonical) and the helpers are those of oracle/golden_ndarray_ops.py. What is restated, per dtype:

- broadcast_add / _sub / _mul are golden_ndarray_ops.binary (mshadow_op::plus, minus, mul).
- broadcast_div and _div_scalar divide in the dtype's own arithmetic, float16 and bfloat16 in
  float32 with one rounding. The scalar goes through std::stod and DType(alpha). Integer division is
  refused by the library, so it has no cases.
- broadcast_maximum is `a if isnan(a) else (a if a > b else b)`, compared in float32 for the 16-bit
  types: a NaN in `b` and -0 against +0 give `b`.
- abs is fabsf / fabs for the float types; an integer goes through double and truncates back.
- clip parses a_min and a_max with dmlc::stof (ClipParam's real_t fields), then compares each
  element with the float bound in C++'s arithmetic: a 16-bit value widens to float, a double
  compares with the widened bound, an integer converts to float. A bound taken converts to the
  dtype (float16 / bfloat16 rounding from float, integers truncating). NaN passes through.

What the reference leaves undefined is not among the cases: abs of an integer whose magnitude does
not fit its type after the trip through double, and an integer clip bound outside the integer range.
"""
import ctypes
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import golden_ndarray_ops as GN  # noqa: E402
import kvoracle as K  # noqa: E402

GOLD = GN.GOLD
DTYPES, FLOATS, SIXTEEN, STORE, F32 = GN.DTYPES, GN.FLOATS, GN.SIXTEEN, GN.STORE, GN.F32
# the operator each array case runs, and the operand ranges it takes from golden_ndarray_ops
ARRAY_OPS = {'broadcast_add': 'plus', 'broadcast_sub': 'minus', 'broadcast_mul': 'mul',
             'broadcast_div': 'plus', 'broadcast_maximum': 'plus', 'abs': 'plus'}
DIVIDES = ('broadcast_div', '_div_scalar')
# (a_min, a_max) as Python's repr writes them
CLIP_BOUNDS = [('-0.5', '0.5'), ('-0.0', '0.0'), ('0.0', '0.0'), ('-1.0', '1.0'),
               ('0.1', '0.30000000000000004'), ('-3.7', '2.5'), ('-1e+38', '1e+38'), ('-inf', 'inf'),
               ('1.0', '1.0'), ('-16777216.0', '16777216.0'), ('65504.0', '65520.0'),
               ('1.00048828125', '1.000732421875'), ('2.0', '-2.0')]


def build():
    """oracle/_ref/libmxref_arith.so, where the reference's sources exist"""
    if os.path.isfile("/root/reference/src/operator/tensor/matrix_op-inl.h"):
        import subprocess
        subprocess.run(["make", "-s", "-f", os.path.join(HERE, "arith_ops.mk")], check=True)


# ------------------------------------------------------------------------------- restatement
def div(a, b, dt):
    with np.errstate(all='ignore'):
        if dt in SIXTEEN:
            return GN.from_f32(GN.to_f32(a, dt) / GN.to_f32(b, dt), dt)
        assert dt in FLOATS
        return (np.asarray(a, STORE[dt]) / np.asarray(b, STORE[dt])).astype(STORE[dt])


def maximum(a, b, dt):
    a, b = np.asarray(a, STORE[dt]), np.asarray(b, STORE[dt])
    x, y = (GN.to_f32(a, dt), GN.to_f32(b, dt)) if dt in SIXTEEN else (a, b)
    with np.errstate(invalid='ignore'):
        pick_a = (x != x) | (x > y)
    return np.where(pick_a, a, b).astype(STORE[dt])


def absolute(a, dt):
    a = np.asarray(a, STORE[dt])
    if dt == 'bfloat16':
        return (a & np.uint16(0x7FFF)).astype(np.uint16)
    if dt in FLOATS:
        return np.abs(a)
    return np.trunc(np.abs(a.astype(np.float64))).astype(STORE[dt])


def clip_bounds(a_min, a_max):
    """(a_min, a_max) as ClipParam parses them: dmlc::stof"""
    return F32(K.dmlc_stof(a_min)), F32(K.dmlc_stof(a_max))


def clip(a, a_min, a_max, dt):
    lo, hi = clip_bounds(a_min, a_max)
    a = np.asarray(a, STORE[dt])
    with np.errstate(invalid='ignore', over='ignore'):
        if dt in SIXTEEN:
            x = GN.to_f32(a, dt)
            r = np.where(x > hi, hi, np.where(x < lo, lo, x)).astype(F32)
            return GN.from_f32(r, dt)
        if dt in FLOATS:
            lo_t, hi_t = STORE[dt](lo), STORE[dt](hi)
            return np.where(a > hi_t, hi_t, np.where(a < lo_t, lo_t, a)).astype(STORE[dt])
        x = a.astype(F32)
        return np.where(x > hi, STORE[dt](math.trunc(float(hi))) if math.isfinite(hi) else 0,
                        np.where(x < lo, STORE[dt](math.trunc(float(lo))) if math.isfinite(lo) else 0,
                                 a)).astype(STORE[dt])


def restate_array(op, a, b, dt):
    if op == 'broadcast_div':
        return div(a, b, dt)
    if op == 'broadcast_maximum':
        return maximum(a, b, dt)
    if op == 'abs':
        return absolute(a, dt)
    return GN.binary(ARRAY_OPS[op], a, b, dt)


# ------------------------------------------------------------------------------------- cases
def _rng(name):
    return GN._rng('arith|' + name)


def array_cases():
    """(name, op, dtype, n)"""
    return [('%s|%s|%d' % (op, dt, n), op, dt, n) for op in ARRAY_OPS for dt in DTYPES
            for n in GN.SIZES if not (op in DIVIDES and dt not in FLOATS)]


# (a, b) pairs that pin maximum's choice: signed zeros, NaN on either side, equal values
MAX_PAIRS = [(-0.0, 0.0), (0.0, -0.0), (math.nan, 1.0), (1.0, math.nan), (math.nan, -math.inf),
             (2.5, 2.5), (-math.inf, math.inf), (math.inf, math.nan)]


def operands(name, op, dt, n):
    a, b = GN.operands('arith|' + name, n, dt, ARRAY_OPS[op])
    if op == 'broadcast_maximum' and dt in FLOATS:
        k = min(n, len(MAX_PAIRS))
        pa, pb = (np.array([p[i] for p in MAX_PAIRS[:k]], np.float64) for i in (0, 1))
        cv = (lambda v: GN.from_f32(v.astype(F32), dt)) if dt in SIXTEEN else (lambda v: v.astype(STORE[dt]))
        a[-k:], b[-k:] = cv(pa), cv(pb)
    if op == 'broadcast_maximum' and dt not in FLOATS and n > 1:
        b[-1] = a[-1]
    return a, b


def scalar_cases():
    """(name, dtype, scalar string) of _div_scalar, floating dtypes only"""
    scalars = GN._differing_parses() + GN.EXTRA_SCALARS + ['inf', '-inf']
    return [('_div_scalar|%s|%03d' % (dt, i), dt, s) for dt in FLOATS for i, s in enumerate(scalars)]


def clip_cases():
    """(name, dtype, a_min, a_max, n): every bound pair at size 37, the first at every size"""
    out = []
    for dt in DTYPES:
        for i, (lo, hi) in enumerate(CLIP_BOUNDS):
            if dt not in FLOATS and not all(math.isfinite(float(v)) and abs(float(v)) < 2 ** 31
                                            for v in (lo, hi)):
                continue
            for n in ((37,) + GN.SIZES if i == 0 else (37,)):
                out.append(('clip|%s|%02d|%d' % (dt, i, n), dt, lo, hi, n))
    return out


def clip_operand(name, dt, lo, hi, n):
    """values inside and outside the bounds, the bounds themselves and their neighbours, NaN, inf"""
    rng = _rng(name)
    lo_f, hi_f = (float(v) for v in clip_bounds(lo, hi))
    if dt in FLOATS:
        x = GN._floats(rng, n, dt, -4, 4)
        edges = [lo_f, hi_f, -0.0, 0.0, math.nan, math.inf, -math.inf, 65504.0, 1.0, -1.0,
                 float(np.nextafter(F32(lo_f), F32(-math.inf))), float(np.nextafter(F32(hi_f), F32(math.inf))),
                 16777217.0, 1 + 2 ** -11]
        e = np.array(edges, np.float64)
        with np.errstate(over='ignore', invalid='ignore'):
            e = GN.from_f32(e.astype(F32), dt) if dt in SIXTEEN else e.astype(STORE[dt])
    else:
        x = rng.integers(-40000000, 40000000, n, dtype=STORE[dt])
        small = rng.integers(-5, 5, n, dtype=STORE[dt])
        x = np.where(rng.random(n) < 0.5, x, small).astype(STORE[dt])
        e = np.array([math.trunc(lo_f), math.trunc(hi_f), 0, 1, -1, 16777217, -16777217, 16777216,
                      2 ** 31 - 1, -2 ** 31], STORE[dt])
    k = min(n, len(e))
    x[:k] = e[:k]
    return x


def inputs(kind, case):
    if kind == 'array':
        name, op, dt, n = case
        a, b = operands(name, op, dt, n)
        return (a,) if op == 'abs' else (a, b)
    if kind == 'scalar':
        return (GN.scalar_operand('arith|' + case[0], case[1]),)
    name, dt, lo, hi, n = case
    return (clip_operand(name, dt, lo, hi, n),)


def restate(kind, case):
    ins = inputs(kind, case)
    if kind == 'array':
        name, op, dt, n = case
        return restate_array(op, ins[0], ins[-1], dt)
    if kind == 'scalar':
        name, dt, s = case
        a = ins[0]
        return div(a, np.full(a.shape, GN.scalar_of(s, dt), STORE[dt]), dt)
    name, dt, lo, hi, n = case
    return clip(ins[0], lo, hi, dt)


def all_cases():
    return ([('array', c) for c in array_cases()] + [('scalar', c) for c in scalar_cases()] +
            [('clip', c) for c in clip_cases()])


def out_dtype(kind, case):
    return case[1] if kind in ('scalar', 'clip') else case[2]


# ------------------------------------------------------------------------------- the library
class RefArith(GN.RefND):
    """the entry points of oracle/_ref/libmxref_arith.so (its mxref_nd_* are golden_ndarray_ops')"""

    def div_max(self, op, a, b, dt):
        a, b = np.ascontiguousarray(a, STORE[dt]), np.ascontiguousarray(b, STORE[dt])
        out = np.empty_like(a)
        self._call(self.lib.mxref_ar_binary, ctypes.c_int(['broadcast_div', 'broadcast_maximum'].index(op)),
                   ctypes.c_int(GN.MX_FLAG[dt]), self._p(a), self._p(b), self._p(out), ctypes.c_int64(a.size))
        return out

    def div_scalar(self, a, s, dt):
        """(the parsed double, the array) of _div_scalar(scalar=s)"""
        a = np.ascontiguousarray(a, STORE[dt])
        out = np.empty_like(a)
        parsed = ctypes.c_double()
        self._call(self.lib.mxref_ar_div_scalar, ctypes.c_int(GN.MX_FLAG[dt]), self._p(a), str(s).encode(),
                   ctypes.byref(parsed), self._p(out), ctypes.c_int64(a.size))
        return parsed.value, out

    def abs(self, a, dt):
        a = np.ascontiguousarray(a, STORE[dt])
        out = np.empty_like(a)
        self._call(self.lib.mxref_ar_abs, ctypes.c_int(GN.MX_FLAG[dt]), self._p(a), self._p(out),
                   ctypes.c_int64(a.size))
        return out

    def clip(self, a, lo, hi, dt):
        """(the parsed (a_min, a_max), the array) of clip(a_min=lo, a_max=hi)"""
        a = np.ascontiguousarray(a, STORE[dt])
        out = np.empty_like(a)
        parsed = np.zeros(2, F32)
        self._call(self.lib.mxref_ar_clip, ctypes.c_int(GN.MX_FLAG[dt]), self._p(a), str(lo).encode(),
                   str(hi).encode(), self._p(parsed), self._p(out), ctypes.c_int64(a.size))
        return parsed, out

    def array_op(self, op, a, b, dt):
        if op in ('broadcast_div', 'broadcast_maximum'):
            return self.div_max(op, a, b, dt)
        if op == 'abs':
            return self.abs(a, dt)
        return self.binary(ARRAY_OPS[op], a, b, dt)


_ref = False


def ref():
    """The reference's code, or None when oracle/_ref/libmxref_arith.so has not been built."""
    global _ref
    if _ref is False:
        path = os.path.join(HERE, "_ref", "libmxref_arith.so")
        _ref = RefArith(path) if os.path.exists(path) else None
    return _ref


def live(kind, case):
    """the output the reference's code gives for a case; None for bfloat16, which it lacks"""
    r = ref()
    dt = out_dtype(kind, case)
    if dt == 'bfloat16':
        return None
    ins = inputs(kind, case)
    if kind == 'array':
        return r.array_op(case[1], ins[0], ins[-1], dt)
    if kind == 'scalar':
        return r.div_scalar(ins[0], case[2], dt)[1]
    return r.clip(ins[0], case[2], case[3], dt)[1]


def gen_arith_ops():
    """tests/golden/arith_ops.npz: every case's output from the reference's code (from the
    restatement for bfloat16), asserted against the restatement on the way. One row per case:
    `names`, `sha256` (32 bytes) and `head` (the first HEAD_BYTES canonical bytes, zero padded)."""
    names, shas, heads = [], [], []
    for kind, case in all_cases():
        dt = out_dtype(kind, case)
        want = restate(kind, case)
        got = live(kind, case)
        if got is None:
            got = want
        assert GN.same(got, want, dt), case
        names.append(case[0])
        shas.append(GN.sha256(got, dt))
        heads.append(GN.head_bytes(got, dt))
    d = dict(names=np.array(names), sha256=np.stack(shas), head=np.stack(heads))
    np.savez_compressed(os.path.join(GOLD, "arith_ops.npz"), **d)
    return d


if __name__ == "__main__":
    build()
    assert ref() is not None, "build oracle/_ref/libmxref_arith.so first"
    d = gen_arith_ops()
    print("wrote", len(d['names']), "cases")
