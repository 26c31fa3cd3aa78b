"""TEST INFRASTRUCTURE ONLY -- gradient clipping by global norm (gluon.utils.clip_global_norm) and
the bulk unscale (amp.unscale): numpy float32 restatements, the reference's own functors (`ref()`
over oracle/_ref/libmxref_clip.so, built from oracle/ref_clip_global_norm.cc by
oracle/clip_global_norm.mk), the seeded cases, and the writer of tests/golden/clip_global_norm.npz:

    make -f oracle/clip_global_norm.mk && python oracle/golden_clip_global_norm.py

Three things are restated. `scale_of(norm, max_norm)` is utils.py:150-151 for any norm, nan and
inf included, pinned to `ref().scale` bit for bit. `restate(norm, max_norm, x)` is what the
library's operator leaves in an array given the norm it computed: x * scale, x itself when the
scale is 1, and x itself when the norm is inf or nan (the reference calls that case undefined; the
library leaves the arrays alone). `multi_scale(x, scalar)` is `_mul_scalar`: the scalar string goes
through std::stod and is then rounded once to float32.

The sum of squares itself is not restated bit for bit: the GPU folds it in its own fixed
association. The array-set cases below therefore come in two kinds. `exact` sets hold small
integers, whose squares sum exactly in float32 in every association, so the norm and every output
are comparable bit for bit. Seeded float sets carry the reference's sequential float32 norm for the
1e-5 tolerance check, and their outputs are compared through `restate` on the norm the GPU returned.
"""
import ctypes
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
F = np.float32
MAX_ARRAYS = 200          # kCNMaxArrays (kernels.h)
TILE = 16384 // 4         # kCNTileBytes in float32 elements
PER_THREAD = 16           # 4 loads of 4 elements


def build():
    """oracle/_ref/libmxref_clip.so, where the reference's sources exist"""
    if os.path.isfile("/root/reference/src/operator/mshadow_op.h"):
        import subprocess
        subprocess.run(["make", "-s", "-f", os.path.join(HERE, "clip_global_norm.mk")], check=True)


class RefClip(object):
    """the entry points of oracle/_ref/libmxref_clip.so"""

    def __init__(self, path):
        self.lib = ctypes.CDLL(path)
        self.lib.mxref_clip_sqrt.restype = ctypes.c_float
        self.lib.mxref_clip_sqrt.argtypes = [ctypes.c_float]
        self.lib.mxref_clip_sum_sq.restype = ctypes.c_float

    def sqrt(self, ss):
        return F(self.lib.mxref_clip_sqrt(ctypes.c_float(float(ss))))

    def scale(self, norm, max_norm):
        out = ctypes.c_float()
        err = ctypes.create_string_buffer(1024)
        rc = self.lib.mxref_clip_scale(ctypes.c_float(float(F(norm))), str(max_norm).encode(),
                                       ctypes.byref(out), err, ctypes.c_int(len(err)))
        if rc != 0:
            raise RuntimeError(err.value.decode())
        return np.frombuffer(bytes(out), F)[0]

    def mul(self, x, scale):
        y = np.ascontiguousarray(x, F).copy()
        self.lib.mxref_clip_mul(y.ctypes.data_as(ctypes.c_void_p), ctypes.c_int64(y.size),
                                ctypes.c_float(float(F(scale))))
        return y

    def mul_scalar(self, x, scalar):
        y = np.ascontiguousarray(x, F).copy()
        err = ctypes.create_string_buffer(1024)
        rc = self.lib.mxref_mul_scalar(y.ctypes.data_as(ctypes.c_void_p), ctypes.c_int64(y.size),
                                       str(scalar).encode(), err, ctypes.c_int(len(err)))
        if rc != 0:
            raise RuntimeError(err.value.decode())
        return y

    def sum_sq(self, arrays):
        arrays = [np.ascontiguousarray(a, F).reshape(-1) for a in arrays]
        n = len(arrays)
        ptrs = (ctypes.c_void_p * max(n, 1))(*[a.ctypes.data for a in arrays])
        sizes = (ctypes.c_int64 * max(n, 1))(*[a.size for a in arrays])
        return F(self.lib.mxref_clip_sum_sq(ptrs, sizes, ctypes.c_int(n)))


_ref = False


def ref():
    """The reference's functors, or None when oracle/_ref/libmxref_clip.so has not been built."""
    global _ref
    if _ref is False:
        path = os.path.join(HERE, "_ref", "libmxref_clip.so")
        _ref = RefClip(path) if os.path.exists(path) else None
    return _ref


# -------------------------------------------------------------------------------- restatement
def parse_scalar(s):
    """std::stod, then one rounding to float32. Python's float() is the same correctly rounded
    decimal-to-double conversion, trailing characters aside (none of the cases has any)."""
    with np.errstate(over='ignore'):
        return F(float(str(s)))


def _min_reduce(dst, src):
    """mshadow::red::minimum::Reduce"""
    if not np.isnan(dst) and not (dst <= src):
        return src
    return dst


def scale_of(norm, max_norm):
    """utils.py:150-151 in float32: min(concat(max_norm / (norm + 1e-8), 1))"""
    with np.errstate(all='ignore'):
        s = parse_scalar(max_norm) / (F(norm) + parse_scalar('1e-08'))
    return _min_reduce(_min_reduce(F(np.inf), F(s)), F(1.0))


def restate(norm, max_norm, x):
    """an array after the library's clip, given the total norm the call computed"""
    x = np.asarray(x, F)
    if not np.isfinite(norm):
        return x.copy()
    s = scale_of(norm, max_norm)
    if s == F(1.0):
        return x.copy()
    with np.errstate(all='ignore'):
        return x * s


def multi_scale(x, scalar):
    """`_mul_scalar` on float32: x * float32(stod(scalar))"""
    with np.errstate(all='ignore'):
        return np.asarray(x, F) * parse_scalar(scalar)


def norm_of(arrays):
    """the reference's sequential float32 fold, restated: exact for the `exact` sets"""
    ss = F(0.0)
    for a in arrays:
        for v in np.asarray(a, F).reshape(-1):
            with np.errstate(over='ignore'):
                ss = F(ss + F(v * v))
    return np.sqrt(ss)


# ------------------------------------------------------------------------------------ cases
# max_norm / scalar strings; the fourth lies above the float32 tie 1 + 2^-24 by less than a double
# resolves, so stod gives the tie and the rounding to float goes to even (1.0), where a direct
# float parse gives 1 + 2^-23; dmlc::stof, which the other operators' parameters go through, differs
# from stod-then-round on several of the others
SCALARS = ['1.0', '0.1', '1e-3', '1.0000000596046447753906250000000001', '16777217', '0.30000000000000004',
           '3.4028235e38', '1e39', '1e-45', '7e-46', '2.5', '1e-7', '0.7', '4.9999995', '5', '5.0000005',
           '1.1754944e-38', '65536.0', '1.52587890625e-05', '0.333333343267440796', '123456.789e-3']


def _bits(v):
    return np.asarray(v, F).view(np.uint32)


def scale_cases():
    """(norm bits, max_norm string) around every branch: norm 0, below / equal to / just above
    max_norm, denormal results, inf and nan norms"""
    norms = [0.0, 1e-45, 1e-8, 1e-7, 0.5, 0.99999994, 1.0, 1.0000001, 2.4999998, 2.5, 2.5000002, 4.9999995,
             5.0, 5.0000005, 1000.0, 16777216.0, 1e30, 3.4028235e38, np.inf, np.nan]
    rng = np.random.default_rng(0xC11B)
    norms += list(np.exp(rng.uniform(-20, 20, 40)))
    cases = [(F(n), m) for n in norms for m in SCALARS]
    for m in SCALARS:          # a norm one ulp on either side of max_norm itself
        v = parse_scalar(m)
        if np.isfinite(v) and 0 < v < F(3e38):
            cases += [(np.nextafter(v, F(0)), m), (v, m), (np.nextafter(v, F(np.inf)), m)]
    return cases


def _set(kind, sizes, max_norm, **kw):
    return dict(kind=kind, sizes=list(sizes), max_norm=max_norm, **kw)


def _sets():
    c = {}
    c['ones_3x3_4x4'] = _set('ones', [9, 16], '1.0')                    # test_gluon.py:1131-1139: norm 5
    c['ones_equal'] = _set('ones', [9, 16], '5')
    c['ones_just_below'] = _set('ones', [9, 16], '4.9999995')
    c['ones_not_clipped'] = _set('ones', [9, 16], '5.0000005')
    c['exact_small_clip'] = _set('exact', [1, 3, 4, 5, 15, 16, 17, 63, 64, 65], '0.7')
    c['exact_small_keep'] = _set('exact', [1, 3, 4, 5, 15, 16, 17, 63, 64, 65], '1e39')
    c['exact_tile_edges'] = _set('exact', [TILE - 1, TILE, TILE + 1, 0, TILE + 5, 2 * TILE + 3], '2.5')
    c['exact_empty_members'] = _set('exact', [0, 7, 0, 0, 33, 0], '0.1')
    c['exact_all_zero'] = _set('zeros', [5, 0, 130], '1.0')             # norm 0: scale = min(1e8, 1)
    c['exact_all_empty'] = _set('exact', [0, 0], '1.0')
    c['exact_parse_tie'] = _set('exact', [40, 41], SCALARS[3])
    c['exact_201'] = _set('exact', [int(s) for s in np.random.default_rng(201).integers(0, 40, 201)], '3')
    c['float_small'] = _set('float', [1, 2, 3, 4, 5, 6, 7, 8, 9, 1027], '0.25')
    c['float_denormal_out'] = _set('float', [100, 37], '1e-45', amp=1e3)
    c['float_big_values'] = _set('float', [64, 129], '1.0', amp=1e18)
    c['float_overflowing_norm'] = _set('float', [64, 129], '1.0', amp=3e38)      # ss overflows: norm inf
    c['float_nan_member'] = _set('float', [3, 20], '2.0', poke=(1, 7, np.nan))   # test_gluon.py:1141-1145
    c['float_inf_member'] = _set('float', [3, 20], '2.0', poke=(0, 2, -np.inf))
    return c


SETS = _sets()


def inputs(case, name):
    """the float32 input arrays of an array-set case, seeded by its name"""
    rng = np.random.default_rng(zlib.crc32(('clip|' + name).encode()))
    arrs = []
    for n in case['sizes']:
        if case['kind'] == 'ones':
            a = np.ones(n, F)
        elif case['kind'] == 'zeros':
            a = np.zeros(n, F)
        elif case['kind'] == 'exact':
            a = rng.integers(-8, 9, n).astype(F)
        else:
            with np.errstate(over='ignore'):
                a = (rng.standard_normal(n) * case.get('amp', 1.0)).astype(F)
        arrs.append(a)
    if 'poke' in case:
        k, i, v = case['poke']
        arrs[k][i] = v
    return arrs


# multi_scale: (sizes, scalar string); inputs are seeded floats with edge values mixed in
SCALE_SETS = {('s%02d' % i): dict(sizes=[1, 5, 16, 67, 0], scalar=s) for i, s in enumerate(SCALARS)}
SCALE_SETS['neg'] = dict(sizes=[33], scalar='-0.5')
SCALE_SETS['zero'] = dict(sizes=[33], scalar='0')
SCALE_SETS['tile_edges'] = dict(sizes=[TILE + 3, TILE, TILE - 1], scalar='0.1')
SCALE_SETS['inv_loss_scale'] = dict(sizes=[9, 200, 31], scalar=str(1.0 / 65536))


def scale_inputs(case, name):
    rng = np.random.default_rng(zlib.crc32(('mscale|' + name).encode()))
    edge = np.array([0.0, -0.0, 1e-45, -1e-38, 3.4028235e38, np.inf, -np.inf, np.nan, 1.0, 65504.0], F)
    arrs = []
    for n in case['sizes']:
        a = (rng.standard_normal(n) * np.exp(rng.uniform(-30, 30, n))).astype(F)
        k = min(n, len(edge))
        a[:k] = edge[:k]
        rng.shuffle(a)
        arrs.append(a)
    return arrs


def gen_clip_global_norm():
    """tests/golden/clip_global_norm.npz, every value from the reference's functors; the
    restatements are asserted against them on the way"""
    r = ref()
    d = {}
    sc = scale_cases()
    out = np.array([r.scale(n, m) for n, m in sc], F)
    assert out.tobytes() == np.array([scale_of(n, m) for n, m in sc], F).tobytes()
    d['scale_norm'] = _bits(np.array([n for n, _ in sc], F))
    d['scale_max_norm'] = np.array([m for _, m in sc])
    d['scale_out'] = _bits(out)
    for name, case in SETS.items():
        xs = inputs(case, name)
        with np.errstate(all='ignore'):
            norm = r.sqrt(r.sum_sq(xs))
        assert _bits(norm) == _bits(norm_of(xs)) or (np.isnan(norm) and np.isnan(norm_of(xs))), name
        d[name + '_norm'] = _bits(norm).reshape(1)
        for i, x in enumerate(xs):
            # what the reference leaves: x * scale always; the library's own rule where they part
            want = restate(norm, case['max_norm'], x)
            if np.isfinite(norm):
                assert want.tobytes() == r.mul(x, r.scale(norm, case['max_norm'])).tobytes(), (name, i)
            d['%s_out%d' % (name, i)] = _bits(want)
    for name, case in SCALE_SETS.items():
        for i, x in enumerate(scale_inputs(case, name)):
            want = r.mul_scalar(x, case['scalar'])
            assert want.tobytes() == multi_scale(x, case['scalar']).tobytes(), (name, i)
            d['mscale_%s_out%d' % (name, i)] = _bits(want)
    np.savez_compressed(os.path.join(GOLD, "clip_global_norm.npz"), **d)
    return d


if __name__ == "__main__":
    build()
    assert ref() is not None, "build oracle/_ref/libmxref_clip.so first"
    d = gen_clip_global_norm()
    print("wrote", len(d), "arrays")
