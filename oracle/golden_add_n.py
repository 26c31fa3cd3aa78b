"""TEST INFRASTRUCTURE ONLY -- add_n / ElementWiseSum: a numpy restatement (`restate`), the
reference's own arithmetic (`ref_dense` over oracle/_ref/libmxref_add_n.so, built from
oracle/ref_add_n.cc by oracle/add_n.mk; `ref_rsp` over libmxref.so's ElementwiseSumRsp), the
seeded `CASES`, and the writer of tests/golden/add_n.npz:

    make -f oracle/add_n.mk && python oracle/golden_add_n.py

A case is a list of inputs of one dtype and shape, each dense or row_sparse (float32). Inputs are
regenerated from the case's name; the fixture holds the outputs only, as raw bits (uint16 for float16
and bfloat16, uint32 for float32, uint64 for float64, the integers as themselves). A dense out is
stored under the case's name, a row_sparse out under name + '_idx' and name + '_val'. The reference
has no bfloat16: those cases are pinned to the restatement only (one float add and one rounding to
nearest even per +).

The arithmetic, per ElementWiseSumComputeExCPU's dispatch (tensor/elemwise_sum.cc:101-125):
  all dense               2-4 inputs a0 + (a1 + (a2 + a3)), else out = a0, out = out + a_i; every +
                          in the dtype (half_t through float, integers wrap)
  all row_sparse          the sorted union of ids, each row +0.0f then the inputs that hold it in order
  > 4 inputs, some dense  out = a0 (zeros when a0 is row_sparse), then dense inputs add every element
                          and row_sparse inputs their stored rows only
  any other mix           row_sparse inputs densified (zeros, then their rows), then the dense rule
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
DTYPES = ['float16', 'bfloat16', 'float32', 'float64', 'uint8', 'int8', 'int32', 'int64']
FLOATS = ['float16', 'bfloat16', 'float32', 'float64']
RAW = {'float16': np.uint16, 'bfloat16': np.uint16, 'float32': np.uint32, 'float64': np.uint64,
       'uint8': np.uint8, 'int8': np.int8, 'int32': np.int32, 'int64': np.int64}
MSHADOW_FLAG = {'float32': 0, 'float64': 1, 'float16': 2, 'uint8': 3, 'int32': 4, 'int8': 5, 'int64': 6}
COUNTS = [1, 2, 3, 4, 5, 9, 200, 201]
SIZE = 533                  # 16-byte vectors and a scalar tail in every dtype
RSP_SHAPE = (13, 41)        # row_sparse and mixed cases


def build():
    """oracle/_ref/libmxref_add_n.so, where the reference's sources exist"""
    if os.path.isfile("/root/reference/src/operator/tensor/elemwise_sum.h"):
        import subprocess
        subprocess.run(["make", "-s", "-f", os.path.join(HERE, "add_n.mk")], check=True)


# --------------------------------------------------------------------------------- arithmetic
def widen_bf16(bits):
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(F)


def round_bf16(x):
    """float32 -> bfloat16 bits, to nearest even (__float2bfloat16_rn); NaN stays NaN"""
    b = np.asarray(x, F).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)
    nan = np.isnan(np.asarray(x, F))
    r[nan] = 0x7FC0
    return r


def values(bits, dtype):
    """raw bits -> numpy values of the dtype (bfloat16: its float32 widening)"""
    bits = np.asarray(bits, RAW[dtype])
    if dtype == 'bfloat16':
        return widen_bf16(bits)
    return bits.view({'float16': np.float16, 'float32': F, 'float64': np.float64}.get(dtype, RAW[dtype]))


def add(a, b, dtype):
    """one + in the dtype on raw bits"""
    with np.errstate(over='ignore', invalid='ignore'):
        if dtype == 'float16':
            r = (a.view(np.float16).astype(F) + b.view(np.float16).astype(F)).astype(np.float16)
            return r.view(np.uint16)
        if dtype == 'bfloat16':
            return round_bf16(widen_bf16(a) + widen_bf16(b))
        if dtype == 'float32':
            return (a.view(F) + b.view(F)).view(np.uint32)
        if dtype == 'float64':
            return (a.view(np.float64) + b.view(np.float64)).view(np.uint64)
        return (a + b).astype(RAW[dtype])   # same-dtype integer arrays wrap


def fold(arrays, dtype):
    """ElementWiseSumCompute_ on raw-bit arrays"""
    n = len(arrays)
    if 2 <= n <= 4:
        acc = arrays[-1]
        for a in reversed(arrays[:-1]):
            acc = add(a, acc, dtype)
        return acc.copy()
    acc = arrays[0].copy()
    for a in arrays[1:]:
        acc = add(acc, a, dtype)
    return acc


def densify(inp, shape, fill=0.0):
    """a row_sparse input (ids, rows) as float32 bits, absent rows `fill`"""
    ids, rows = inp
    d = np.full(shape, fill, F)
    d[ids] = rows
    return d.view(np.uint32)


def restate(case, inputs):
    """the sum of a case: raw bits of a dense out, or (ids, rows) of a row_sparse out"""
    dtype, st = case['dtype'], case['stypes']
    if all(s == 'row_sparse' for s in st):
        shape = case['shape']
        ids = np.unique(np.concatenate([i for i, _ in inputs] + [np.zeros(0, np.int64)])).astype(np.int64)
        out = np.zeros((len(ids),) + tuple(shape[1:]), F)
        pos = {int(r): k for k, r in enumerate(ids)}
        for i, rows in inputs:
            for r, row in zip(i, rows):
                out[pos[int(r)]] = out[pos[int(r)]] + row
        return ids, out
    if all(s == 'default' for s in st):
        return fold(inputs, dtype)
    shape = case['shape']
    if len(st) > 4:   # ElementwiseSumContainsDnsImpl
        out = inputs[0].view(F).copy() if st[0] == 'default' else np.zeros(shape, F)
        with np.errstate(over='ignore', invalid='ignore'):
            for k, (s, a) in enumerate(zip(st, inputs)):
                if k == 0 and s == 'default':
                    continue
                if s == 'default':
                    out = out + a.view(F)
                else:
                    ids, rows = a
                    out[ids] = out[ids] + rows
        return out.view(np.uint32)
    return fold([a if s == 'default' else densify(a, shape) for s, a in zip(st, inputs)], 'float32')


# ------------------------------------------------------------------------------ the reference
class RefAddN(object):
    """mxref_add_n over oracle/_ref/libmxref_add_n.so: every form with at least one dense input"""

    def __init__(self, path):
        self.lib = ctypes.CDLL(path)

    def __call__(self, case, inputs):
        dtype, st = case['dtype'], case['stypes']
        shape = case['shape']
        rows = shape[0] if len(shape) > 1 else 1
        row_len = int(np.prod(shape[1:])) if len(shape) > 1 else int(np.prod(shape))
        n = len(inputs)
        keep, vals, ids, nnr = [], [], [], []
        for s, a in zip(st, inputs):
            if s == 'default':
                v, i, k = np.ascontiguousarray(a), np.zeros(1, np.int64), rows
            else:
                i = np.ascontiguousarray(a[0], np.int64) if len(a[0]) else np.zeros(1, np.int64)
                v = np.ascontiguousarray(a[1], F) if len(a[0]) else np.zeros(1, F)
                k = len(a[0])
            keep += [v, i]
            vals.append(v.ctypes.data)
            ids.append(i.ctypes.data)
            nnr.append(k)
        out = np.zeros(rows * row_len, RAW[dtype])
        err = ctypes.create_string_buffer(4096)
        rc = self.lib.mxref_add_n(
            ctypes.c_int(n), (ctypes.c_int * n)(*[0 if s == 'default' else 1 for s in st]),
            (ctypes.c_void_p * n)(*vals), (ctypes.c_void_p * n)(*ids), (ctypes.c_int64 * n)(*nnr),
            ctypes.c_int(MSHADOW_FLAG[dtype]), ctypes.c_int64(rows), ctypes.c_int64(row_len),
            out.ctypes.data_as(ctypes.c_void_p), err, ctypes.c_int(len(err)))
        if rc != 0:
            raise RuntimeError(err.value.decode())
        return out.reshape(shape)


_ref = False


def ref_dense():
    """The reference's dense-out add_n, or None when oracle/_ref/libmxref_add_n.so has not been built."""
    global _ref
    if _ref is False:
        path = os.path.join(HERE, "_ref", "libmxref_add_n.so")
        _ref = RefAddN(path) if os.path.exists(path) else None
    return _ref


def ref_rsp():
    """The reference's ElementwiseSumRsp (libmxref.so), or None when it has not been built."""
    import kvoracle
    r = kvoracle.ref()
    return r if r is not None and r.has_sparse() else None


def ref(case, inputs):
    """the reference's output of a case (dense bits, or (ids, rows))"""
    if all(s == 'row_sparse' for s in case['stypes']):
        held = [(i, r) for i, r in inputs if len(i)]
        if not held:
            return np.zeros(0, np.int64), np.zeros((0,) + tuple(case['shape'][1:]), F)
        idx, val = ref_rsp().rsp_reduce([i for i, _ in held], [r for _, r in held])
        return idx, val.reshape((len(idx),) + tuple(case['shape'][1:]))
    return ref_dense()(case, inputs)


# -------------------------------------------------------------------------------------- cases
SPECIAL = {
    'float16': [0x0000, 0x8000, 0x7C00, 0xFC00, 0x7E00, 0x7BFF, 0xFBFF, 0x0001],
    'bfloat16': [0x0000, 0x8000, 0x7F80, 0xFF80, 0x7FC0, 0x7F7F, 0xFF7F, 0x0001],
    'float32': [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7F7FFFFF, 0xFF7FFFFF, 0x00000001],
    'float64': [0, 0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000,
                0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF, 1],
}


def _dense(rng, dtype, size):
    """random raw values: floats of mixed magnitudes (large ones overflow in the 16-bit types), ~6 %
    signed zeros, infinities, NaN and extremes; integers over their whole range (sums wrap)"""
    if dtype in ('uint8', 'int8', 'int32', 'int64'):
        info = np.iinfo(RAW[dtype])
        return rng.integers(info.min, info.max, size, dtype=RAW[dtype], endpoint=True)
    scale = rng.choice([1e-3, 1.0, 3e2, 3e4], size)
    x = rng.standard_normal(size) * scale
    if dtype == 'float16':
        raw = x.astype(np.float16).view(np.uint16)
    elif dtype == 'bfloat16':
        raw = round_bf16(x.astype(F))
    elif dtype == 'float32':
        raw = (x * rng.choice([1.0, 1e30], size)).astype(F).view(np.uint32)
    else:
        raw = (x * rng.choice([1.0, 1e300], size)).view(np.uint64)
    k = size // 16
    at = rng.choice(size, k, replace=False)
    raw[at] = np.asarray(SPECIAL[dtype], RAW[dtype])[rng.integers(0, len(SPECIAL[dtype]), k)]
    return raw


def _rsp(rng, shape, ids, neg_zero=True):
    """(ids, rows) of a float32 row_sparse input; some values -0.0"""
    ids = sorted(set(ids))
    rows = rng.standard_normal((len(ids),) + tuple(shape[1:])).astype(F)
    if neg_zero and len(ids):
        rows.reshape(-1)[rng.choice(rows.size, max(1, rows.size // 20), replace=False)] = -0.0
    return np.asarray(ids, np.int64), rows


def _cases():
    c = {}
    for dt in DTYPES:
        for n in COUNTS:
            c['%s_n%d' % (dt, n)] = dict(dtype=dt, stypes=['default'] * n, shape=(SIZE,))
    for dt in FLOATS:   # every element of a case: -0.0 + -0.0 keeps the sign, -0.0 + +0.0 does not
        for n in (2, 5):
            c['%s_zeros_n%d' % (dt, n)] = dict(dtype=dt, stypes=['default'] * n, shape=(SIZE,), zeros=True)
    R = 'row_sparse'
    D = 'default'
    rs = dict(dtype='float32', shape=RSP_SHAPE)
    c['rsp_empty'] = dict(rs, stypes=[R] * 3, rows=[[], [], []])
    c['rsp_one'] = dict(rs, stypes=[R], rows=[[1, 4, 12]])
    c['rsp_disjoint'] = dict(rs, stypes=[R] * 3, rows=[[0, 5], [2, 7, 11], [12]])
    c['rsp_overlap'] = dict(rs, stypes=[R] * 4, rows=[[1, 3, 5, 7], [3, 4, 5], [], [0, 5, 7, 12]])
    c['rsp_every_row'] = dict(rs, stypes=[R] * 2, rows=[list(range(13)), list(range(13))])
    c['rsp_some_every_row'] = dict(rs, stypes=[R] * 3, rows=[[2, 9], list(range(13)), [9]])
    c['rsp_n20'] = dict(rs, stypes=[R] * 20, rows=[[(3 * k + j) % 13 for j in range(k % 4)] for k in range(20)])
    c['rsp_n40_all'] = dict(rs, stypes=[R] * 40, rows=[list(range(13))] * 40)
    # > 4 inputs with a dense one; row 6 is absent from every row_sparse input and -0.0 in every
    # dense one at column 3, so the reference leaves it -0.0 there
    c['mix_gt4_dense_first'] = dict(rs, stypes=[D, R, D, R, R], rows=[None, [0, 2], None, [2, 12], []], negzero=(6, 3))
    c['mix_gt4_rsp_first'] = dict(rs, stypes=[R, D, D, R, D, R], rows=[[1, 5], None, None, [], None, [5, 7]],
                                  negzero=(6, 3))
    c['mix_gt4_one_dense'] = dict(rs, stypes=[R, R, R, D, R], rows=[[0], [12], [], None, [0, 12]], negzero=(6, 3))
    c['mix_gt4_n9'] = dict(rs, stypes=[D, R] * 4 + [D], rows=[r for k in range(4) for r in (None, [k, k + 3])] + [None],
                           negzero=(11, 40))
    c['mix_gt4_n201'] = dict(rs, stypes=[D, R, R] * 67,
                             rows=[r for k in range(67) for r in (None, [k % 13], [(5 * k) % 13])], negzero=None)
    # <= 4 inputs, mixed: the storage fallback densifies, so absent rows add +0.0
    c['mix_le4_dr'] = dict(rs, stypes=[D, R], rows=[None, [0, 3]], negzero=(6, 3))
    c['mix_le4_rd'] = dict(rs, stypes=[R, D], rows=[[4], None], negzero=(6, 3))
    c['mix_le4_drd'] = dict(rs, stypes=[D, R, D], rows=[None, []], negzero=(6, 3))
    c['mix_le4_rrdr'] = dict(rs, stypes=[R, R, D, R], rows=[[0, 1], [1], None, [12]], negzero=(6, 3))
    return c


CASES = _cases()


def inputs(case, name):
    """the inputs of a case, seeded by its name: raw-bit arrays (dense) or (ids, float32 rows)"""
    rng = np.random.default_rng(zlib.crc32(('add_n|' + name).encode()))
    dtype, shape = case['dtype'], case['shape']
    out = []
    rows = case.get('rows')
    for k, s in enumerate(case['stypes']):
        if s == 'row_sparse':
            out.append(_rsp(rng, shape, rows[k]))
            continue
        size = int(np.prod(shape))
        if case.get('zeros'):
            raw = np.asarray(SPECIAL[dtype][:2], RAW[dtype])[rng.integers(0, 2, size)]
        else:
            raw = _dense(rng, dtype, size)
        raw = raw.reshape(shape)
        if case.get('negzero'):
            raw[case['negzero']] = np.asarray(SPECIAL[dtype][1], RAW[dtype])
        out.append(raw)
    return out


def key_of(name):
    return [name + '_idx', name + '_val'] if all(s == 'row_sparse' for s in CASES[name]['stypes']) else [name]


def gen_add_n():
    """tests/golden/add_n.npz: the reference's outputs (every dtype but bfloat16), checked against
    the restatement, and the restatement's for bfloat16"""
    d = {}
    for name, case in CASES.items():
        ins = inputs(case, name)
        want = restate(case, ins)
        rsp = isinstance(want, tuple)
        if case['dtype'] in MSHADOW_FLAG:
            got = ref(case, ins)
            if rsp:
                assert np.array_equal(got[0], want[0]) and same_bits(got[1], want[1]), name
            else:
                assert same_bits(got, want, case['dtype']), name
        if rsp:
            d[name + '_idx'], d[name + '_val'] = want[0], want[1].view(np.uint32)
        else:
            d[name] = want
    np.savez_compressed(os.path.join(GOLD, "add_n.npz"), **d)


def nan_mask(bits, dtype):
    if dtype not in FLOATS:
        return np.zeros(np.shape(bits), bool)
    return np.isnan(values(bits, dtype))


def same_bits(a, b, dtype='float32'):
    """equal bit for bit, except that NaNs compare by position only (payloads differ by platform)"""
    a = np.asarray(a).view(RAW[dtype]) if np.asarray(a).dtype.kind == 'f' else np.asarray(a, RAW[dtype])
    b = np.asarray(b).view(RAW[dtype]) if np.asarray(b).dtype.kind == 'f' else np.asarray(b, RAW[dtype])
    if a.shape != b.shape:
        return False
    na, nb = nan_mask(a, dtype), nan_mask(b, dtype)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na], b[~nb]))


if __name__ == "__main__":
    build()
    assert ref_dense() is not None, "build oracle/_ref/libmxref_add_n.so first"
    assert ref_rsp() is not None, "build oracle/_ref/libmxref.so first (kvoracle.build(ref=True))"
    gen_add_n()
