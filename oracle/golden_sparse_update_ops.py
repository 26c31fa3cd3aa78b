"""TEST INFRASTRUCTURE ONLY -- the row_sparse forms of ftrl_update and _sparse_adagrad_update: a numpy
float32 restatement (`restate`), the reference's own CPU kernels (`RefSparseUpdate` over
oracle/_ref/libmxref_sparse_update.so, built from oracle/ref_sparse_update_ops.cc by
oracle/sparse_update_ops.mk), the seeded `CASES`, and the writer of tests/golden/sparse_update_ops.npz:

    make -f oracle/sparse_update_ops.mk && python oracle/golden_sparse_update_ops.py

Both take one call on flat buffers: `stypes` / `nnr` per operand (0 default, 1 row_sparse; a
row_sparse weight or state holds all rows or none), `bufs` (the gradient's nnr rows, every other
operand a rows x row_len table) and the gradient's ids. A state with no rows comes back zero-filled
with nnr == rows (FillDnsZerosRspImpl). Inputs are regenerated from each case's seed wherever the
fixture is read, so the fixture holds outputs only.
"""
import ctypes
import os
import subprocess
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import golden_update_ops as GU  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
F = np.float32
RSP, DNS = 1, 0
FULL_MAX = 1024    # tables up to this many elements keep their outputs in full
HEAD = GU.HEAD


def build():
    """oracle/_ref/libmxref_sparse_update.so, where the reference's sources exist"""
    if os.path.isfile("/root/reference/src/operator/optimizer_op-inl.h"):
        subprocess.run(["make", "-s", "-f", os.path.join(HERE, "sparse_update_ops.mk")], check=True)


class RefSparseUpdate(object):
    """mxref_sparse_update over oracle/_ref/libmxref_sparse_update.so"""

    def __init__(self, path):
        self.lib = ctypes.CDLL(path)

    def __call__(self, op, stypes, nnr, bufs, gidx, rows, row_len, inplace=True, **params):
        """runs one call in place on `bufs` (float32, C-contiguous) and `nnr` (a list); raises
        RuntimeError with the reference's message when it refuses"""
        n = len(bufs)
        assert all(b.dtype == F and b.flags.c_contiguous for b in bufs)
        st = (ctypes.c_int * n)(*stypes)
        nr = (ctypes.c_int64 * n)(*nnr)
        ptrs = (ctypes.c_void_p * n)(*[b.ctypes.data for b in bufs])
        ids = np.ascontiguousarray(gidx, np.int64)
        keys = [k.encode() for k in params]
        vals = [str(v).encode() for v in params.values()]
        err = ctypes.create_string_buffer(4096)
        rc = self.lib.mxref_sparse_update(
            op.encode(), ctypes.c_int(n), st, nr, ptrs, ids.ctypes.data_as(ctypes.c_void_p),
            ctypes.c_int64(rows), ctypes.c_int64(row_len), ctypes.c_int(1 if inplace else 0),
            ctypes.c_int(len(keys)), (ctypes.c_char_p * len(keys))(*keys),
            (ctypes.c_char_p * len(vals))(*vals), err, ctypes.c_int(len(err)))
        if rc != 0:
            raise RuntimeError(err.value.decode())
        nnr[:] = list(nr)


_ref = False


def ref():
    """The reference's kernels, or None when oracle/_ref/libmxref_sparse_update.so has not been built."""
    global _ref
    if _ref is False:
        path = os.path.join(HERE, "_ref", "libmxref_sparse_update.so")
        _ref = RefSparseUpdate(path) if os.path.exists(path) else None
    return _ref


# -------------------------------------------------------------------------------- restatement
def restate(op, stypes, nnr, bufs, gidx, rows, row_len, inplace=True, **params):
    """numpy restatement of one call, in place on `bufs` / `nnr` like RefSparseUpdate.__call__"""
    P = dict(params)
    for i in range(2, len(bufs)):                     # FillDnsZerosRspImpl of an empty state
        if stypes[i] == RSP and nnr[i] == 0:
            bufs[i][...] = 0
            nnr[i] = rows
    if nnr[1] == 0:
        return
    assert inplace
    idx = np.asarray(gidx, np.int64)
    w, g = bufs[0][idx], bufs[1]
    if op in ('ftrl_update', '_sparse_ftrl_update'):
        # FtrlDnsRspDnsKernel computes FtrlUpdateKernel's tree per element: the dense restatement
        out, (z, n) = GU.restate('ftrl_update', [w, g, bufs[2][idx], bufs[3][idx]], P)
        bufs[2][idx], bufs[3][idx] = z, n
    else:
        # AdagradDnsRspDnsKernel<cpu> (optimizer_op-inl.h:2507-2531)
        lr = GU.stof(P['lr'])
        eps = GU.stof(P['epsilon']) if 'epsilon' in P else F(1.0e-7)
        rescale = GU.stof(P.get('rescale_grad', 1.0))
        clip = GU.stof(P.get('clip_gradient', -1.0))
        gr = g * rescale
        if clip >= 0:
            gr = GU._clip(gr, clip)
        h = bufs[2][idx] + gr * gr
        out = w - (gr / np.sqrt(h + eps)) * lr
        bufs[2][idx] = h
    bufs[0][idx] = out


# ------------------------------------------------------------------------------------ cases
ROW_LENS = [1, 3, 4, 5, 512]
ROWSETS = ['none', 'one', 'all', 'subset']
FORMS = {'ftrl': ('ftrl_update', RSP), 'adagrad': ('_sparse_adagrad_update', RSP),
         'adagrad_dns': ('_sparse_adagrad_update', DNS)}
VARIANTS = {  # (params, states start empty)
    'ftrl': {'plain': (dict(lr=0.1, lamda1=0.01, beta=1, wd=0.0, rescale_grad=1.0), True),
             'clip_wd': (dict(lr=0.1, lamda1=0.01, beta=1, wd=0.001, rescale_grad=0.5, clip_gradient=0.3),
                         False)},
    'adagrad': {'plain': (dict(lr=0.05, wd=0.0, epsilon=1e-07, rescale_grad=1.0), True),
                'clip': (dict(lr=0.05, wd=0.0, epsilon=1e-06, rescale_grad=0.5, clip_gradient=0.3), False)},
}
VARIANTS['adagrad_dns'] = {k: (p, False) for k, (p, _) in VARIANTS['adagrad'].items()}


def table_rows(row_len):
    return 9 if row_len >= 512 else 23


def _cases():
    c = {}
    for form, variants in VARIANTS.items():
        op, wst = FORMS[form]
        for vname, (params, empty) in variants.items():
            for row_len in ROW_LENS:
                for rs in ROWSETS:
                    c['%s_%s_L%d_%s' % (form, vname, row_len, rs)] = dict(
                        form=form, op=op, wstype=wst, rows=table_rows(row_len), row_len=row_len,
                        rowsets=[rs], params=params, empty=empty)
            for row_len in (3, 512):                   # three chained steps over different rows
                c['%s_%s_L%d_chain3' % (form, vname, row_len)] = dict(
                    form=form, op=op, wstype=wst, rows=table_rows(row_len), row_len=row_len,
                    rowsets=['subset', 'subset', 'all'], params=params, empty=empty)
    return c


CASES = _cases()


def pick_rows(rng, rs, rows):
    if rs == 'none':
        return np.zeros(0, np.int64)
    if rs == 'one':
        return np.array([rows // 2], np.int64)
    if rs == 'all':
        return np.arange(rows, dtype=np.int64)
    inner = rng.choice(np.arange(1, rows - 1), size=max(1, (rows - 2) // 3), replace=False)
    return np.unique(np.concatenate([[0, rows - 1], inner])).astype(np.int64)


def inputs(case, name=None):
    """(tables [w, states...] as rows x row_len, per-step [(gidx, gval)], states' initial nnr)"""
    rows, L = case['rows'], case['row_len']
    key = name or '%s|%d|%d|%s|%d' % (case['form'], rows, L, ','.join(case['rowsets']), case['empty'])
    rng = np.random.default_rng(zlib.crc32(key.encode()))
    u = lambda *s: rng.uniform(-1, 1, s).astype(F)     # noqa: E731
    w = u(rows, L)
    ftrl = case['op'] != '_sparse_adagrad_update'
    if ftrl:                                  # z around +-lamda1 (incl. exact zeros), n >= 0
        z = (u(rows, L) * F(0.02)).astype(F)
        z.reshape(-1)[::7] = 0
        states = [z, (rng.uniform(0, 0.5, (rows, L))).astype(F)]
    else:
        states = [rng.uniform(0, 1, (rows, L)).astype(F)]
    if case['empty']:
        states = [np.zeros_like(s) for s in states]
    steps = []
    for rs in case['rowsets']:
        ids = pick_rows(rng, rs, rows)
        g = u(len(ids), L)
        if ftrl:
            g = (g * F(0.004)).astype(F)      # small: |z| stays near lamda1, w*sqrt terms matter
            g.reshape(-1)[::11] = 0
        steps.append((ids, g))
    st_nnr = [0 if (case['empty'] and case['wstype'] == RSP) else rows for _ in states]
    return [w] + states, steps, st_nnr


def run(fn, case, name=None):
    """all steps of a case through fn (ref() or restate): final tables and the states' nnr"""
    tables, steps, st_nnr = inputs(case, name)
    tables = [t.copy() for t in tables]
    nst = len(tables) - 1
    st = case['wstype']
    stypes = [st, RSP] + [st] * nst
    nnr_states = list(st_nnr)
    for ids, g in steps:
        nnr = [case['rows'] if st == RSP else 0, len(ids)] + nnr_states
        bufs = [tables[0], np.ascontiguousarray(g)] + tables[1:]
        fn(case['op'], stypes, nnr, bufs, ids, case['rows'], case['row_len'], True, **case['params'])
        nnr_states = nnr[2:]
    return tables, nnr_states


def fixture_entries(name, case, tables, nnr_states):
    d = {'%s|nnr' % name: np.array(nnr_states, np.int64)}
    for tag, a in zip(['w'] + ['s%d' % i for i in range(len(tables) - 1)], tables):
        a = np.ascontiguousarray(a)
        if a.size <= FULL_MAX:
            d['%s|%s' % (name, tag)] = a
        else:
            d['%s|%s|sha256' % (name, tag)] = GU.digest(a)
            d['%s|%s|head' % (name, tag)] = a.reshape(-1)[:HEAD].copy()
    return d


def gen_sparse_update_ops():
    """tests/golden/sparse_update_ops.npz: outputs of the reference's own kernels"""
    d = {}
    for name, case in CASES.items():
        d.update(fixture_entries(name, case, *run(ref(), case)))
    np.savez_compressed(os.path.join(GOLD, "sparse_update_ops.npz"), **d)


if __name__ == "__main__":
    build()
    assert ref() is not None, "build oracle/_ref/libmxref_sparse_update.so first"
    gen_sparse_update_ops()
