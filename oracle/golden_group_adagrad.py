"""TEST INFRASTRUCTURE ONLY -- _contrib_group_adagrad_update (GroupAdaGrad's lazy row update): a numpy
float32 restatement (`restate`), the reference's own CPU kernel (`ref()` over
oracle/_ref/libmxref_group_adagrad.so, built from oracle/ref_group_adagrad.cc by
oracle/group_adagrad.mk), the seeded `CASES`, and the writer of tests/golden/group_adagrad.npz:

    make -f oracle/group_adagrad.mk && python oracle/golden_group_adagrad.py

One call runs on flat buffers, with the convention of golden_sparse_update_ops: `stypes` / `nnr` per
operand (0 default, 1 row_sparse; a row_sparse weight or history holds all rows or none), `bufs`
(weight rows x L, the gradient's nnr rows x L, history rows x 1) and the gradient's ids. A history
with no rows comes back zero-filled with nnr == rows (FillDnsZerosRspImpl).

The reference folds each row's sum of squares strictly left to right in float32 (its CPU loop,
built without fast-math, cannot be reassociated). `restate(..., fold='tree')` and `fold='pairwise'`
sum in a warp-tree and in numpy's pairwise order instead; the generator asserts that for every form,
variant and L >= 32 both give other bits than the fixture on some case, so the fixture tells the
orders apart (check_order_sensitivity).
"""
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import golden_sparse_update_ops as GS  # noqa: E402
import golden_update_ops as GU  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
F = np.float32
RSP, DNS = GS.RSP, GS.DNS
OP = '_contrib_group_adagrad_update'
FULL_MAX = GS.FULL_MAX
HEAD = GS.HEAD


def build():
    """oracle/_ref/libmxref_group_adagrad.so, where the reference's sources exist"""
    if os.path.isfile("/root/reference/src/operator/contrib/optimizer_op-inl.h"):
        import subprocess
        subprocess.run(["make", "-s", "-f", os.path.join(HERE, "group_adagrad.mk")], check=True)


_ref = False


def ref():
    """The reference's kernel (same front-end as golden_sparse_update_ops.RefSparseUpdate), or None
    when oracle/_ref/libmxref_group_adagrad.so has not been built."""
    global _ref
    if _ref is False:
        path = os.path.join(HERE, "_ref", "libmxref_group_adagrad.so")
        _ref = GS.RefSparseUpdate(path) if os.path.exists(path) else None
    return _ref


# -------------------------------------------------------------------------------- restatement
def _sum_squares(sq, fold):
    """row sums of sq (n x L float32) in the given order"""
    if fold == 'seq':                       # ((0 + sq_0) + sq_1) + ...: add.accumulate is sequential
        return np.add.accumulate(sq, axis=1, dtype=F)[:, -1] if sq.shape[1] else np.zeros(len(sq), F)
    if fold == 'pairwise':                  # numpy's own reduction order
        return sq.sum(axis=1, dtype=F)
    # 'tree': 32 lanes fold strided elements, then a butterfly over the lanes
    n, L = sq.shape
    pad = np.zeros((n, -(-L // 32) * 32), F)
    pad[:, :L] = sq
    part = np.add.accumulate(pad.reshape(n, -1, 32), axis=1, dtype=F)[:, -1, :]
    while part.shape[1] > 1:
        h = part.shape[1] // 2
        part = (part[:, :h] + part[:, h:]).astype(F)
    return part[:, 0]


def restate(op, stypes, nnr, bufs, gidx, rows, row_len, inplace=True, fold='seq', **params):
    """numpy restatement of one call, in place on `bufs` / `nnr` like the reference library"""
    assert op == OP
    if stypes[0] == RSP and nnr[2] == 0:      # FillDnsZerosRspImpl of an empty history
        bufs[2][...] = 0
        nnr[2] = rows
    assert inplace
    if nnr[1] == 0:
        return
    lr = GU.stof(params['lr'])
    eps = GU.stof(params['epsilon']) if 'epsilon' in params else F(1.0e-5)
    rescale = GU.stof(params.get('rescale_grad', 1.0))
    clip = GU.stof(params.get('clip_gradient', -1.0))
    idx = np.asarray(gidx, np.int64)
    gr = (bufs[1].reshape(len(idx), row_len) * rescale).astype(F)
    if clip >= 0:
        gr = GU._clip(gr, clip)
    ssq = _sum_squares((gr * gr).astype(F), fold)
    h = bufs[2].reshape(rows)
    h[idx] = h[idx] + ssq / F(row_len)
    den = np.sqrt(h[idx] + eps).astype(F)
    w = bufs[0].reshape(rows, row_len)
    w[idx] = w[idx] - (lr * gr) / den[:, None]


# ------------------------------------------------------------------------------------ cases
ROW_LENS = [1, 3, 4, 5, 31, 32, 33, 512, 1000, 4099]
ROWSETS = GS.ROWSETS
VARIANTS = {  # (params, history starts empty)
    'plain': (dict(lr=0.05, epsilon=1e-05, rescale_grad=1.0), True),
    'clip0': (dict(lr=0.1, epsilon=1e-06, rescale_grad=1.0, clip_gradient=0.0), True),
    'clip': (dict(lr=0.05, epsilon=1e-05, rescale_grad=0.25, clip_gradient=0.5), False),
    'rescale': (dict(lr=0.2, epsilon=3e-07, rescale_grad=1 / 96), False),
}


def table_rows(row_len):
    return 5 if row_len > 512 else 9 if row_len >= 512 else 23


def _cases():
    c = {}
    for form, wst in (('rsp', RSP), ('dns', DNS)):
        for vname, (params, empty) in VARIANTS.items():
            for L in ROW_LENS:
                for rs in ROWSETS:
                    c['%s_%s_L%d_%s' % (form, vname, L, rs)] = dict(
                        form=form, wstype=wst, shape=(table_rows(L), L), rowsets=[rs], params=params,
                        empty=empty and wst == RSP)
            for L in (3, 33, 512, 4099):          # three chained steps over different rows
                c['%s_%s_L%d_chain3' % (form, vname, L)] = dict(
                    form=form, wstype=wst, shape=(table_rows(L), L), rowsets=['subset', 'subset', 'all'],
                    params=params, empty=empty and wst == RSP)
        for rs in ('subset', 'all'):                # a 3-D weight: rows of 4 x 8
            c['%s_3d_%s' % (form, rs)] = dict(form=form, wstype=wst, shape=(23, 4, 8), rowsets=[rs, rs],
                                              params=VARIANTS['clip'][0], empty=wst == RSP)
    return c


CASES = _cases()


def row_len(case):
    return int(np.prod(case['shape'][1:]))


def inputs(case, name=None):
    """(weight rows x L, history rows x 1, per-step [(gidx, gval)], the history's initial nnr).
    Gradients mix magnitudes (1e3 beside 0.1) so that the order of the sum of squares shows."""
    rows, L = case['shape'][0], row_len(case)
    key = name or 'ga|%s|%s|%s|%d' % (case['form'], case['shape'], ','.join(case['rowsets']), case['empty'])
    rng = np.random.default_rng(zlib.crc32(key.encode()))
    w = rng.uniform(-1, 1, (rows, L)).astype(F)
    h = np.zeros((rows, 1), F) if case['empty'] else rng.uniform(0, 2, (rows, 1)).astype(F)
    steps = []
    for rs in case['rowsets']:
        ids = GS.pick_rows(rng, rs, rows)
        # about half the squares are below half an ulp of a running sum >= 1e6 (the first square
        # already is): a left fold drops each of them, a tree sums some of them first
        scale = np.where(rng.random((len(ids), L)) < 0.5, F(1e3), F(0.15)).astype(F)
        scale[:, 0] = F(1e3)
        g = (rng.uniform(0.5, 1, (len(ids), L)).astype(F) * scale).astype(F)
        g[rng.random((len(ids), L)) < 0.5] *= F(-1)
        steps.append((ids, g))
    return w, h, steps, (0 if case['empty'] else rows)


def run(fn, case, name=None, **kw):
    """all steps of a case through fn (ref() or restate): final weight, history and the history's nnr"""
    w, h, steps, nnr_h = inputs(case, name)
    w, h = w.copy(), h.copy()
    st = case['wstype']
    rows, L = case['shape'][0], row_len(case)
    for ids, g in steps:
        nnr = [rows if st == RSP else 0, len(ids), nnr_h if st == RSP else 0]
        fn(OP, [st, RSP, st], nnr, [w, np.ascontiguousarray(g), h], ids, rows, L, True,
           **dict(case['params'], **kw))
        nnr_h = nnr[2]
    return [w, h], [nnr_h]


def _same(a, b):
    return all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(a, b))


def check_order_sensitivity():
    """For every form, variant and L >= 32, some case's weight or history changes when the sum of
    squares is taken as a warp-tree, and some when it is taken in numpy's pairwise order. clip0 is
    left out: it clips every gradient to 0, so every order sums zeros."""
    found = {}
    for name, case in CASES.items():
        if row_len(case) < 32 or name.split('_')[1] == 'clip0' or case['rowsets'] == ['none']:
            continue
        group = name.rsplit('_', 1)[0] if '_L' in name else name.split('_')[0] + '_3d'
        want, _ = run(restate, case)
        for fold in ('tree', 'pairwise'):
            found.setdefault((group, fold), False)
            if not found[(group, fold)]:
                found[(group, fold)] = not _same(run(restate, case, fold=fold)[0], want)
    missing = sorted(k for k, v in found.items() if not v)
    assert not missing, missing
    return sorted(found)


def fixture_entries(name, tables, nnr):
    return GS.fixture_entries(name, None, tables, nnr)


def gen_group_adagrad():
    """tests/golden/group_adagrad.npz: outputs of the reference's own kernel"""
    check_order_sensitivity()
    d = {}
    for name, case in CASES.items():
        tables, nnr = run(ref(), case)
        t2, n2 = run(restate, case)
        assert nnr == n2 and _same(tables, t2), name
        d.update(fixture_entries(name, tables, nnr))
    np.savez_compressed(os.path.join(GOLD, "group_adagrad.npz"), **d)


if __name__ == "__main__":
    build()
    assert ref() is not None, "build oracle/_ref/libmxref_group_adagrad.so first"
    gen_group_adagrad()
