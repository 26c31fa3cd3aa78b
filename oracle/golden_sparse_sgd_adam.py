"""TEST INFRASTRUCTURE ONLY -- sgd_update, sgd_mom_update and adam_update on a row_sparse weight that
holds every row: the seeded `CASES` and the writer of tests/golden/sparse_sgd_adam_ops.npz.

    make -C oracle oracle ref && python oracle/golden_sparse_sgd_adam.py

Such a weight's values are the dense row-major table, so the reference runs the dense-weight kernels
on them (SGDUpdateRspImpl, SGDMomLazyUpdateRspImpl / SGDMomStdUpdateRspImpl, AdamLazyUpdateRspImpl /
AdamStdUpdateRspImpl, optimizer_op-inl.h:534-545, 851-870, 949-969, 1464-1487, 1513-1528). Those
kernels are already restated in oracle/kvoracle.c and pinned to the reference's own SGDDnsRspKernel,
SGDMomDnsRspDnsKernel, AdamDnsRspDnsKernel and *StdDnsRspDnsKernel (`run(K.ref(), ...)` calls the
compiled reference kernels through oracle/_ref/libmxref.so). The NDArray-level dispatch around them
is restated in `step`: the form is chosen from lazy_update and the states' storage type
(StdOptStorageType, :877-921), and a row_sparse state with no rows is zero-filled to every row first
(FillDnsZerosRspImpl). Inputs are regenerated from each case's seed wherever the fixture is read, so
the fixture holds outputs only, in golden_sparse_update_ops' layout.
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
import kvoracle as K  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
F = np.float32
RSP, DNS = GS.RSP, GS.DNS
NAME = "sparse_sgd_adam_ops"

# name: (operator, number of states, the states' storage type, lazy_update)
FORMS = {
    'sgd_lazy': ('sgd_update', 0, None, True),
    'sgd_std': ('sgd_update', 0, None, False),
    'mom_rsp_lazy': ('sgd_mom_update', 1, RSP, True),
    'mom_rsp_std': ('sgd_mom_update', 1, RSP, False),
    'mom_dns_lazy': ('sgd_mom_update', 1, DNS, True),     # dense states: the standard form
    'mom_dns_std': ('sgd_mom_update', 1, DNS, False),
    'adam_rsp_lazy': ('adam_update', 2, RSP, True),
    'adam_rsp_std': ('adam_update', 2, RSP, False),
    'adam_dns_lazy': ('adam_update', 2, DNS, True),
    'adam_dns_std': ('adam_update', 2, DNS, False),
}
# momentum 0 and 0.9; clip_gradient absent, 0 and hit; wd and rescale_grad off and on
PARAMS = {
    'plain': dict(lr=0.1, wd=0.0, rescale_grad=1.0),
    'wd_rescale': dict(lr=0.1, wd=0.01, rescale_grad=0.5),
    'clip0': dict(lr=0.1, wd=0.001, rescale_grad=1.0, clip_gradient=0.0),
    'cliphit': dict(lr=0.1, wd=0.0, rescale_grad=2.0, clip_gradient=0.3),
}
ROW_LENS = [1, 3, 4, 133, 260]      # 1, odd, the float4 width, and past a warp's 128-element sweep
ROWSETS = ['none', 'one', 'ends', 'all', 'subset']
BIG_ROWS = 20000                    # 2 500 CTAs of 8 row warps: more than one wave on an H100


def params_of(form, pname):
    op = FORMS[form][0]
    p = dict(PARAMS[pname])
    if op == 'sgd_mom_update':
        p['momentum'] = 0.0 if pname == 'plain' else 0.9
    if op == 'adam_update':
        p.update(lr=0.01, beta1=0.9, beta2=0.999, epsilon=1e-08)
    p['lazy_update'] = FORMS[form][3]
    return p


def _cases():
    c = {}
    i = 0
    for form, (op, nst, sst, lazy) in FORMS.items():
        for pname in PARAMS:
            for L in ROW_LENS:
                rs = ROWSETS[i % len(ROWSETS)]
                i += 1
                c['%s_%s_L%d_%s' % (form, pname, L, rs)] = dict(
                    form=form, rows=GS.table_rows(L) if L < 260 else 9, row_len=L, rowsets=[rs],
                    params=params_of(form, pname), empty=(i % 2 == 0))
        for rs in ROWSETS:
            c['%s_wd_rescale_L5_%s' % (form, rs)] = dict(
                form=form, rows=23, row_len=5, rowsets=[rs], params=params_of(form, 'wd_rescale'),
                empty=rs in ('none', 'one'))
        # three chained steps; a row_sparse state starts with no rows
        c['%s_cliphit_L4_chain3' % form] = dict(
            form=form, rows=23, row_len=4, rowsets=['subset', 'ends', 'all'],
            params=params_of(form, 'cliphit'), empty=True)
    for form in ('sgd_std', 'mom_rsp_lazy', 'mom_dns_std', 'adam_rsp_lazy', 'adam_rsp_std'):
        c['%s_big_%s' % (form, 'subset')] = dict(
            form=form, rows=BIG_ROWS, row_len=4, rowsets=['subset', 'all'],
            params=params_of(form, 'wd_rescale'), empty=True)
    return c


CASES = _cases()


def pick_rows(rng, rs, rows):
    if rs == 'ends':
        return np.array([0, rows - 1], np.int64)
    return GS.pick_rows(rng, rs, rows)


def inputs(name):
    """(tables [w, states...] as rows x row_len, per-step [(gidx, gval)], the states' initial nnr)"""
    case = CASES[name]
    rows, L = case['rows'], case['row_len']
    nst, sst = FORMS[case['form']][1], FORMS[case['form']][2]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    u = lambda *s: rng.uniform(-1, 1, s).astype(F)     # noqa: E731
    w = u(rows, L)
    states = [u(rows, L) * F(0.1), rng.uniform(0, 0.01, (rows, L)).astype(F)][:nst]
    empty = case['empty'] and sst == RSP
    if empty:
        states = [np.zeros_like(s) for s in states]
    steps = []
    for rs in case['rowsets']:
        ids = pick_rows(rng, rs, rows)
        steps.append((ids, u(len(ids), L)))
    return [w] + states, steps, [0 if empty else rows for _ in states]


def step(b, op, tables, nnr, sst, ids, g, params):
    """one call of `op` in place on `tables` ([w, states...] as rows x row_len) and the row_sparse
    states' `nnr` through backend b (K.get_oracle() or K.ref()); params: the operator's keyword
    arguments, which it parses from their str() (lazy_update included)"""
    P = dict(params)
    lazy = str(P.pop('lazy_update', True)) == 'True' and sst != DNS
    f = {k: GU.stof(v) for k, v in P.items()}
    kw = dict(lr=f['lr'], wd=f.get('wd', F(0)), rescale=f.get('rescale_grad', F(1)),
              clip=f['clip_gradient'] if 'clip_gradient' in f else None)
    if op == 'adam_update':
        kw.update(beta1=f.get('beta1', F(0.9)), beta2=f.get('beta2', F(0.999)),
                  eps=f.get('epsilon', F(1e-8)))
    if op == 'sgd_mom_update':
        kw['momentum'] = f.get('momentum', F(0))
    rows = tables[0].shape[0]
    for i in range(len(tables) - 1):          # FillDnsZerosRspImpl of a state with no rows
        if sst == RSP and nnr[i] == 0:
            tables[1 + i][...] = 0
            nnr[i] = rows
    if lazy and len(ids) == 0:
        return                                # the lazy form touches nothing
    fn = {'sgd_update': 'sgd', 'sgd_mom_update': 'sgd_mom', 'adam_update': 'adam'}[op]
    getattr(b, '%s_%srsp_update' % (fn, '' if lazy else 'std_'))(
        *tables, np.ascontiguousarray(ids, np.int64), np.ascontiguousarray(g), **kw)


def run(b, name):
    """all steps of case `name` through backend b: final tables and the row_sparse states' nnr"""
    case = CASES[name]
    op, _, sst, _ = FORMS[case['form']]
    tables, steps, nnr = inputs(name)
    tables = [t.copy() for t in tables]
    for ids, g in steps:
        step(b, op, tables, nnr, sst, ids, g, case['params'])
    return tables, (nnr if sst == RSP else [])


def gen():
    """tests/golden/sparse_sgd_adam_ops.npz: outputs of the reference's own kernels, which the
    restatement must equal on every case"""
    assert K.ref() is not None, "build oracle/_ref/libmxref.so first (make -C oracle ref)"
    d = {}
    for name in CASES:
        tables, nnr = run(K.ref(), name)
        mine, mine_nnr = run(K.get_oracle(), name)
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(tables, mine)), name
        assert nnr == mine_nnr
        d.update(GS.fixture_entries(name, CASES[name], tables, nnr))
    np.savez_compressed(os.path.join(GOLD, NAME + ".npz"), **d)
    return len(CASES)


if __name__ == "__main__":
    print(gen(), "cases")
