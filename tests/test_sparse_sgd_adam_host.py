"""sgd_update, sgd_mom_update and adam_update on row_sparse weights, without a GPU: the C restatement
(oracle/kvoracle.c) equals tests/golden/sparse_sgd_adam_ops.npz on every case, and so do the
reference's own kernels where they are built here; the reference's SGD, ccSGD and Adam classes
reproduce tests/golden/updater_trajectories_sparse_sgd_adam.npz; the tests/compat mirror of those
classes issues the same operator calls with the same parameter strings, creates states of the same
storage types and has the same signatures."""
import inspect

import numpy as np
import pytest

import golden_sparse_sgd_adam as GSA
import golden_sparse_update_ops as GS
import golden_update_ops as GU
import kvoracle as K
import ref_python as RP
import ref_python_sparse_sgd_adam as RSA

live = pytest.mark.skipif(K.ref() is None, reason="needs the reference's kernels (oracle/_ref/libmxref.so)")
live_py = pytest.mark.skipif(not RSA.available(), reason="needs /root/reference and oracle/_ref/libmxref.so")


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def check(gold, name, tables, nnr):
    case = GSA.CASES[name]
    want = GS.fixture_entries(name, case, tables, nnr)
    assert sorted(want) == sorted(k for k in gold.files if k.startswith(name + '|'))
    for k, v in want.items():
        assert eq(v, gold[k]), k


def test_fixture_covers_every_form_and_edge(golden):
    gold = golden(GSA.NAME)
    names = {k.split('|')[0] for k in gold.files}
    assert names == set(GSA.CASES)
    for form in GSA.FORMS:
        mine = [c for c in GSA.CASES.values() if c['form'] == form]
        assert {c['row_len'] for c in mine} >= {1, 3, 4, 133, 260}
        assert {rs for c in mine for rs in c['rowsets']} == set(GSA.ROWSETS)
        assert {('clip_gradient' in c['params'], c['params'].get('clip_gradient')) for c in mine} == \
            {(False, None), (True, 0.0), (True, 0.3)}
    assert any(c['rows'] * c['row_len'] > GS.FULL_MAX * 64 for c in GSA.CASES.values())


@pytest.mark.parametrize("name", sorted(GSA.CASES))
def test_restatement_matches_golden(golden, name):
    check(golden(GSA.NAME), name, *GSA.run(K.get_oracle(), name))


@live
@pytest.mark.parametrize("name", sorted(GSA.CASES))
def test_reference_kernels_match_golden(golden, name):
    check(golden(GSA.NAME), name, *GSA.run(K.ref(), name))


@live_py
def test_reference_classes_match_trajectories(golden):
    gold = golden("updater_trajectories_sparse_sgd_adam")
    with RSA.reference_python_sparse_sgd_adam() as (opt, _):
        for name, case in RSA.trajectory_cases().items():
            for step, (ws, sts) in enumerate(RSA.run_trajectory(opt, case)):
                for k, (w, st) in enumerate(zip(ws, sts)):
                    assert RSA.matches(gold, "%s_step%d_w%d" % (name, step, k), w), (name, step, k)
                    assert len(st) == RSA.n_states(gold, name, step, k)
                    for i, s in enumerate(st):
                        assert RSA.matches(gold, "%s_step%d_w%d_s%d" % (name, step, k, i), s), (name, step, k, i)


# ------------------------------------------------------------------ the tests/compat mirror
@live_py
@pytest.mark.parametrize("name", sorted(RSA.trajectory_cases()))
def test_compat_mirror_vs_reference(golden, name):
    """the mirror classes over the same stand-in arrays and operators as the reference's classes:
    the same operator calls with the same parameter strings, the same tables and states"""
    from compat import mxnet_optimizer as B
    from compat import mxnet_optimizer_sparse_sgd as M
    case = RSA.trajectory_cases()[name]
    with RSA.reference_python_sparse_sgd_adam() as (opt, _):
        RP.LOG[:] = []
        want = RSA.run_trajectory(opt, case)
        want_log = list(RP.LOG)
        saved = [(m, dict(m.__dict__)) for m in (B, M)]
        try:
            for m in (B, M):
                m.__dict__.update(RP.op_table())
                m.__dict__.update(RSA.op_table())
            RP.LOG[:] = []
            got = RSA.run_trajectory(M, case)
            got_log = list(RP.LOG)
        finally:
            for m, d in saved:
                m.__dict__.clear()
                m.__dict__.update(d)
    assert got_log == want_log and len(want_log) == 4 * len(case['shapes'])
    assert {n for n, _ in want_log} <= {'sgd_update', 'sgd_mom_update', 'adam_update'}
    gold = golden("updater_trajectories_sparse_sgd_adam")
    for step, ((wg, sg), (ww, sw)) in enumerate(zip(got, want)):
        for k in range(len(wg)):
            assert eq(wg[k], ww[k]) and RSA.matches(gold, "%s_step%d_w%d" % (name, step, k), ww[k]), (name, step, k)
            assert len(sg[k]) == len(sw[k])
            for i, (a, b) in enumerate(zip(sg[k], sw[k])):
                assert eq(a, b) and RSA.matches(gold, "%s_step%d_w%d_s%d" % (name, step, k, i), b), (name, step, k, i)


@live_py
def test_compat_mirror_state_stypes_and_signatures():
    from compat import mxnet_optimizer_sparse_sgd as M
    with RSA.reference_python_sparse_sgd_adam() as (opt, _):
        w = RSA.RSU.RspNDArray((5, 3), np.arange(5), np.ones((5, 3), np.float32))
        for cls, kw in [('SGD', dict(momentum=0.9)), ('ccSGD', dict(momentum=0.9)), ('Adam', {})]:
            for lazy in (True, False):
                ref_st = getattr(opt, cls)(lazy_update=lazy, **kw).create_state(0, w)
                ref_st = list(ref_st) if isinstance(ref_st, tuple) else [ref_st]
                M.__dict__['zeros'], saved = RSA.RSU.zeros, M.__dict__['zeros']
                try:
                    st = getattr(M, cls)(lazy_update=lazy, **kw).create_state(0, w)
                finally:
                    M.__dict__['zeros'] = saved
                st = list(st) if isinstance(st, tuple) else [st]
                assert [s.stype for s in st] == [s.stype for s in ref_st] == \
                    ['row_sparse' if lazy else 'default'] * len(st)
        for cls in ('SGD', 'ccSGD', 'Adam'):
            for meth in ('__init__', 'create_state', 'update'):
                assert inspect.signature(getattr(getattr(M, cls), meth)) == \
                    inspect.signature(getattr(getattr(opt, cls), meth)), (cls, meth)


def test_compat_mirror_is_not_registered():
    from compat import mxnet_optimizer as B
    from compat import mxnet_optimizer_sparse_sgd as M
    reg = B.Optimizer.opt_registry
    assert reg['sgd'] is B.SGD and reg['adam'] is B.Adam and 'ccsgd' not in reg
    assert M.SGD is not B.SGD and issubclass(M.ccSGD, M.SGD) and issubclass(M.Adam, B.Adam)

