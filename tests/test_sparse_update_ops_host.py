"""The row_sparse forms of ftrl_update and _sparse_adagrad_update without a GPU: the operator names
and the alias resolve, the numpy restatement (oracle/golden_sparse_update_ops.py) equals
tests/golden/sparse_update_ops.npz everywhere and the reference's own kernels live (fixture cases plus
random layouts), the tests/compat mirror of Ftrl and AdaGrad issues the reference classes' operator
calls and reaches their tables and states, and the row-gather kernels compile for sm_90a without
spills."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import golden_sparse_update_ops as GS
import ref_python as RP
import ref_python_sparse_update as RPS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
live = pytest.mark.skipif(GS.ref() is None, reason="needs oracle/_ref/libmxref_sparse_update.so")
live_py = pytest.mark.skipif(not RPS.available(), reason="needs /root/reference and oracle/_ref/ libraries")


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_sparse_update_operators_are_registered():
    import anand_mxnet_b200 as mx
    for name in ['ftrl_update', '_sparse_ftrl_update', '_sparse_adagrad_update']:
        h = ctypes.c_void_p()
        assert mx.base._LIB.NNGetOpHandle(name.encode(), ctypes.byref(h)) == 0 and h.value, name
    assert callable(mx.nd.sparse.ftrl_update) and callable(mx.nd.sparse.adagrad_update)


def test_fixture_covers_every_case():
    g = np.load(os.path.join(ROOT, "tests", "golden", "sparse_update_ops.npz"))
    assert {k.split('|')[0] for k in g.files} == set(GS.CASES)
    assert {c['row_len'] for c in GS.CASES.values()} == {1, 3, 4, 5, 512}
    assert {c['form'] for c in GS.CASES.values()} == {'ftrl', 'adagrad', 'adagrad_dns'}


def check(g, name, tables, nnr):
    assert eq(np.array(nnr, np.int64), g['%s|nnr' % name]), name
    for tag, a in zip(['w'] + ['s%d' % i for i in range(len(tables) - 1)], tables):
        if a.size <= GS.FULL_MAX:
            assert eq(a, g['%s|%s' % (name, tag)]), (name, tag)
        else:
            assert eq(a.reshape(-1)[:GS.HEAD], g['%s|%s|head' % (name, tag)]), (name, tag)
            assert eq(GS.GU.digest(a), g['%s|%s|sha256' % (name, tag)]), (name, tag)


@pytest.mark.parametrize("name", sorted(GS.CASES))
def test_restatement_matches_golden(golden, name):
    check(golden("sparse_update_ops"), name, *GS.run(GS.restate, GS.CASES[name]))


@live
@pytest.mark.parametrize("name", sorted(GS.CASES))
def test_restatement_matches_live_reference(name):
    case = GS.CASES[name]
    t1, n1 = GS.run(GS.ref(), case)
    t2, n2 = GS.run(GS.restate, case)
    assert n1 == n2 and all(eq(a, b) for a, b in zip(t1, t2)), name


def random_case(seed):
    rng = np.random.default_rng(seed)
    form = ['ftrl', 'adagrad', 'adagrad_dns'][seed % 3]
    op, wst = GS.FORMS[form]
    params = dict(lr=float(rng.choice([0.1, 0.01, 0.37])), rescale_grad=float(rng.choice([1.0, 0.5, 1 / 96])))
    if rng.random() < 0.5:
        params['clip_gradient'] = float(rng.choice([0.0, 0.05, 0.7]))
    if form == 'ftrl':
        params.update(lamda1=float(rng.choice([0.01, 0.003])), beta=float(rng.choice([1.0, 0.5])))
        if rng.random() < 0.5:
            params['wd'] = float(rng.choice([1e-4, 0.01]))
    elif rng.random() < 0.5:
        params['epsilon'] = float(rng.choice([1e-7, 3.3e-07, 1e-3]))
    steps = int(rng.integers(1, 4))
    return dict(form=form, op=op, wstype=wst, rows=int(rng.integers(3, 40)),
                row_len=int(rng.choice([1, 2, 3, 4, 5, 7, 8, 16, 33])),
                rowsets=[str(rng.choice(GS.ROWSETS)) for _ in range(steps)], params=params,
                empty=bool(wst == GS.RSP and rng.random() < 0.5))


@live
@pytest.mark.parametrize("seed", range(50))
def test_restatement_matches_live_reference_random(seed):
    """random form, table, row sets, steps and parameters (clip on / off, rescale, wd for Ftrl)"""
    case = random_case(seed)
    t1, n1 = GS.run(GS.ref(), case, 'random%d' % seed)
    t2, n2 = GS.run(GS.restate, case, 'random%d' % seed)
    assert n1 == n2 and all(eq(a, b) for a, b in zip(t1, t2)), case


@live
def test_reference_refusals():
    """the reference's dispatch as restated in the oracle library refuses what the GPU operators
    refuse: missing weight rows, wd for AdaGrad, a distinct out, mixed storage types"""
    r, rows, L = GS.ref(), 4, 3
    t = lambda: np.ones((rows, L), np.float32)  # noqa: E731
    g, ids = np.ones((1, L), np.float32), np.array([1])
    cases = [
        ('ftrl_update', [1, 1, 1, 1], [rows - 1, 1, 0, 0], True, {}, 'all rows containing non-zeros'),
        ('ftrl_update', [1, 1, 0, 1], [rows, 1, 0, 0], True, {}, 'Inconsistent storage type'),
        ('ftrl_update', [1, 1, 1, 1], [rows, 1, 0, 0], False, {}, 'kWriteInplace'),
        ('_sparse_adagrad_update', [1, 1, 1], [rows, 1, 0], True, {'wd': 0.1}, 'does not support wd'),
        ('_sparse_adagrad_update', [0, 1, 1], [0, 1, 0], True, {}, 'unsupported storage types'),
        ('_sparse_adagrad_update', [1, 1, 1], [rows, 1, 0], False, {}, 'kWriteInplace'),
    ]
    for op, st, nnr, inplace, extra, msg in cases:
        bufs = [t(), g] + [t() for _ in st[2:]]
        with pytest.raises(RuntimeError, match=msg):
            r(op, st, list(nnr), bufs, ids, rows, L, inplace, lr=0.1, **extra)


# ------------------------------------------------------------------ the tests/compat mirror
@live_py
@pytest.mark.parametrize("name", sorted(RPS.trajectory_cases()))
def test_compat_mirror_vs_reference(golden, name):
    from compat import mxnet_optimizer as B
    from compat import mxnet_optimizer_update as U
    from compat import mxnet_optimizer_sparse as M
    case = RPS.trajectory_cases()[name]
    with RPS.reference_python_sparse_update() as (opt, _):
        RP.LOG[:] = []
        want = RPS.run_trajectory(opt, case)
        want_log = list(RP.LOG)
        saved = [(m, dict(m.__dict__)) for m in (B, U, M)]
        try:
            for m in (B, U, M):
                m.__dict__.update(RP.op_table())
                m.__dict__.update(RPS.op_table())
            RP.LOG[:] = []
            got = RPS.run_trajectory(M, case)
            got_log = list(RP.LOG)
        finally:
            for m, d in saved:
                m.__dict__.clear()
                m.__dict__.update(d)
    assert got_log == want_log and len(want_log) == 4 * len(case['shapes'])
    gold = golden("updater_trajectories_sparse")
    for step, ((wg, sg), (ww, sw)) in enumerate(zip(got, want)):
        for k in range(len(wg)):
            assert eq(wg[k], ww[k]) and eq(ww[k], gold["%s_step%d_w%d" % (name, step, k)]), (name, step, k)
            for i, (a, b) in enumerate(zip(sg[k], sw[k])):
                assert eq(a, b) and eq(b, gold["%s_step%d_w%d_s%d" % (name, step, k, i)]), (name, step, k, i)
    for k, s in enumerate(case['shapes']):        # rows no gradient lists keep their initial values
        cold = RPS.cold_rows(s)
        assert eq(want[-1][0][k][cold], case['w0'][k][cold])


def test_compat_adagrad_dense_gradient_is_refused():
    from compat import mxnet_optimizer_sparse as M
    opt = M.AdaGrad(learning_rate=0.1)

    class Dense(M.NDArray):
        def __init__(self):
            pass
        stype = 'default'
    with pytest.raises(NotImplementedError, match='square / clip / division'):
        opt.update(0, Dense(), Dense(), None)


def test_ptxas_no_spills_row_updates(tmp_path):
    """the five row-gather instantiations (Ftrl, AdaGrad, lazy SGD, SGD-momentum and Adam) and the id
    fill of rowsparse_kernels.cu: no spills, no stack frame"""
    from anand_mxnet_b200 import build as B
    src = os.path.join(B.CSRC, "rowsparse_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o",
                                                     str(tmp_path / "r.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    blocks = re.split(r"Compiling entry function ", r.stderr)[1:]   # one per kernel
    found = [(b.split("'")[1],) + re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, "
                                            r"(\d+) bytes spill loads", b).groups()
             for b in blocks if re.match(r"'\w*(rsp_row_update_kernel|fill_row_ids_kernel)", b)]
    assert len(found) == 6, r.stderr[-4000:]
    assert all(f == '0' and s == '0' and l == '0' for _, f, s, l in found), found
