"""_contrib_group_adagrad_update (GroupAdaGrad) without a GPU: the operator name resolves, the numpy
restatement (oracle/golden_group_adagrad.py) equals tests/golden/group_adagrad.npz and the
reference's own kernel live (fixture cases plus random layouts), the fixture tells a sequential sum
of squares from a warp-tree or pairwise one, the reference's dispatch refuses what the GPU operator
refuses, the tests/compat mirror issues the reference class's operator calls and reaches its tables
and histories, and the row kernel compiles for sm_90a without spills."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import golden_group_adagrad as GG
import ref_python as RP
import ref_python_group_adagrad as RPG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
live = pytest.mark.skipif(GG.ref() is None, reason="needs oracle/_ref/libmxref_group_adagrad.so")
live_py = pytest.mark.skipif(not RPG.available(), reason="needs /root/reference and oracle/_ref/ libraries")


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_group_adagrad_operator_is_registered():
    import anand_mxnet_b200 as mx
    h = ctypes.c_void_p()
    assert mx.base._LIB.NNGetOpHandle(b'_contrib_group_adagrad_update', ctypes.byref(h)) == 0 and h.value
    assert callable(mx.nd.contrib.group_adagrad_update)


def test_fixture_covers_every_case():
    g = np.load(os.path.join(ROOT, "tests", "golden", "group_adagrad.npz"))
    assert {k.split('|')[0] for k in g.files} == set(GG.CASES)
    assert {GG.row_len(c) for c in GG.CASES.values()} == {1, 3, 4, 5, 31, 32, 33, 512, 1000, 4099}
    assert {c['shape'] for c in GG.CASES.values() if len(c['shape']) == 3} == {(23, 4, 8)}


def check(g, name, tables, nnr):
    assert eq(np.array(nnr, np.int64), g['%s|nnr' % name]), name
    for tag, a in zip(['w', 's0'], tables):
        if a.size <= GG.FULL_MAX:
            assert eq(a, g['%s|%s' % (name, tag)]), (name, tag)
        else:
            assert eq(a.reshape(-1)[:GG.HEAD], g['%s|%s|head' % (name, tag)]), (name, tag)
            assert eq(GG.GU.digest(a), g['%s|%s|sha256' % (name, tag)]), (name, tag)


@pytest.mark.parametrize("name", sorted(GG.CASES))
def test_restatement_matches_golden(golden, name):
    check(golden("group_adagrad"), name, *GG.run(GG.restate, GG.CASES[name]))


def test_fixture_is_order_sensitive(golden):
    """a warp-tree or pairwise sum of squares would fail the fixture: for every form, variant and
    L >= 32 some case differs from the sequential fold in each of the two orders"""
    groups = GG.check_order_sensitivity()
    assert len(groups) == 2 * 2 * (3 * 5 + 1)   # (tree, pairwise) x forms x (variants x L, 3-D)


@live
@pytest.mark.parametrize("name", sorted(GG.CASES))
def test_restatement_matches_live_reference(name):
    case = GG.CASES[name]
    t1, n1 = GG.run(GG.ref(), case)
    t2, n2 = GG.run(GG.restate, case)
    assert n1 == n2 and all(eq(a, b) for a, b in zip(t1, t2)), name


def random_case(seed):
    rng = np.random.default_rng(seed)
    wst = [GG.RSP, GG.DNS][seed % 2]
    params = dict(lr=float(rng.choice([0.1, 0.01, 0.37])), rescale_grad=float(rng.choice([1.0, 0.5, 1 / 96])))
    if rng.random() < 0.5:
        params['clip_gradient'] = float(rng.choice([0.0, 0.05, 0.7, 300.0]))
    if rng.random() < 0.5:
        params['epsilon'] = float(rng.choice([1e-7, 3.3e-07, 1e-3]))
    steps = int(rng.integers(1, 4))
    return dict(form='rsp' if wst == GG.RSP else 'dns', wstype=wst,
                shape=(int(rng.integers(3, 40)), int(rng.choice([1, 2, 7, 8, 16, 31, 64, 100, 513, 600]))),
                rowsets=[str(rng.choice(GG.ROWSETS)) for _ in range(steps)], params=params,
                empty=bool(wst == GG.RSP and rng.random() < 0.5))


@live
@pytest.mark.parametrize("seed", range(50))
def test_restatement_matches_live_reference_random(seed):
    """random form, table, row sets, steps and parameters (clip on / off / 0, rescale, epsilon)"""
    case = random_case(seed)
    t1, n1 = GG.run(GG.ref(), case, 'random%d' % seed)
    t2, n2 = GG.run(GG.restate, case, 'random%d' % seed)
    assert n1 == n2 and all(eq(a, b) for a, b in zip(t1, t2)), case


@live
def test_reference_refusals():
    """the reference's parser and dispatch, as compiled and restated in the oracle library, refuse
    what the GPU operator refuses: missing weight rows, a partial history, wd, a distinct out, the
    all-dense form, mixed storage types"""
    r, rows, L = GG.ref(), 4, 3
    g, ids = np.ones((1, L), np.float32), np.array([1])
    cases = [
        ([1, 1, 1], [rows - 1, 1, 0], True, {}, 'weights with all rows containing non-zeros'),
        ([1, 1, 1], [rows, 1, rows - 1], True, {}, 'states with all rows containing non-zeros'),
        ([1, 1, 1], [rows, 1, 0], True, {'wd': 0.0}, "Cannot find argument 'wd'"),
        ([1, 1, 1], [rows, 1, 0], False, {}, 'kWriteInplace'),
        ([0, 1, 0], [0, 1, 0], False, {}, 'kWriteInplace'),
        ([0, 0, 0], [0, 0, 0], True, {}, 'is not implemented for'),
        ([0, 1, 1], [0, 1, 0], True, {}, 'Operator not implemented'),
        ([1, 1, 0], [rows, 1, 0], True, {}, 'Operator not implemented'),
        ([1, 0, 1], [rows, 0, 0], True, {}, 'Operator not implemented'),
    ]
    for st, nnr, inplace, extra, msg in cases:
        bufs = [np.ones((rows, L), np.float32), g, np.ones((rows, 1), np.float32)]
        with pytest.raises(RuntimeError, match=msg):
            r(GG.OP, st, list(nnr), bufs, ids, rows, L, inplace, lr=0.1, **extra)


# ------------------------------------------------------------------ the tests/compat mirror
@live_py
def test_list_scheduler_matches_reference_factor_scheduler():
    with RPG.reference_python_group_adagrad() as (_, _, sched):
        s = sched.FactorScheduler(step=2, factor=0.5, base_lr=0.1)
        assert [s(n) for n in range(1, 5)] == [RPG.ListSched()(n) for n in range(1, 5)]


@live_py
@pytest.mark.parametrize("name", sorted(RPG.trajectory_cases()))
def test_compat_mirror_vs_reference(golden, name):
    from compat import mxnet_optimizer as B
    from compat import mxnet_optimizer_contrib as M
    case = RPG.trajectory_cases()[name]
    with RPG.reference_python_group_adagrad() as (opt, contrib, sched):
        RP.LOG[:] = []
        want = RPG.run_trajectory(opt, contrib.GroupAdaGrad, case,
                                  sched.FactorScheduler(step=2, factor=0.5, base_lr=0.1))
        want_log = list(RP.LOG)
        saved = [(m, dict(m.__dict__)) for m in (B, M)]
        try:
            for m in (B, M):
                m.__dict__.update(RP.op_table())
                m.__dict__.update(RPG.op_table())
            RP.LOG[:] = []
            got = RPG.run_trajectory(M, M.GroupAdaGrad, case, RPG.ListSched())
            got_log = list(RP.LOG)
        finally:
            for m, d in saved:
                m.__dict__.clear()
                m.__dict__.update(d)
    assert got_log == want_log and len(want_log) == 4 * len(case['shapes'])
    gold = golden("updater_trajectories_group_adagrad")
    for step, ((wg, hg), (ww, hw)) in enumerate(zip(got, want)):
        for k in range(len(wg)):
            assert eq(wg[k], ww[k]) and eq(ww[k], gold["%s_step%d_w%d" % (name, step, k)]), (name, step, k)
            assert eq(hg[k], hw[k]) and eq(hw[k], gold["%s_step%d_w%d_s0" % (name, step, k)]), (name, step, k)
    for k, s in enumerate(case['shapes']):        # rows no gradient lists keep their initial values
        cold = RPG.RPS.cold_rows(s)
        assert eq(want[-1][0][k][cold], case['w0'][k][cold])


def test_compat_group_adagrad_dense_gradient_is_refused():
    from compat import mxnet_optimizer_contrib as M
    opt = M.GroupAdaGrad(learning_rate=0.1)

    class Dense(M.NDArray):
        def __init__(self):
            pass
        stype = 'default'
    with pytest.raises(NotImplementedError, match='mean / square / clip / sqrt'):
        opt.update(0, Dense(), Dense(), None)


def test_ptxas_no_spills(tmp_path):
    """the four instantiations of rsp_group_adagrad_kernel (vector / scalar, one tile / longer rows)"""
    from anand_mxnet_b200 import build as B
    src = os.path.join(B.CSRC, "rowsparse_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o",
                                                     str(tmp_path / "r.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    blocks = re.split(r"Compiling entry function ", r.stderr)[1:]   # one per kernel
    found = [(b.split("'")[1],) + re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", b).groups()
             for b in blocks if re.match(r"'\w*rsp_group_adagrad_kernel", b)]
    assert len(found) == 4, r.stderr[-4000:]
    assert all(s == '0' and l == '0' for _, s, l in found), found
