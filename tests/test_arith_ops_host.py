"""The Adamax / Nadam / AdaDelta arithmetic operators without a GPU: their table in csrc/arith_ops.cc
follows the operator-table rules, the numpy restatement (oracle/golden_arith_ops.py) equals
tests/golden/arith_ops.npz and the reference's own functors, the oracle reproduces
tests/golden/updater_trajectories_arith.npz from the reference's unmodified optimizer classes, the
tests/compat mirror issues those classes' operator sequence and reaches their results, and the
elementwise kernels compile for sm_90a without spills."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import golden_arith_ops as GA
import golden_ndarray_ops as GN
import ref_python as RP
import ref_python_arith as RPA
from test_op_table_host import CSRC, source

live = pytest.mark.skipif(GA.ref() is None, reason="needs oracle/_ref/libmxref_arith.so")
live_py = pytest.mark.skipif(not RPA.available(), reason="needs /root/reference and oracle/_ref/ libraries")

OPERATORS = ["broadcast_add", "broadcast_sub", "broadcast_mul", "broadcast_div", "broadcast_maximum",
             "_div_scalar", "abs", "clip"]


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


# ------------------------------------------------------------------------------ operator table
def test_operators_resolve_and_the_table_holds_them():
    import anand_mxnet_b200 as mx
    h = ctypes.c_void_p()
    for name in OPERATORS:
        assert mx.base._LIB.NNGetOpHandle(name.encode(), ctypes.byref(h)) == 0 and h.value, name
    rows = re.findall(r'\{"([^"]+)",\s*\w+,', source("arith_ops.cc"))
    assert rows == OPERATORS


def test_arith_handlers_follow_the_table_rules():
    """test_op_table_host.py's rules on arith_ops.cc: no handler looks at its name, the shared
    helpers and the unknown-key wording are not defined again, the kernel is reached through the
    one Elementwise"""
    src = source("arith_ops.cc")
    for pat in (r'\bn\s*[!=]=\s*"', r'\bname\s*[!=]=\s*"', r'\.find\("_', r'\.rfind\("', r'\bn\[0\]',
                r'strn?cmp\(', r'op\.name\s*[!=]='):
        assert not re.search(pat, src), pat
    for helper in ("Required", "OutOr", "InPlace", "RejectUnknownKeys", "Elementwise", "StodD"):
        pat = re.compile(r"^[A-Za-z][\w:<>,*& ]*?\b%s\([^;{}]*\)\s*\{" % helper, re.M)
        assert not pat.search(src), helper
    assert '"Cannot find argument' not in src
    assert "LaunchElementwise" not in src
    assert len(re.findall(r"^void Elementwise\(", source("ops.cc"), re.M)) == 1


def test_python_binding():
    import anand_mxnet_b200 as mx
    for f in ("clip", "abs", "maximum", "sqrt"):
        assert callable(getattr(mx.nd, f)), f
    for m in ("__truediv__", "__itruediv__"):
        assert m in mx.nd.NDArray.__dict__, m


# ------------------------------------------------------------------------------ fixture
@pytest.fixture(scope="module")
def fixture():
    d = np.load(os.path.join(GA.GOLD, "arith_ops.npz"))
    return {str(n): (s, h) for n, s, h in zip(d['names'], d['sha256'], d['head'])}


def test_fixture_covers_every_case_and_operator(fixture):
    cases = GA.all_cases()
    assert sorted(fixture) == sorted(c[0] for _, c in cases)
    ops = {c[0].split('|')[0] for _, c in cases}
    assert ops == set(OPERATORS)
    for dt in GA.DTYPES:
        for op in OPERATORS:
            if op in GA.DIVIDES and dt not in GA.FLOATS:
                continue
            assert any(c[0].startswith('%s|%s|' % (op, dt)) for _, c in cases), (op, dt)


def test_restatement_matches_fixture(fixture):
    for kind, case in GA.all_cases():
        dt = GA.out_dtype(kind, case)
        got = GA.restate(kind, case)
        sha, head = fixture[case[0]]
        assert np.array_equal(GN.sha256(got, dt), sha) and np.array_equal(GN.head_bytes(got, dt), head), case[0]


def test_restatement_edges():
    """the choices the fixture pins, spelled out"""
    f32 = np.float32
    got = GA.maximum(np.array([-0.0, 0.0, np.nan, 1.0], f32), np.array([0.0, -0.0, 1.0, np.nan], f32), 'float32')
    assert got.view(np.uint32).tolist()[:2] == [0, 0x80000000] and np.isnan(got[2]) and np.isnan(got[3])
    got = GA.clip(np.array([-1.0, 1.0, -0.0, np.nan], f32), '-0.0', '0.0', 'float32')
    assert got.view(np.uint32).tolist()[:3] == [0x80000000, 0, 0x80000000] and np.isnan(got[3])
    # an integer compares with the bound in float: 16777217 is not above 16777216.0
    got = GA.clip(np.array([16777217, 16777218, -16777218], np.int32), '-16777216.0', '16777216.0', 'int32')
    assert got.tolist() == [16777217, 16777216, -16777216]
    # an int64 takes abs through double
    assert GA.absolute(np.array([-(2 ** 53 + 1)], np.int64), 'int64').tolist() == [2 ** 53]
    got = GA.div(np.array([1.0, -1.0, 0.0], f32), np.array([0.0, 0.0, 0.0], f32), 'float32')
    assert got[0] == np.inf and got[1] == -np.inf and np.isnan(got[2])


@live
def test_restatement_matches_live_reference():
    for kind, case in GA.all_cases():
        dt = GA.out_dtype(kind, case)
        if dt == 'bfloat16' or (kind == 'array' and case[3] > 5000):
            continue
        assert GN.same(GA.live(kind, case), GA.restate(kind, case), dt), case[0]


@live
def test_scalar_and_bound_parses_match_live_reference():
    a = np.ones(1, np.float32)
    for s in GN._differing_parses()[:40] + GN.EXTRA_SCALARS:
        parsed, _ = GA.ref().div_scalar(a, s, 'float32')
        assert parsed == float(s), s
    for lo, hi in GA.CLIP_BOUNDS + [('0.1', '1e-08'), ('-3.7', '123456.789')]:
        parsed, _ = GA.ref().clip(a, lo, hi, 'float32')
        want = GA.clip_bounds(lo, hi)
        assert parsed.view(np.uint32).tolist() == np.array(want, np.float32).view(np.uint32).tolist(), (lo, hi)


# ------------------------------------------------------------------------------ trajectories
@live_py
def test_oracle_reproduces_trajectory_fixture(golden):
    gold = golden("updater_trajectories_arith")
    with RPA.reference_python_arith() as (opt, _):
        names = set()
        for name, case in RPA.trajectory_cases().items():
            ws, gs = RPA.run_trajectory(opt, case)
            for step in range(4):
                for k in range(len(case['shapes'])):
                    names.add("%s_step%d_w%d" % (name, step, k))
                    assert eq(ws[step][k], gold["%s_step%d_w%d" % (name, step, k)]), (name, step, k)
                    if case['opt'][0] == 'AdaDelta':
                        names.add("%s_step%d_g%d" % (name, step, k))
                        assert eq(gs[step][k], gold["%s_step%d_g%d" % (name, step, k)]), (name, step, k)
    assert names == set(gold.files)


def test_trajectory_cases_cover_every_option():
    cases = RPA.trajectory_cases()
    for cls in RPA.CLASSES:
        mine = [c['opt'][1] for c in cases.values() if c['opt'][0] == cls]
        assert any('clip_gradient' not in kw for kw in mine), cls
        assert any(kw.get('clip_gradient') for kw in mine), cls
        assert any(kw.get('wd') for kw in mine) and any(not kw.get('wd') for kw in mine), cls
        assert any(kw.get('multi_precision') for kw in mine), cls
    assert any(c['opt'][1].get('clip_gradient', 1) == 0 for c in cases.values())


def _mirror():
    """tests/compat/mxnet_optimizer_arith.py (and its base class module) with the operator functions
    they import replaced by the harness's, so that both front-ends run the reference's operators"""
    from compat import mxnet_optimizer as B
    from compat import mxnet_optimizer_arith as M
    saved = [(m, dict(m.__dict__)) for m in (B, M)]
    for m in (B, M):
        m.__dict__.update(RPA.op_table())
    return M, saved


@live_py
@pytest.mark.parametrize("name", sorted(RPA.trajectory_cases()))
def test_compat_mirror_vs_reference(name):
    """the mirror issues the reference class's operators with the same parameter strings, in the
    same order, and reaches the same weights, gradients and states"""
    case = RPA.trajectory_cases()[name]
    with RPA.reference_python_arith() as (opt, _):
        RP.LOG[:] = []
        want = RPA.run_trajectory(opt, case)
        want_log = list(RP.LOG)
        M, saved = _mirror()
        try:
            RP.LOG[:] = []
            got = RPA.run_trajectory(M, case)
            got_log = list(RP.LOG)
        finally:
            for m, d in saved:
                m.__dict__.clear()
                m.__dict__.update(d)
    assert got_log == want_log and len(want_log) > 0
    for part in range(2):
        for step, (a_s, b_s) in enumerate(zip(got[part], want[part])):
            for k, (a, b) in enumerate(zip(a_s, b_s)):
                assert eq(a, b), (name, part, step, k)


@live_py
def test_compat_mirror_signatures_match_reference():
    """same classes, constructor defaults and methods as the reference's (the bodies are held by
    test_compat_mirror_vs_reference)"""
    import ast
    from compat import mxnet_optimizer_arith as M
    path = os.path.join(RP.REF_PY, "optimizer", "optimizer.py")

    def sig(tree, cls):
        node = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls][0]
        init = [f for f in node.body if isinstance(f, ast.FunctionDef) and f.name == '__init__'][0]
        return ([ast.unparse(b) for b in node.bases], [ast.unparse(d) for d in node.decorator_list],
                [a.arg for a in init.args.args], [ast.unparse(d) for d in init.args.defaults],
                init.args.kwarg.arg if init.args.kwarg else None)
    ref_tree = ast.parse(open(path).read())
    mine_tree = ast.parse(open(M.__file__).read())
    for cls in RPA.CLASSES:
        assert sig(mine_tree, cls) == sig(ref_tree, cls), cls
        for meth in ('create_state', 'update'):
            assert callable(getattr(getattr(M, cls), meth)), (cls, meth)


def test_ptxas_no_spills(tmp_path):
    from anand_mxnet_b200 import build as B
    src = os.path.join(CSRC, "misc_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o",
                                                     str(tmp_path / "m.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    assert len(re.findall(r"Compiling entry function '\w*ew_kernel\w*' for 'sm_90a'", r.stderr)) == 6
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) >= 6 and all(s == ('0', '0') for s in spills), spills
