"""The dense-gradient AdaGrad / GroupAdaGrad operators without a GPU: their table in csrc/reduce_ops.cc
follows the operator-table rules, the numpy restatement (oracle/golden_dense_adagrad.py) equals
tests/golden/dense_adagrad_ops.npz and the reference's own code, a naive, a pairwise and a warp-tree
fold of the mean each miss the fixture, the oracle reproduces
tests/golden/updater_trajectories_dense_adagrad.npz from the reference's unmodified classes, the
tests/compat mirror issues those classes' operator sequence and reaches their results, and the
row-mean kernels compile for sm_90a without spills."""
import ctypes
import inspect
import os
import re
import subprocess

import numpy as np
import pytest

import golden_dense_adagrad as GD
import golden_ndarray_ops as GN
import ref_python as RP
import ref_python_dense_adagrad as RPD
from test_op_table_host import CSRC, source

live = pytest.mark.skipif(GD.ref() is None, reason="needs oracle/_ref/libmxref_dense_adagrad.so")
live_py = pytest.mark.skipif(not RPD.available(), reason="needs /root/reference and oracle/_ref/ libraries")

OPERATORS = ["square", "mean"]


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


# ------------------------------------------------------------------------------ operator table
def test_operators_resolve_and_the_table_holds_them():
    import anand_mxnet_b200 as mx
    h = ctypes.c_void_p()
    for name in OPERATORS:
        assert mx.base._LIB.NNGetOpHandle(name.encode(), ctypes.byref(h)) == 0 and h.value, name
    rows = re.findall(r'\{"([^"]+)",\s*\w+,', source("reduce_ops.cc"))
    assert rows == OPERATORS


def test_reduce_handlers_follow_the_table_rules():
    """test_op_table_host.py's rules on reduce_ops.cc: no handler looks at its name, the shared
    helpers and the unknown-key wording are not defined again, the elementwise kernel is reached
    through Elementwise / ElementwiseRows only"""
    for f in ("reduce_ops.cc", "arith_ops.cc"):
        src = source(f)
        for pat in (r'\bn\s*[!=]=\s*"', r'\bname\s*[!=]=\s*"', r'\.find\("_', r'\.rfind\("', r'\bn\[0\]',
                    r'strn?cmp\(', r'op\.name\s*[!=]='):
            assert not re.search(pat, src), (f, pat)
        for helper in ("Required", "OutOr", "InPlace", "RejectUnknownKeys", "Elementwise", "StodD",
                       "ElementwiseRows"):
            pat = re.compile(r"^[A-Za-z][\w:<>,*& ]*?\b%s\([^;{}]*\)\s*\{" % helper, re.M)
            assert not pat.search(src), (f, helper)
        assert '"Cannot find argument' not in src
        assert "LaunchElementwise" not in src
    assert len(re.findall(r"^void ElementwiseRows\(", source("ops.cc"), re.M)) == 1


def test_python_binding():
    import anand_mxnet_b200 as mx
    for f in ("square", "mean"):
        assert callable(getattr(mx.nd, f)), f
    assert 'mean' in mx.nd.NDArray.__dict__
    assert list(inspect.signature(mx.nd.mean).parameters) == ['data', 'axis', 'keepdims', 'exclude', 'out']


# ------------------------------------------------------------------------------ fixture
@pytest.fixture(scope="module")
def fixture():
    d = np.load(os.path.join(GD.GOLD, "dense_adagrad_ops.npz"))
    return {str(n): (s, h) for n, s, h in zip(d['names'], d['sha256'], d['head'])}


def test_fixture_covers_every_case_and_operator(fixture):
    cases = GD.all_cases()
    assert sorted(fixture) == sorted(c[0] for _, c in cases)
    for dt in GD.DTYPES:
        assert any(k == 'square' and c[1] == dt for k, c in cases), dt
        for op in GD.BINARY:
            if op == 'broadcast_div' and dt not in GD.FLOATS:
                continue
            assert any(k == 'broadcast' and c[1] == op and c[2] == dt for k, c in cases), (op, dt)
    means = [c for k, c in cases if k == 'mean']
    for dt in GD.FLOATS:
        mine = [c for c in means if c[1] == dt]
        cols = {c[2][-1] for c in mine}
        assert {1, 2, 31, 32, 33, GD.TILE - 1, GD.TILE + 1, 2 * GD.TILE + 1} <= cols and max(cols) > 1000
        assert any(int(np.prod(c[2][:-1])) > GD.WAVE for c in mine)
        assert any(len(c[2]) == 3 for c in mine)
        assert {c[3] for c in mine} >= {'1', '-1', '(1,)', '(-1,)'}
        assert {c[4] for c in mine} == {'True', 'False'}
        assert {c[5] for c in mine} >= {'mixed', 'inf', 'nan'}


def test_restatement_matches_fixture(fixture):
    for kind, case in GD.all_cases():
        dt = GD.out_dtype(kind, case)
        got = np.ravel(GD.restate(kind, case))
        sha, head = fixture[case[0]]
        assert np.array_equal(GN.sha256(got, dt), sha) and np.array_equal(GN.head_bytes(got, dt), head), case[0]


def test_restatement_edges():
    """the choices the fixture pins, spelled out"""
    # an integer squares through float: 4097^2 = 16785409 is not a float
    assert GD.square(np.array([4097, 46340], np.int32), 'int32').tolist() == [16785408, 2147395584]
    assert GD.square(np.array([300.0], np.float16), 'float16')[0] == np.inf
    # a single -0.0 folds to +0.0 (0 + -0 = +0)
    m = GD.mean_rows(np.array([[-0.0]], np.float32), 'float32')
    assert m.view(np.uint32).tolist() == [0]
    # the count rounds to the dtype: bfloat16(4099) is 4096
    x = np.full((1, 4099), 0x3F80, np.uint16)   # bfloat16 ones
    s = GD.row_fold_kahan(x, 'bfloat16')
    assert GN.bf16_to_f32(GD.mean_rows(x, 'bfloat16'))[0] == GN.bf16_to_f32(GN.bf16_from_f32(s / np.float32(4096)))[0]
    # inf mid-row resets the residual: inf stays inf after a finite tail
    assert GD.mean_rows(np.array([[1.0, 3e38, 3e38, 1.0]], np.float32), 'float32')[0] == np.inf


@pytest.mark.parametrize("fold", sorted(GD.FOLDS))
def test_other_folds_miss_the_fixture(fixture, fold):
    """a naive, a pairwise and a warp-tree fold each give other bits than the reference's on some
    case of every dtype"""
    for dt in GD.FLOATS:
        missed = 0
        for kind, case in GD.all_cases():
            if kind != 'mean' or case[1] != dt:
                continue
            x = GD.inputs(kind, case)[0]
            got = np.ravel(GD.mean_rows(x, dt, GD.FOLDS[fold]))
            missed += not np.array_equal(GN.sha256(got, dt), fixture[case[0]][0])
        assert missed > 0, (fold, dt)


@live
def test_restatement_matches_live_reference():
    for kind, case in GD.all_cases():
        dt = GD.out_dtype(kind, case)
        if dt == 'bfloat16':
            continue
        assert GN.same(GD.live(kind, case), GD.restate(kind, case), dt), case[0]


@live
def test_mean_parameters_match_live_reference():
    """axis spellings and keepdims as ReduceAxesParam parses them, and the shape it gives"""
    x = GD.mean_operand('p', 'float32', (3, 4, 5), 'mixed')
    want = GD.mean_rows(x, 'float32')
    for axis in ('2', '-1', '(2,)', '(-1,)', '[2]'):
        for keep, shape in (('True', (3, 4, 1)), ('False', (3, 4)), ('0', (3, 4)), ('1', (3, 4, 1))):
            got = GD.ref().mean(x, 'float32', axis=axis, keepdims=keep)
            assert got.shape == shape and eq(got.reshape(3, 4), want), (axis, keep)


# ------------------------------------------------------------------------------ trajectories
@live_py
def test_oracle_reproduces_trajectory_fixture(golden):
    gold = golden("updater_trajectories_dense_adagrad")
    names = set()
    with RPD.reference_python_dense_adagrad() as (opt, contrib):
        for name, case in RPD.trajectory_cases().items():
            ws, hs = RPD.run_trajectory(opt, RPD.classes(opt, contrib)[case['opt'][0]], case)
            for step in range(4):
                for k in range(len(case['shapes'])):
                    key = "%s_step%d_w%d" % (name, step, k)
                    names.update([key, key + "_s0"])
                    assert eq(ws[step][k], gold[key]), key
                    assert eq(hs[step][k], gold[key + "_s0"]), key
    assert names == set(gold.files)


def test_trajectory_cases_cover_every_option():
    cases = RPD.trajectory_cases()
    ada = [c for c in cases.values() if c['opt'][0] == 'AdaGrad']
    kws = [c['opt'][1] for c in ada]
    assert any('clip_gradient' not in kw for kw in kws) and any(kw.get('clip_gradient') for kw in kws)
    assert any(kw.get('clip_gradient', 1) == 0 for kw in kws)
    assert any(kw.get('wd') for kw in kws) and any(not kw.get('wd') for kw in kws)
    assert any(kw.get('rescale_grad', 1) != 1 for kw in kws)
    assert any(kw.get('multi_precision') and c['dtype'] == 'float16' for kw, c in zip(kws, ada))
    assert {len(s) for s in ada[0]['shapes']} >= {1, 2, 4}
    group = [c for c in cases.values() if c['opt'][0] == 'GroupAdaGrad']
    assert any('clip_gradient' in c['opt'][1] for c in group)
    assert any('clip_gradient' not in c['opt'][1] for c in group)
    cols = {s[1] for c in group for s in c['shapes']}
    assert 1 in cols and max(cols) > GD.TILE


def _mirror():
    """tests/compat/mxnet_optimizer_dense_adagrad.py (and the modules of its base classes) with the
    operator functions they import replaced by the harness's, so that both front-ends run the
    reference's operators"""
    from compat import mxnet_optimizer as B
    from compat import mxnet_optimizer_contrib as C
    from compat import mxnet_optimizer_dense_adagrad as M
    from compat import mxnet_optimizer_sparse as S
    saved = [(m, dict(m.__dict__)) for m in (B, C, S, M)]
    for m in (B, C, S, M):
        m.__dict__.update(RPD.op_table())
    return M, saved


@live_py
@pytest.mark.parametrize("name", sorted(RPD.trajectory_cases()))
def test_compat_mirror_vs_reference(name):
    """the mirror issues the reference class's operators with the same parameter strings, in the
    same order, and reaches the same weights and histories"""
    case = RPD.trajectory_cases()[name]
    cls = case['opt'][0]
    with RPD.reference_python_dense_adagrad() as (opt, contrib):
        RP.LOG[:] = []
        want = RPD.run_trajectory(opt, RPD.classes(opt, contrib)[cls], case)
        want_log = list(RP.LOG)
        M, saved = _mirror()
        try:
            RP.LOG[:] = []
            got = RPD.run_trajectory(M, getattr(M, cls), case)
            got_log = list(RP.LOG)
        finally:
            for m, d in saved:
                m.__dict__.clear()
                m.__dict__.update(d)
    assert got_log == want_log and len(want_log) > 0
    assert any(op == 'square' for op, _ in want_log)
    for part in range(2):
        for step, (a_s, b_s) in enumerate(zip(got[part], want[part])):
            for k, (a, b) in enumerate(zip(a_s, b_s)):
                assert eq(a, b), (name, part, step, k)


@live_py
def test_compat_mirror_signatures_match_reference():
    """same constructor arguments and defaults as the reference's classes, and the methods (the
    bodies are held by test_compat_mirror_vs_reference)"""
    import ast
    from compat import mxnet_optimizer_dense_adagrad as M

    def ref_sig(path, cls):
        tree = ast.parse(open(path).read())
        node = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls][0]
        init = [f for f in node.body if isinstance(f, ast.FunctionDef) and f.name == '__init__'][0]
        return ([a.arg for a in init.args.args], [ast.literal_eval(d) for d in init.args.defaults],
                init.args.kwarg.arg if init.args.kwarg else None)

    def my_sig(cls):
        ps = list(inspect.signature(cls.__init__).parameters.values())
        return ([p.name for p in ps if p.kind == p.POSITIONAL_OR_KEYWORD],
                [p.default for p in ps if p.kind == p.POSITIONAL_OR_KEYWORD and p.default is not p.empty],
                next((p.name for p in ps if p.kind == p.VAR_KEYWORD), None))
    paths = {'AdaGrad': os.path.join(RP.REF_PY, "optimizer", "optimizer.py"),
             'GroupAdaGrad': os.path.join(RP.REF_PY, "optimizer", "contrib.py")}
    for cls in RPD.CLASSES:
        assert my_sig(getattr(M, cls)) == ref_sig(paths[cls], cls), cls
        for meth in ('create_state', 'update'):
            assert callable(getattr(getattr(M, cls), meth)), (cls, meth)


def test_mirror_classes_are_not_registered():
    """the registry keeps the row_sparse mirrors under the names AdaGrad and GroupAdaGrad"""
    from compat import mxnet_optimizer as B
    from compat import mxnet_optimizer_contrib as C
    from compat import mxnet_optimizer_dense_adagrad as M
    from compat import mxnet_optimizer_sparse as S
    reg = B.Optimizer.opt_registry
    assert reg['adagrad'] is S.AdaGrad and reg['groupadagrad'] is C.GroupAdaGrad
    assert M.AdaGrad not in reg.values() and M.GroupAdaGrad not in reg.values()


def test_ptxas_no_spills(tmp_path):
    from anand_mxnet_b200 import build as B
    src = os.path.join(CSRC, "reduce_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o",
                                                     str(tmp_path / "r.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    assert len(re.findall(r"Compiling entry function '\w*row_mean_kernel\w*' for 'sm_90a'", r.stderr)) == 4
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) == 4 and all(s == ('0', '0') for s in spills), spills
