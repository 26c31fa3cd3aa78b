"""Pins the numpy restatements that tests/test_update_ops_edges_gpu.py holds the kernels to, at the
inputs that file adds, to the reference's own CPU operators, bit for bit with NaN as NaN:

  * the dense operators (golden_update_ops.restate against oracle/_ref/libmxref_update.so) with
    special values in the weight, the gradient and every state, out as the weight and as a separate
    array; at every hyper-parameter edge of update_edges.HYPER; and mp_nag_mom_update's float16
    edges (overflow boundary, subnormals, a weight that disagrees with its master);
  * the row_sparse Ftrl / AdaGrad forms (golden_sparse_update_ops) and GroupAdaGrad
    (golden_group_adagrad) with special values in the gradient rows, the tables and the states;
  * the dense operators on a densified row_sparse gradient (absent rows read +0.0) with special
    values in the stored rows and in the weight and state rows the gradient does not store.

The reference has no bfloat16 CPU kernel: the float16 cases pin mp_nag's float32 part, and
to_bf16_bits is checked against torch's bfloat16 rounding. The launch constants the GPU test derives
its sizes from, and the sizes themselves, are checked here too. Skipped where oracle/_ref/ is not
built."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import golden_group_adagrad as GG  # noqa: E402
import golden_ndarray_ops as GN  # noqa: E402
import golden_sparse_update_ops as GS  # noqa: E402
import golden_update_ops as GU  # noqa: E402
import update_edges as E  # noqa: E402

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")

N = 1031
ANCHORS = [0, N // 2, N - E.WINDOW]
F = np.float32


@pytest.fixture(scope="module")
def ref():
    if GU.ref() is None:
        pytest.skip("oracle/_ref/libmxref_update.so is not built")
    return GU.ref()


def same(a, b):
    dt = 'float16' if a.dtype == np.float16 else 'float32'
    return GN.same(a, b, dt)


def check_dense(op, dtype, ins, params, distinct_out):
    case = dict(op=op, dtype=dtype, params=params, distinct_out=distinct_out)
    want_out, want_st = GU.run_ref(case, ins)
    out, st = GU.restate(op, ins, params, distinct_out, dtype)
    assert same(out, want_out), (op, 'out')
    for k, (a, b) in enumerate(zip(st, want_st)):
        assert same(a, b), (op, 's%d' % k)


def dense_cases():
    return [(op, 'float16' if op == 'mp_nag_mom_update' else 'float32') for op in GU.OPS]


# ------------------------------------------------------------------------------- dense operators
@pytest.mark.parametrize("distinct_out", [False, True], ids=['out_is_w', 'distinct_out'])
@pytest.mark.parametrize("op,dtype", dense_cases())
def test_special_values_match_reference(ref, op, dtype, distinct_out):
    """NaN, +-Inf, +-0 and +-1e-40 in every operand and state, under the golden variants' parameters
    and under every hyper-parameter edge"""
    variants = list(GU.VARIANTS[op].values()) + list(E.HYPER[op].values())
    for k, params in enumerate(variants):
        ins = E.special_inputs(op, N, dtype, ANCHORS, seed=k)
        check_dense(op, dtype, ins, params, distinct_out)


@pytest.mark.parametrize("op,dtype,name", [c for c in E.hyper_cases() if c[1] != 'bfloat16'])
def test_hyper_edges_match_reference(ref, op, dtype, name):
    ins, params = E.hyper_inputs(op, dtype, name, N)
    check_dense(op, dtype, ins, params, False)


def test_clip_edge_gradients_land_on_clip():
    """the clip_exact inputs reach exactly +-clip after rescaling, and values either side of it"""
    for op, dtype, name in E.hyper_cases():
        if name != 'clip_exact':
            continue
        p = E.HYPER[op][name]
        clip = GU.stof(p.get('clip_gradient', p.get('clip_grad')))
        g = E.clip_gradients(p, dtype)
        g = GU.bf16_bits_to_f32(g) if dtype == 'bfloat16' else g.astype(F)
        r = GU.stof(p['rescale_grad']) * g
        for s in (F(1), F(-1)):
            assert np.any(r == s * clip) and np.any(s * r > clip) and np.any(np.abs(r) < clip), (op, dtype)


def test_ftrl_z_at_lamda1_is_exact():
    """the g = 0 elements of the Ftrl edge inputs keep z at +-lamda1 through the step, on the edge of
    the strict |z| > lamda1 (there the quotient's numerator sgn*lamda1 - z is exactly +0, so > and
    >= give the same bits; the inputs still pin the result at the edge)"""
    for name, params in E.HYPER['ftrl_update'].items():
        ins, params = E.hyper_inputs('ftrl_update', 'float32', name, N)
        _, (z, _) = GU.restate('ftrl_update', ins, params)
        lam = GU.stof(params['lamda1'])
        hit = (ins[1] == 0) & (np.abs(ins[2]) == lam)
        assert hit.sum() >= 4 and np.array_equal(z[hit], ins[2][hit]), name


def test_rmspropalex_negative_variance_present():
    ins = E.dense_inputs('rmspropalex_update', N)
    _, st = GU.restate('rmspropalex_update', ins, E.HYPER['rmspropalex_update']['clip_exact'])
    assert np.isnan(st[2]).sum() >= N // 20


def test_mp_nag_float16_edges_match_reference(ref):
    """the float16 overflow boundary and subnormals, with a weight that disagrees with its master"""
    ins = E.mp_edge_inputs(N, 'float16', ANCHORS)
    assert np.all(ins[0] != ins[3].astype(np.float16))
    for distinct_out in (False, True):
        check_dense('mp_nag_mom_update', 'float16', [a.copy() for a in ins], E.MP_EDGE_PARAMS, distinct_out)
    out, _ = GU.restate('mp_nag_mom_update', ins, E.MP_EDGE_PARAMS)
    lo = ANCHORS[0]
    assert [float(x) for x in out[lo:lo + 4]] == [65504.0, 65504.0, 65504.0, np.inf]
    for name, params in E.HYPER['mp_nag_mom_update'].items():
        ins = E.mp_edge_inputs(N, 'float16', ANCHORS)
        check_dense('mp_nag_mom_update', 'float16', ins, params, False)


def test_to_bf16_bits_matches_torch():
    """round to nearest even on ties (normal, overflow, subnormal), NaN and overflow, as torch rounds"""
    torch = pytest.importorskip("torch")
    x = np.concatenate([E.MASTER_EDGES, np.array([3.4028235e38, -3.4028235e38, 1.0, -2.5], F),
                        np.random.default_rng(0).standard_normal(4096).astype(F)])
    want = torch.from_numpy(x.copy()).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    got = GU.to_bf16_bits(x)
    nan = np.isnan(x)
    assert np.array_equal(got[~nan], want[~nan])
    assert np.all((got[nan] & 0x7FFF) > 0x7F80) and np.all((want[nan] & 0x7FFF) > 0x7F80)
    assert GU.to_bf16_bits(E._bits(0x7F7F8000))[0] == 0x7F80       # the overflow tie rounds to +Inf


# --------------------------------------------------------------------------- row_sparse forms
@pytest.fixture(scope="module")
def sparse_ref():
    if GS.ref() is None:
        pytest.skip("oracle/_ref/libmxref_sparse_update.so is not built")
    return GS.ref()


@pytest.mark.parametrize("L", [4, 5])
@pytest.mark.parametrize("form", sorted(GS.FORMS))
def test_rsp_forms_special_values_match_reference(sparse_ref, form, L):
    op, wst = GS.FORMS[form]
    rows = 37
    tables, ids, g = E.rsp_tables(form, rows, L, 15, seed=L)
    got = {}
    for fn in (sparse_ref, GS.restate):
        t = [a.copy() for a in tables]
        nnr = [rows if wst == GS.RSP else 0, len(ids)] + [rows if wst == GS.RSP else 0] * (len(t) - 1)
        fn(op, [wst, GS.RSP] + [wst] * (len(t) - 1), nnr, [t[0], g.copy()] + t[1:], ids, rows, L, True,
           **E.RSP_PARAMS[form])
        got[fn is sparse_ref] = t
    for a, b in zip(got[True], got[False]):
        assert GN.same(a, b, 'float32'), form


@pytest.fixture(scope="module")
def ga_ref():
    if GG.ref() is None:
        pytest.skip("oracle/_ref/libmxref_group_adagrad.so is not built")
    return GG.ref()


@pytest.mark.parametrize("L", [4, 5, 40, 1000])
@pytest.mark.parametrize("wst", [GG.DNS, GG.RSP], ids=['dns', 'rsp'])
def test_group_adagrad_special_values_match_reference(ga_ref, wst, L):
    rows = 29
    w, h, ids, g = E.ga_tables(rows, L, 12, seed=L)
    got = {}
    for fn in (ga_ref, GG.restate):
        ww, hh = w.copy(), h.copy()
        nnr = [rows if wst == GG.RSP else 0, len(ids), rows if wst == GG.RSP else 0]
        fn(GG.OP, [wst, GG.RSP, wst], nnr, [ww, g.copy(), hh], ids, rows, L, True, **E.GA_PARAMS)
        got[fn is ga_ref] = (ww, hh)
    for a, b in zip(got[True], got[False]):
        assert GN.same(a, b, 'float32'), (wst, L)
    assert np.isnan(got[True][1][ids]).any()


@pytest.mark.parametrize("L", [2, 4, 6])
@pytest.mark.parametrize("op", [op for op in GU.OPS if op != 'mp_nag_mom_update'])
def test_rsp_grad_special_values_match_reference(ref, op, L):
    rows = 41
    ids = E.pick_ids(np.random.default_rng(L), rows, 13)
    w, g, states = E.rspg_inputs(op, rows, L, ids, seed=L)
    dense = E.densify((rows, L), ids, g)
    for params in list(GU.VARIANTS[op].values())[-1:] + list(E.HYPER[op].values()):
        ins = [w.reshape(-1), dense.reshape(-1)] + [s.reshape(-1) for s in states]
        check_dense(op, 'float32', [a.copy() for a in ins], params, False)


# ----------------------------------------------------------------------------- launch geometry
def test_launch_constants_and_sizes():
    """the constants are found once each in the kernels' source, and every size the GPU test runs
    sits where it is meant to: the wrap sizes past one full pass with a tail, GroupAdaGrad's row
    counts past one pass of its warps"""
    c = E.C
    assert c['kNumSMs'] == 132 and E.UPDATE_THREADS == c['kNumSMs'] * c['update_cap'] * c['kThreads']
    for V in (4, 8):
        n = E.wrap_size(V)
        assert E.UPDATE_THREADS < n // V < 2 * E.UPDATE_THREADS and n % V != 0
        assert sorted(E.small_sizes(V)) == list(range(V - 1, V + 2)) + list(range(2 * V, 3 * V))
    assert E.GA_WARPS == c['kNumSMs'] * c['ga_cap'] * c['kWarpsPerBlock']
    assert 5 <= E.GA_TILE < 1000
