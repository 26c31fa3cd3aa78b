"""The NAG / Signum / RMSProp / FTML / Ftrl / AdaGrad / GroupAdaGrad operators on the GPU at the
edges of their three kernels, bit for bit (NaN as NaN) against the numpy restatements, computed at
run time, that tests/test_update_ops_edges_host.py pins to the reference's operators:

  * update_kernel (dense, and the row_sparse-gradient pass): 16-byte groups (V = 4 float32 or 8
    16-bit elements) in a grid-stride loop whose grid is capped, then a scalar tail. Sizes V-1, V,
    V+1, 2V+k for every tail k, and a body past one full stride of the capped grid with a tail, on
    the vector and on the scalar path; one operand at a time misaligned by one element or by 8
    bytes; out as the weight and as a separate array; special values in the body, the tail and
    across the wrap; every hyper-parameter edge; mp_nag_mom_update's 16-bit edges;
  * rsp_row_update_kernel (row_sparse Ftrl / AdaGrad) on tables of tens of thousands of rows, and
    the dense-table AdaGrad on misaligned table views;
  * rsp_group_adagrad_kernel with more gradient rows than its capped grid has warps, on each of
    its variants (vector one-tile, scalar one-tile, multi-tile).

The launch constants come from the kernels' source (oracle/update_edges.py), so the sizes follow a
retuned cap."""
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

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]

F = np.float32
OPS = [op for op in GU.OPS if op != 'mp_nag_mom_update']
OP_DTYPES = [(op, 'float32') for op in OPS] + [('mp_nag_mom_update', 'float16'), ('mp_nag_mom_update', 'bfloat16')]


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200
    return anand_mxnet_b200


def same(a, b, dt):
    if dt == 'float16':
        a, b = np.asarray(a).view(np.float16), np.asarray(b).view(np.float16)
    return GN.same(np.ascontiguousarray(a).reshape(-1), np.ascontiguousarray(b).reshape(-1), dt)


def up(mx, a, dt, offset=0):
    """a GPU array holding `a`; offset > 0: a view `offset` elements into a larger array"""
    pad = np.zeros(offset, a.dtype)
    full = np.concatenate([pad, a.reshape(-1)])
    if dt == 'bfloat16':
        nd = mx.nd.array(GU.bf16_bits_to_f32(full), mx.gpu(0), 'bfloat16')
    else:
        nd = mx.nd.array(full, mx.gpu(0), full.dtype)
    return nd[offset:offset + a.size] if offset else nd


def down(nd, dt):
    a = nd.asnumpy().reshape(-1)
    return GU.to_bf16_bits(a) if dt == 'bfloat16' else a


def run_dense(mx, op, dtype, ins, params, offsets=None, distinct_out=False):
    """the operator on GPU copies of ins ([w, g, states...]); offsets: {'w'|'g'|'out'|'s<k>': elements}.
    Returns (out, states) from the GPU, and checks that a separate out left the weight as it was."""
    offsets = offsets or {}
    dts = E.operand_dtypes(op, dtype)
    keys = ['w', 'g'] + ['s%d' % k for k in range(len(ins) - 2)]
    nds = [up(mx, a, dt, offsets.get(k, 0)) for a, dt, k in zip(ins, dts, keys)]
    if distinct_out:
        out = up(mx, np.zeros_like(ins[0]), dtype, offsets.get('out', 0))
    else:
        out = nds[0]
    getattr(mx.nd, op)(*nds, out=out, **params)
    if distinct_out:
        assert same(down(nds[0], dtype), ins[0], dtype), 'the weight must stay untouched'
    return down(out, dtype), [s.asnumpy().reshape(-1) for s in nds[2:]]


def check_dense(mx, op, dtype, ins, params, what, **kw):
    got_out, got_st = run_dense(mx, op, dtype, ins, params, **kw)
    out, st = GU.restate(op, ins, params, kw.get('distinct_out', False), dtype)
    assert same(got_out, out, dtype), (what, 'out')
    for k, (a, b) in enumerate(zip(got_st, st)):
        assert same(a, b, 'float32'), (what, 's%d' % k)
    return got_out, got_st


def plain_params(op):
    return GU.VARIANTS[op][sorted(v for v in GU.VARIANTS[op] if v.startswith('clip_wd'))[-1]]


# ---------------------------------------------------------------------------------- dense sizes
def size_cases():
    out = []
    for op, dt in OP_DTYPES:
        V = E.vec_width(dt)
        for n in E.small_sizes(V) + [E.wrap_size(V)]:
            out.append(pytest.param(op, dt, n, id='%s-%s-%d' % (op, dt, n)))
    return out


@pytest.mark.parametrize("op,dtype,n", size_cases())
def test_dense_sizes(mx, op, dtype, n):
    """vector body and scalar tail at every tail length, and past one grid stride; the wrap size
    also on the scalar path (every operand one element into its allocation)"""
    ins = E.dense_inputs(op, n, dtype)
    params = plain_params(op)
    check_dense(mx, op, dtype, ins, params, 'aligned')
    if n == E.wrap_size(E.vec_width(dtype)):
        offs = {k: 1 for k in ['w', 'g'] + ['s%d' % k for k in range(len(ins) - 2)]}
        check_dense(mx, op, dtype, ins, params, 'scalar path', offsets=offs)


# ------------------------------------------------------------------------------------ alignment
def align_cases():
    out = []
    for op, dt in OP_DTYPES:
        operands = ['w', 'w_only', 'g', 'out'] + ['s%d' % k for k in range(GU.N_STATES[op])]
        for which in operands:
            for unit in ('elem', '8B'):
                out.append(pytest.param(op, dt, which, unit, id='%s-%s-%s-%s' % (op, dt, which, unit)))
    return out


@pytest.mark.parametrize("op,dtype,which,unit", align_cases())
def test_dense_one_operand_misaligned(mx, op, dtype, which, unit):
    """one operand off a 16-byte boundary (by one element, or by 8 bytes) moves the whole tensor to
    the scalar path with the aligned result, bit for bit. 'w' misaligns the weight that is also
    out, 'w_only' the weight beside an aligned separate out, 'out' a separate out beside an aligned
    weight"""
    V = E.vec_width(dtype)
    n = V * 1024 + V - 1
    ins = E.special_inputs(op, n, dtype, [0, n // 2, n - E.WINDOW], seed=len(which))
    params = plain_params(op)
    distinct = which in ('w_only', 'out')
    off = 1 if unit == 'elem' else 8 // (4 if dtype == 'float32' else 2)
    key = 'w' if which == 'w_only' else which
    want = check_dense(mx, op, dtype, ins, params, 'aligned', distinct_out=distinct)
    got = check_dense(mx, op, dtype, ins, params, which, distinct_out=distinct, offsets={key: off})
    assert same(got[0], want[0], dtype)
    for a, b in zip(got[1], want[1]):
        assert same(a, b, 'float32')


def out_cases():
    out = []
    for op, dt in OP_DTYPES:
        V = E.vec_width(dt)
        for n in (V - 1, 2 * V + V - 1, E.wrap_size(V)):
            out.append(pytest.param(op, dt, n, id='%s-%s-%d' % (op, dt, n)))
    return out


@pytest.mark.parametrize("op,dtype,n", out_cases())
def test_dense_distinct_out(mx, op, dtype, n):
    """out a separate array at every size class: the weight is untouched, out and the states are
    the restatement's (for NAG the momentum then reads the old weight)"""
    ins = E.special_inputs(op, n, dtype, [0, E.wrap_anchor(E.vec_width(dtype)) - E.WINDOW // 2, n - E.WINDOW])
    check_dense(mx, op, dtype, ins, plain_params(op), 'distinct out', distinct_out=True)


def test_nag_out_is_w_differs_from_distinct_out_at_wrap(mx):
    """nag_mom_update's momentum reads the weight as it is after out was stored: with out = w that
    is the new weight, with a separate out the old one. Both, past one grid stride, and they differ"""
    n = E.wrap_size(4)
    ins = E.dense_inputs('nag_mom_update', n)
    params = plain_params('nag_mom_update')
    _, st_inplace = check_dense(mx, 'nag_mom_update', 'float32', ins, params, 'out is w')
    _, st_distinct = check_dense(mx, 'nag_mom_update', 'float32', ins, params, 'distinct', distinct_out=True)
    tail = slice(E.wrap_anchor(4), n)
    assert not same(st_inplace[0][tail], st_distinct[0][tail], 'float32')


# ------------------------------------------------------------------------------- special values
@pytest.mark.parametrize("path", ['vector', 'scalar'])
@pytest.mark.parametrize("op,dtype", OP_DTYPES)
def test_dense_special_values(mx, op, dtype, path):
    """NaN, +-Inf, +-0 and +-1e-40 in every operand and state: at the start of the body, in its
    middle, across the first element of the grid-stride loop's second pass and in the tail; two
    steps (the second clipped) so the states carry them"""
    V = E.vec_width(dtype)
    n = E.wrap_size(V)
    vec = path == 'vector'
    wrap = E.wrap_anchor(V, vec) - E.WINDOW // 2
    ins = E.special_inputs(op, n, dtype, [0, n // 3, wrap, n - E.WINDOW], seed=V + vec)
    offs = {} if vec else {k: 1 for k in ['w', 'g'] + ['s%d' % k for k in range(len(ins) - 2)]}
    for params in list(GU.VARIANTS[op].values())[:1] + [plain_params(op)]:
        out, st = check_dense(mx, op, dtype, ins, params, (path, params), offsets=offs)
        ins = [out, ins[1]] + st


# ------------------------------------------------------------------------ hyper-parameter edges
@pytest.mark.parametrize("op,dtype,name", E.hyper_cases())
def test_dense_hyper_edges(mx, op, dtype, name):
    """the edges of update_edges.HYPER with the operands that make them bite, on the vector path
    (body and tail) and on the scalar path"""
    V = E.vec_width(dtype)
    n = V * 1024 + V - 1
    ins, params = E.hyper_inputs(op, dtype, name, n)
    check_dense(mx, op, dtype, ins, params, name)
    check_dense(mx, op, dtype, ins, params, name + ' scalar', offsets={'g': 1})


# ----------------------------------------------------------------------- mp_nag 16-bit edges
@pytest.mark.parametrize("dtype", ['float16', 'bfloat16'])
@pytest.mark.parametrize("size", ['small', 'wrap'])
def test_mp_nag_16bit_edges(mx, dtype, size):
    """the float16 overflow boundary, float16 / bfloat16 subnormals and bfloat16 ties in the
    rounding of the new master, subnormal 16-bit gradients, and a 16-bit weight that disagrees with
    its master (the operator reads the master only), in the body, the tail and across the wrap"""
    n = 8 * 16 + 5 if size == 'small' else E.wrap_size(8)
    anchors = [0, n - E.MASTER_EDGES.size - 8] + ([E.wrap_anchor(8) - 20] if size == 'wrap' else [])
    ins = E.mp_edge_inputs(n, dtype, anchors)
    for distinct in (False, True):
        out, _ = check_dense(mx, 'mp_nag_mom_update', dtype, [a.copy() for a in ins], E.MP_EDGE_PARAMS,
                             'edges', distinct_out=distinct)
    if dtype == 'float16':
        assert [float(x) for x in out.view(np.float16)[:4]] == [65504.0, 65504.0, 65504.0, np.inf]


# --------------------------------------------------------------------- row_sparse Ftrl / AdaGrad
def rsp(mx, vals, ids, shape):
    return mx.nd.sparse.row_sparse_array((vals.reshape((len(ids),) + tuple(shape[1:])), np.asarray(ids)),
                                         shape=shape, ctx=mx.gpu(0), dtype=np.float32)


def table(mx, a, stype):
    if stype == GS.DNS:
        return mx.nd.array(a, mx.gpu(0))
    return rsp(mx, a, np.arange(a.shape[0]), a.shape)


def restate_rsp(form, tables, ids, g, rows, L):
    op, wst = GS.FORMS[form]
    t = [a.copy() for a in tables]
    nnr = [rows if wst == GS.RSP else 0, len(ids)] + [rows if wst == GS.RSP else 0] * (len(t) - 1)
    GS.restate(op, [wst, GS.RSP] + [wst] * (len(t) - 1), nnr, [t[0], g.copy()] + t[1:], ids, rows, L, True,
               **E.RSP_PARAMS[form])
    return t


def call_rsp(mx, form, nds, g):
    f = mx.nd.ftrl_update if form == 'ftrl' else mx.nd.sparse.adagrad_update
    f(nds[0], g, *nds[1:], out=nds[0], **E.RSP_PARAMS[form])


@pytest.mark.parametrize("L", [4, 5, 64])
@pytest.mark.parametrize("form", sorted(GS.FORMS))
def test_rsp_row_update_many_rows(mx, form, L):
    """tens of thousands of gradient rows (one warp each) over a larger table, specials in the
    gradient, the weight and the states; rows the gradient does not list stay bitwise"""
    rows = 60000 if L < 64 else 12000
    tables, ids, g = E.rsp_tables(form, rows, L, rows * 5 // 6, seed=L)
    wst = GS.FORMS[form][1]
    nds = [table(mx, a, wst) for a in tables]
    call_rsp(mx, form, nds, rsp(mx, g, ids, (rows, L)))
    want = restate_rsp(form, tables, ids, g, rows, L)
    for k, (nd, w) in enumerate(zip(nds, want)):
        assert same(nd.asnumpy(), w, 'float32'), (form, L, k)


@pytest.mark.parametrize("which", ['w', 'h', 'both'])
@pytest.mark.parametrize("unit", ['elem', '8B'])
@pytest.mark.parametrize("L", [4, 8])
def test_dense_adagrad_misaligned_table_view(mx, L, unit, which):
    """_sparse_adagrad_update on a dense weight and history that are views starting off a 16-byte
    boundary (one table, so every row is misaligned): the scalar row path, with the results of the
    restatement"""
    torch = pytest.importorskip("torch")
    rows = 3001
    tables, ids, g = E.rsp_tables('adagrad_dns', rows, L, 1500, seed=L + len(unit))
    off = 1 if unit == 'elem' else 2
    nds, keep = [], []
    for k, a in enumerate(tables):
        o = off if which == 'both' or which == ('w', 'h')[k] else 0
        base = torch.zeros(rows * L + 4, dtype=torch.float32, device='cuda:0')
        view = base[o:o + rows * L].view(rows, L)
        view.copy_(torch.from_numpy(a))
        keep.append((base, o))
        nds.append(mx.nd.from_torch(view))
    torch.cuda.synchronize()
    call_rsp(mx, 'adagrad_dns', nds, rsp(mx, g, ids, (rows, L)))
    want = restate_rsp('adagrad_dns', tables, ids, g, rows, L)
    for nd, w in zip(nds, want):
        assert same(nd.asnumpy(), w, 'float32'), (L, unit, which)
    mx.nd.waitall()
    for base, o in keep:
        b = base.cpu().numpy()
        assert not b[:o].any() and not b[o + rows * L:].any(), 'written outside the view'


# --------------------------------------------------------------------------------- GroupAdaGrad
GA_CASES = [  # (row_len, variant it selects, table form)
    (4, 'vec_one_tile', GG.DNS), (4, 'vec_one_tile', GG.RSP), (5, 'scalar_one_tile', GG.DNS),
    (1000, 'vec_multi_tile', GG.DNS)]


@pytest.mark.parametrize("L,variant,wst", GA_CASES, ids=['%d-%s-%s' % (c[0], c[1], 'rsp' if c[2] else 'dns')
                                                          for c in GA_CASES])
def test_group_adagrad_past_one_grid_pass(mx, L, variant, wst):
    """more gradient rows than the capped grid has warps, so each warp's row loop runs again (and
    the one-tile variants prefetch a next row); NaN in one lane's run of the row fold, +-Inf,
    specials in the weight and the history"""
    assert (L <= E.GA_TILE) == variant.endswith('one_tile') and (L % 4 == 0) == variant.startswith('vec')
    nnr = 2 * E.GA_WARPS + 5 if L < 64 else E.GA_WARPS + 1000
    rows = nnr + nnr // 8
    w, h, ids, g = E.ga_tables(rows, L, nnr, seed=L)
    wn = table(mx, w, wst)
    hn = table(mx, h, wst)
    mx.nd.contrib.group_adagrad_update(wn, rsp(mx, g, ids, (rows, L)), hn, out=wn, **E.GA_PARAMS)
    ww, hh = w.copy(), h.copy()
    nr = [rows if wst == GG.RSP else 0, len(ids), rows if wst == GG.RSP else 0]
    GG.restate(GG.OP, [wst, GG.RSP, wst], nr, [ww, g.copy(), hh], ids, rows, L, True, **E.GA_PARAMS)
    assert same(wn.asnumpy(), ww, 'float32'), 'weight'
    assert same(hn.asnumpy(), hh, 'float32'), 'history'
    assert np.isnan(hh[ids[E.GA_WARPS:]]).any()


# --------------------------------------------------------------------- row_sparse gradient pass
def check_rspg(mx, op, rows, L, ids, seed):
    w, g, states = E.rspg_inputs(op, rows, L, ids, seed)
    shape = (rows, L)
    params = plain_params(op)
    wn = mx.nd.array(w, mx.gpu(0))
    sn = [mx.nd.array(s, mx.gpu(0)) for s in states]
    getattr(mx.nd, op)(wn, rsp(mx, g, ids, shape), *sn, out=wn, **params)
    out, st = GU.restate(op, [w, E.densify(shape, ids, g)] + states, params)
    assert same(wn.asnumpy(), out, 'float32'), (op, L, 'out')
    for k, (a, b) in enumerate(zip(sn, st)):
        assert same(a.asnumpy(), b, 'float32'), (op, L, k)


@pytest.mark.parametrize("L", [2, 4, 6])
@pytest.mark.parametrize("op", OPS)
def test_rsp_grad_row_lens(mx, op, L):
    """row_len 4 is one 16-byte group; 2 and 6 take the scalar path on aligned operands; specials in
    the stored rows and in the weight and state rows, stored or not"""
    rows = 4099
    ids = E.pick_ids(np.random.default_rng(L), rows, rows // 3)
    check_rspg(mx, op, rows, L, ids, seed=L)


@pytest.mark.parametrize("L", [4, 6])
@pytest.mark.parametrize("op", OPS)
def test_rsp_grad_rows_straddle_first_pass(mx, op, L):
    """a table past UPDATE_THREADS groups (row_len 4) or elements (row_len 6), with stored rows on
    both sides of where a capped grid's first pass ends"""
    per = 4 if L == 4 else 1                      # elements per item of the launch
    edge = E.wrap_anchor(4, L == 4) // L          # the row holding the first element past one pass
    rows = edge + 2000
    rng = np.random.default_rng(L + 1)
    ids = np.unique(np.concatenate([np.arange(edge - 3, edge + 4), rng.choice(rows, rows // 50, replace=False),
                                    [0, rows - 1]])).astype(np.int64)
    assert ids.min() * L < E.UPDATE_THREADS * per <= ids.max() * L
    check_rspg(mx, op, rows, L, ids, seed=L + 7)
