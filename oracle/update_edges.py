"""TEST INFRASTRUCTURE ONLY -- the edge cases of the NAG / Signum / RMSProp / FTML / Ftrl / AdaGrad /
GroupAdaGrad operators' kernels, shared by tests/test_update_ops_edges_host.py (which pins the numpy
restatements to the reference's own CPU operators at exactly these inputs) and
tests/test_update_ops_edges_gpu.py (which holds the sm_90a kernels to those restatements):

  * the launch geometry read from the kernels' source (kNumSMs, the block sizes and the grid caps of
    update_kernel and rsp_group_adagrad_kernel), so the sizes that wrap a grid follow a retuned cap;
  * special values (NaN, +-Inf, +-0, +-1e-40) spread over every operand and state;
  * the hyper-parameter edges of every operator, with the operands that make them bite: gradients
    whose rescaled value is exactly +-clip (and one or two ulps either side), Ftrl z exactly
    +-lamda1, RMSPropAlex states with n - g*g < 0;
  * mp_nag_mom_update's 16-bit edges: the float16 overflow boundary, subnormal halves, bfloat16
    ties, and a 16-bit weight that disagrees with its float32 master;
  * row_sparse tables (Ftrl, AdaGrad, GroupAdaGrad) and row_sparse gradients with special values in
    the stored rows and in the rows the gradient does not store.
"""
import os
import re

import numpy as np

import golden_update_ops as GU

F = np.float32
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(_ROOT, "anand_mxnet_b200", "csrc")


# ------------------------------------------------------------------------------ launch geometry
def _one(pattern, text, what):
    found = re.findall(pattern, text)
    if len(found) != 1:
        raise LookupError("%d matches for %s" % (len(found), what))
    return int(found[0])


def read_constants(csrc=CSRC):
    """kNumSMs, update_kernel's block size and grid cap (in CTAs per SM), and rsp_group_adagrad_kernel's
    warps per block, grid cap and tile, as the source declares them"""
    def text(name):
        with open(os.path.join(csrc, name)) as f:
            return f.read()
    common, upd, rsp = text("common.h"), text("update_kernel.cuh"), text("rowsparse_kernels.cu")
    launch = rsp.split("void LaunchRspRowUpdateOp(", 1)[1].split("kUpdGroupAdaGrad", 1)[0]
    return {
        'kNumSMs': _one(r"constexpr\s+int\s+kNumSMs\s*=\s*(\d+)\s*;", common, "kNumSMs"),
        'kThreads': _one(r"constexpr\s+int\s+kThreads\s*=\s*(\d+)\s*;", upd, "kThreads"),
        'update_cap': _one(r"std::min<size_t>\(want,\s*kNumSMs\s*\*\s*(\d+)\)", upd, "update_kernel's grid cap"),
        'kWarpsPerBlock': _one(r"constexpr\s+int\s+kWarpsPerBlock\s*=\s*(\d+)\s*;", rsp, "kWarpsPerBlock"),
        'ga_cap': _one(r"kNumSMs\s*\*\s*(\d+)\)\);", launch, "the row update's grid cap"),
        'kGaPer': _one(r"constexpr\s+int\s+kGaPer\s*=\s*(\d+)\s*;", rsp, "kGaPer"),
    }


C = read_constants()
# threads of a capped update_kernel grid: one pass of its grid-stride loop
UPDATE_THREADS = C['kNumSMs'] * C['update_cap'] * C['kThreads']
# warps of rsp_group_adagrad_kernel's capped grid: one pass of its row loop
GA_WARPS = C['kNumSMs'] * C['ga_cap'] * C['kWarpsPerBlock']
GA_TILE = 32 * C['kGaPer']      # rows up to this length take the ONE_TILE variant


def vec_width(dtype):
    """elements per 16-byte group"""
    return 4 if dtype == 'float32' else 8


def small_sizes(V):
    """V-1, V, V+1 and 2V+k for every tail k"""
    return [V - 1, V, V + 1] + [2 * V + k for k in range(V)]


def wrap_size(V):
    """a vector body past one full grid stride (a partial second pass) followed by a tail"""
    return V * UPDATE_THREADS + V * 1000 + (3 if V == 4 else 5)


def wrap_anchor(V, vec=True):
    """the first element of the grid-stride loop's second pass, vector or scalar"""
    return (V if vec else 1) * UPDATE_THREADS


# ----------------------------------------------------------------------------- special values
SPECIALS = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1e-40, -1e-40], F)
WINDOW = 48


def specials_as(dt, vals):
    """float32 specials in an operand's storage: float16 values, or bfloat16 bit patterns"""
    if dt == 'float16':
        return vals.astype(np.float16)
    if dt == 'bfloat16':
        return GU.to_bf16_bits(vals)
    return vals


def put_specials(arrays, dts, anchors, seed, window=WINDOW, density=0.5):
    """in place: in a `window`-element run from each anchor (clamped into the array), each array takes
    a special value at about `density` of the elements, drawn independently per array, so an
    element mixes specials in several operands with ordinary values in the others"""
    rng = np.random.default_rng(seed)
    n = arrays[0].size
    for a in anchors:
        lo = max(0, min(a, n - window))
        hi = min(n, lo + window)
        for x, dt in zip(arrays, dts):
            flat = x.reshape(-1)
            m = rng.random(hi - lo) < density
            v = specials_as(dt, SPECIALS[rng.integers(0, SPECIALS.size, hi - lo)])
            flat[lo:hi][m] = v[m]


def operand_dtypes(op, dtype):
    """storage of [weight, grad, states...]"""
    ns = GU.N_STATES[op]
    return [dtype, dtype] + ['float32'] * ns


def dense_inputs(op, n, dtype='float32'):
    """golden_update_ops.inputs at n; RMSPropAlex's states also hold n < g*g (a negative square root)
    at every 13th element"""
    ins = GU.inputs(dict(op=op, dtype=dtype, n=n))
    if op == 'rmspropalex_update':
        ins[2][::13] = F(0.01)
        ins[3][::13] = F(0.5)
    return ins


def special_inputs(op, n, dtype, anchors, seed=0):
    ins = dense_inputs(op, n, dtype)
    put_specials(ins, operand_dtypes(op, dtype), anchors, seed)
    return ins


# --------------------------------------------------------------------------- hyper-parameters
def _nag(**kw):
    p = dict(lr=0.05, momentum=0.9, wd=0.001, rescale_grad=0.1, clip_gradient=0.5)
    p.update(kw)
    return p


def _rms(alex, **kw):
    p = dict(lr=0.001, gamma1=0.9, epsilon=1e-08, wd=0.01, rescale_grad=0.1, clip_gradient=0.5)
    if alex:
        p['gamma2'] = 0.9
    p.update(kw)
    return p


def _ftml(**kw):
    p = dict(lr=0.01, beta1=0.6, beta2=0.999, epsilon=1e-08, wd=0.001, rescale_grad=0.1, clip_grad=0.5, t=3)
    p.update(kw)
    return p


def _ftrl(**kw):
    p = dict(lr=0.1, lamda1=0.01, beta=1.0, wd=0.001, rescale_grad=0.1, clip_gradient=0.5)
    p.update(kw)
    return p


# clip_exact: clip on, wd 0 where wd*w joins the gradient before the clip, so the rescaled gradients
# of clip_gradients() land exactly on +-clip
_NAG = {'clip0': _nag(clip_gradient=0.0), 'clip_exact': _nag(), 'momentum0': _nag(momentum=0.0)}
HYPER = {
    'nag_mom_update': _NAG,
    'mp_nag_mom_update': _NAG,
    'signsgd_update': {'clip0': dict(lr=0.01, wd=0.01, rescale_grad=0.1, clip_gradient=0.0)},
    'signum_update': {'clip0': dict(lr=0.01, momentum=0.9, wd=0.001, wd_lh=0.01, rescale_grad=0.1, clip_gradient=0.0),
                      'clip_exact': dict(lr=0.01, momentum=0.9, wd=0.001, wd_lh=0.01, rescale_grad=0.1,
                                         clip_gradient=0.5),
                      'momentum0': dict(lr=0.01, momentum=0.0, wd=0.001, rescale_grad=0.1, clip_gradient=0.5)},
    'rmsprop_update': {'clip0': _rms(False, clip_gradient=0.0), 'clip_exact': _rms(False, wd=0.0),
                       'clip_weights0': _rms(False, clip_weights=0.0), 'gamma1_0': _rms(False, gamma1=0.0),
                       'gamma1_1': _rms(False, gamma1=1.0)},
    'rmspropalex_update': {'clip0': _rms(True, clip_gradient=0.0), 'clip_exact': _rms(True, wd=0.0),
                           'clip_weights0': _rms(True, clip_weights=0.0), 'gamma1_0': _rms(True, gamma1=0.0),
                           'gamma1_1': _rms(True, gamma1=1.0)},
    # beta1 = 1: dt = 0 (out = -z/0); beta2 = 1: dt = Inf; large t: powf(beta2, t) near 0, then
    # subnormal
    'ftml_update': {'clip0': _ftml(clip_grad=0.0), 'clip_exact': _ftml(wd=0.0), 'beta1_0': _ftml(beta1=0.0),
                    'beta1_1': _ftml(beta1=1.0), 'beta2_1': _ftml(beta2=1.0), 't20000': _ftml(t=20000),
                    't100000': _ftml(t=100000)},
    'ftrl_update': {'clip0': _ftrl(clip_gradient=0.0), 'clip_exact': _ftrl(), 'lamda1_0': _ftrl(lamda1=0.0),
                    'beta0': _ftrl(beta=0.0)},
}


def hyper_cases():
    """(op, dtype, name) of every hyper-parameter edge"""
    out = []
    for op, cases in HYPER.items():
        for dt in (('float16', 'bfloat16') if op == 'mp_nag_mom_update' else ('float32',)):
            out += [(op, dt, name) for name in cases]
    return out


def clip_gradients(params, dtype):
    """gradients whose rescaled value is +-clip, and their 1- and 2-ulp neighbours (in the
    gradient's storage); clip 0: +-0, +-1e-40 and +-1"""
    clip = float(GU.stof(params.get('clip_gradient', params.get('clip_grad', -1.0))))
    rescale = GU.stof(params.get('rescale_grad', 1.0))
    if clip <= 0:
        g = np.array([0.0, -0.0, 1e-40, -1e-40, 1.0, -1.0], F)
        return specials_as(dtype, g)
    if dtype == 'bfloat16':
        c = GU.to_bf16_bits(np.array([clip / float(rescale)], F)).astype(np.int32)
        g = np.concatenate([c + d for d in (-2, -1, 0, 1, 2)]).astype(np.uint16)
        return np.concatenate([g, g | np.uint16(0x8000)])
    st = np.float16 if dtype == 'float16' else F
    c = st(clip / float(rescale))
    g = [c]
    for d in (np.inf, -np.inf):
        x = c
        for _ in range(2):
            x = np.nextafter(x, st(d))
            g.append(x)
    g = np.array(g, st)
    return np.concatenate([g, -g])


def hyper_inputs(op, dtype, name, n):
    """dense_inputs at n with the clip edge gradients at the start and the end; Ftrl also gets z at
    +-lamda1 and one ulp either side with g = 0 (then z is unchanged by the step, so the strict
    |z| > lamda1 decides the element)"""
    params = HYPER[op][name]
    ins = dense_inputs(op, n, dtype)
    g = clip_gradients(params, dtype)
    k = min(g.size, n)
    ins[1][:k] = g[:k]
    ins[1][n - k:] = g[g.size - k:]
    if op == 'ftrl_update':
        lam = GU.stof(params['lamda1'])
        z = []
        for s in (F(1), F(-1)):
            b = s * lam
            z += [b, np.nextafter(b, F(np.inf)), np.nextafter(b, F(-np.inf))]
        z = np.array(z, F)
        for start in (k, max(0, n - k - z.size)):
            m = min(z.size, n - start)
            if m > 0:
                ins[1][start:start + m] = 0
                ins[2][start:start + m] = z[:m]
    return ins, params


# ------------------------------------------------------------------------- mp_nag 16-bit edges
def _bits(*b):
    return np.array(b, np.uint32).view(F)


# float32 master values whose 16-bit rounding is an edge: the float16 overflow boundary (65504
# stays, 65519 rounds down, 65520 overflows), float16 subnormals and their ties, bfloat16 ties
# (even below, odd above, one ulp past), the bfloat16 overflow tie and FLT_MAX, bfloat16
# subnormal ties, and the specials
MASTER_EDGES = np.concatenate([
    np.array([65504, 65519, np.nextafter(F(65520), F(0)), 65520, 65536, 1e5, -65504, -65519, -65520,
              2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -25, 2.0 ** -26, -2.0 ** -25, 1e-7, 5.9e-8,
              2.0 ** -14, 2.0 ** -14 - 2.0 ** -25, 6.0e-5], F),
    _bits(0x3F808000, 0x3F818000, 0x3F808001, 0xBF808000, 0xBF818000, 0x7F7F8000, 0x7F7FFFFF,
          0x7F7F7FFF, 0x00008000, 0x00018000, 0x80008000, 0x00000001),
    SPECIALS])
MP_EDGE_PARAMS = dict(lr=0.05, momentum=0.9, wd=0.0, rescale_grad=0.5)


def subnormal_grads(dtype):
    """16-bit subnormal gradients"""
    if dtype == 'bfloat16':
        return np.array([0x0001, 0x8003, 0x007F, 0x0040], np.uint16)
    return np.array([2.0 ** -24, -3 * 2.0 ** -24, 1e-5, -6.0e-5], np.float16)


def mp_edge_inputs(n, dtype, anchors):
    """mp_nag_mom_update operands with a 16-bit weight that disagrees with its master everywhere (the
    operator reads only the master); at each anchor a run where the master holds MASTER_EDGES with
    g = 0 and mom = 0, so with wd = 0 out is the master rounded to 16 bits, then a run of subnormal
    16-bit gradients"""
    w16, g16, mom, w32 = GU.inputs(dict(op='mp_nag_mom_update', dtype=dtype, n=n))
    w16 = specials_as(dtype, (w32 * F(-0.75) + F(0.375)).astype(F))
    e, sg = MASTER_EDGES, subnormal_grads(dtype)
    for a in anchors:
        lo = max(0, min(a, n - e.size - sg.size))
        m = min(e.size, n - lo)
        w32[lo:lo + m] = e[:m]
        g16[lo:lo + m] = 0
        mom[lo:lo + m] = 0
        s = lo + m
        k = min(sg.size, n - s)
        g16[s:s + k] = sg[:k]
    return [w16, g16, mom, w32]


# -------------------------------------------------------------------------- row_sparse tables
def pick_ids(rng, rows, count):
    """`count` sorted distinct row ids of [0, rows), the first and the last among them"""
    inner = rng.choice(np.arange(1, rows - 1), size=count - 2, replace=False)
    return np.unique(np.concatenate([[0, rows - 1], inner])).astype(np.int64)


def rsp_tables(form, rows, L, nnr, seed, specials=True):
    """tables [w, states...] (rows x L), gradient ids and rows of golden_sparse_update_ops' forms
    'ftrl' / 'adagrad' / 'adagrad_dns', with its distributions; specials at about 2 % of the
    elements of every table and of the gradient"""
    rng = np.random.default_rng(seed)
    u = lambda *s: rng.uniform(-1, 1, s).astype(F)      # noqa: E731
    w = u(rows, L)
    if form == 'ftrl':
        z = (u(rows, L) * F(0.02)).astype(F)
        z.reshape(-1)[::7] = 0
        states = [z, rng.uniform(0, 0.5, (rows, L)).astype(F)]
    else:
        states = [rng.uniform(0, 1, (rows, L)).astype(F)]
    ids = pick_ids(rng, rows, nnr)
    g = u(len(ids), L)
    if form == 'ftrl':
        g = (g * F(0.004)).astype(F)
        g.reshape(-1)[::11] = 0
    if specials:
        for x in [w, g] + states:
            flat = x.reshape(-1)
            m = rng.random(flat.size) < 0.02
            flat[m] = SPECIALS[rng.integers(0, SPECIALS.size, int(m.sum()))]
    return [w] + states, ids, g


RSP_PARAMS = {
    'ftrl': dict(lr=0.1, lamda1=0.01, beta=1, wd=0.001, rescale_grad=0.5, clip_gradient=0.3),
    'adagrad': dict(lr=0.05, wd=0.0, epsilon=1e-06, rescale_grad=0.5, clip_gradient=0.3),
}
RSP_PARAMS['adagrad_dns'] = RSP_PARAMS['adagrad']


def ga_tables(rows, L, nnr, seed):
    """GroupAdaGrad's weight (rows x L), history (rows x 1), gradient ids and rows: a NaN in one
    lane's run of the fold (element 16k + j) of every 5th gradient row, +-Inf in others, specials in
    the weight and the history"""
    rng = np.random.default_rng(seed)
    w = rng.uniform(-1, 1, (rows, L)).astype(F)
    h = rng.uniform(0, 2, (rows, 1)).astype(F)
    ids = pick_ids(rng, rows, nnr)
    g = rng.uniform(-1, 1, (len(ids), L)).astype(F)
    per = C['kGaPer']
    nan_rows = np.arange(0, len(ids), 5)
    cols = np.minimum(rng.integers(0, max(1, L // per), nan_rows.size) * per + rng.integers(0, per, nan_rows.size),
                      L - 1)
    g[nan_rows, cols] = np.nan
    inf_rows = np.arange(2, len(ids), 7)
    g[inf_rows, rng.integers(0, L, inf_rows.size)] = np.where(inf_rows % 2 == 0, F(np.inf), F(-np.inf))
    for x in (w, h):
        flat = x.reshape(-1)
        m = rng.random(flat.size) < 0.02
        flat[m] = SPECIALS[rng.integers(0, SPECIALS.size, int(m.sum()))]
    return w, h, ids, g


GA_PARAMS = dict(lr=0.05, epsilon=1e-05, rescale_grad=0.25, clip_gradient=0.5)


def rspg_inputs(op, rows, L, ids, seed):
    """a dense weight and states (rows x L, golden_update_ops' distributions) and the stored rows of
    a row_sparse gradient at `ids`, with specials in the stored rows and in the weight and state
    rows, stored or not"""
    ins = [x.reshape(rows, L) for x in dense_inputs(op, rows * L)]
    rng = np.random.default_rng(seed)
    g = ins[1][ids].copy()
    for x in [ins[0], g] + ins[2:]:
        flat = x.reshape(-1)
        m = rng.random(flat.size) < 0.03
        flat[m] = SPECIALS[rng.integers(0, SPECIALS.size, int(m.sum()))]
    return ins[0], g, ins[2:]


def densify(shape, ids, vals):
    """the reference's cast of a row_sparse gradient: +0.0 everywhere, then the stored rows"""
    d = np.zeros(shape, F)
    d[np.asarray(ids, np.int64)] = vals
    return d
