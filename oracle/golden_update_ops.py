"""TEST INFRASTRUCTURE ONLY -- the single-tensor optimizer operators of the reference's NAG / Signum /
RMSProp / FTML / Ftrl optimizers: a numpy float32 restatement (`restate`), the reference's own CPU
code (`RefUpdateOps` over oracle/_ref/libmxref_update.so, built from oracle/ref_update_ops.cc by
oracle/update_ops.mk), the seeded `CASES`, and the writer of tests/golden/update_ops.npz:

    make -f oracle/update_ops.mk && python oracle/golden_update_ops.py

Inputs are regenerated from each case's seed wherever the fixture is read, so the fixture holds
outputs only: every output array in full for small cases, and for large ones its SHA-256 plus the
first elements. Every restated expression tree is the reference kernel's as written
(src/operator/optimizer_op-inl.h); numpy float32 arithmetic rounds once per operation, like the
reference's CPU build (no FMA contraction).
"""
import ctypes
import ctypes.util
import hashlib
import os
import subprocess
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import kvoracle as K  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
F = np.float32
OPS = ['nag_mom_update', 'mp_nag_mom_update', 'signsgd_update', 'signum_update', 'rmsprop_update',
       'rmspropalex_update', 'ftml_update', 'ftrl_update']
N_STATES = {'nag_mom_update': 1, 'mp_nag_mom_update': 2, 'signsgd_update': 0, 'signum_update': 1,
            'rmsprop_update': 1, 'rmspropalex_update': 3, 'ftml_update': 3, 'ftrl_update': 2}
FULL_MAX = 64      # cases up to this size keep their outputs in full
HEAD = 16          # elements kept beside the digest of a larger output


def build():
    """oracle/_ref/libmxref_update.so, where the reference's sources exist"""
    if os.path.isfile("/root/reference/src/operator/optimizer_op-inl.h"):
        subprocess.run(["make", "-s", "-f", os.path.join(HERE, "update_ops.mk")], check=True)


class RefUpdateOps(K.Ref):
    """op_invoke over oracle/_ref/libmxref_update.so (same entry point as libmxref.so's)"""

    def __init__(self, path):
        self.lib = ctypes.CDLL(path)


_ref = False


def ref():
    """The reference's operators, or None when oracle/_ref/libmxref_update.so has not been built."""
    global _ref
    if _ref is False:
        path = os.path.join(HERE, "_ref", "libmxref_update.so")
        _ref = RefUpdateOps(path) if os.path.exists(path) else None
    return _ref


# ------------------------------------------------------------------------------ scalar plumbing
def stof(v):
    """a float field: python str() -> dmlc::stof"""
    return F(K.dmlc_stof(str(v)))


def stod(s):
    """dmlc::stod == ParseFloat<double, true> (dmlc/strtonum.h:99-254), the parser of double fields
    (FTML's epsilon): double(int part) + double(frac digits)/double(10^k), then scaled by 1e8 / 10
    steps in double. Not a correctly rounded conversion."""
    p = s.strip()
    sign = 1.0
    if p[:1] in '+-':
        sign = -1.0 if p[0] == '-' else 1.0
        p = p[1:]
    low = p.lower()
    if low.startswith('inf'):
        return sign * float('inf')
    if low.startswith('nan'):
        return float('nan')
    i = 0
    predec = 0
    while i < len(p) and p[i].isdigit():
        predec = predec * 10 + int(p[i])
        i += 1
    value = float(predec)
    if i < len(p) and p[i] == '.':
        i += 1
        val2, pow10, cnt = 0, 1, 0
        while i < len(p) and p[i].isdigit():
            if cnt < 19:
                val2 = val2 * 10 + int(p[i])
                pow10 *= 10
            cnt += 1
            i += 1
        value += float(val2) / float(pow10)
    if i < len(p) and p[i] in 'eE':
        i += 1
        frac = False
        if i < len(p) and p[i] in '+-':
            frac = p[i] == '-'
            i += 1
        expon = 0
        while i < len(p) and p[i].isdigit():
            expon = expon * 10 + int(p[i])
            i += 1
        scale = 1.0
        while expon >= 8:
            scale *= 1e8
            expon -= 8
        while expon > 0:
            scale *= 10.0
            expon -= 1
        value = value / scale if frac else value * scale
    return sign * value


_libm = ctypes.CDLL(ctypes.util.find_library('m'))
_libm.powf.restype = ctypes.c_float
_libm.powf.argtypes = [ctypes.c_float, ctypes.c_float]


def powf(a, b):
    """glibc ::powf, what power::Map(float, float) calls (math_functions-inl.h:58-61,126)"""
    return F(_libm.powf(float(a), float(b)))


# -------------------------------------------------------------------------------- restatement
def _clip(x, b):
    return np.where(x > b, b, np.where(x < -b, -b, x)).astype(F)     # mshadow_op::clip


def _sign_int(x):
    return ((x > 0).astype(np.int32) - (x < 0).astype(np.int32)).astype(F)


def to_bf16_bits(x):
    """float32 -> bfloat16 bit patterns, round to nearest even (__float2bfloat16_rn)"""
    b = np.ascontiguousarray(x, F).view(np.uint32).astype(np.uint64)
    r = (b + 0x7FFF + ((b >> 16) & 1)) >> 16
    return np.where(np.isnan(x), 0x7FC0, r).astype(np.uint16)


def bf16_bits_to_f32(h):
    return (np.asarray(h, np.uint16).astype(np.uint32) << 16).view(F)


def restate(op, ins, params, distinct_out=False, dtype='float32'):
    """numpy restatement of one operator call. ins: [weight, grad, states...] (16-bit weights /
    grads of mp_nag_mom_update: float16 arrays, or bfloat16 bit patterns as uint16 with
    dtype='bfloat16'). Returns (out, [states after]); inputs are not modified."""
    P = dict(params)
    lr = stof(P['lr'])
    wd = stof(P.get('wd', 0.0))
    rescale = stof(P.get('rescale_grad', 1.0))
    clip = stof(P.get('clip_gradient', -1.0))
    one = F(1)
    s = [np.array(a, F) for a in ins[2:]]
    if op == 'mp_nag_mom_update':
        g = bf16_bits_to_f32(ins[1]) if dtype == 'bfloat16' else ins[1].astype(F)
        w = None
    else:
        w, g = np.array(ins[0], F), np.array(ins[1], F)
    if op in ('nag_mom_update', 'mp_nag_mom_update'):
        # optimizer_op-inl.h:1061-1138
        momentum = stof(P.get('momentum', 0.0))
        w0 = s[1] if op == 'mp_nag_mom_update' else w
        cg = rescale * g
        if clip >= 0:
            cg = _clip(cg, clip)
        mom = momentum * s[0]
        out = (w0 - mom) + (momentum + one) * (mom - lr * (cg + wd * w0))
        w1 = out if (op == 'mp_nag_mom_update' or not distinct_out) else w0
        s[0] = mom - lr * (cg + wd * w1)
        if op == 'mp_nag_mom_update':
            s[1] = out.copy()
            out = to_bf16_bits(out) if dtype == 'bfloat16' else out.astype(np.float16)
        return out, s
    if op == 'signsgd_update':
        # 2344-2356: clip_gradient, rescale_grad unused
        return (one - lr * wd) * w - lr * _sign_int(g), s
    if op == 'signum_update':
        # 2412-2431
        momentum = stof(P.get('momentum', 0.0))
        wd_lh = stof(P.get('wd_lh', 0.0))
        om = one - momentum
        t = om * _clip(rescale * g, clip) if clip >= 0 else (om * rescale) * g
        s[0] = (momentum * s[0] - (om * wd) * w) - t
        return (one - lr * wd_lh) * w + lr * _sign_int(s[0]), s
    if op in ('rmsprop_update', 'rmspropalex_update'):
        # 1953-1986, 2052-2077
        gamma1 = stof(P.get('gamma1', 0.95))
        gamma2 = stof(P.get('gamma2', 0.9))
        eps = stof(P.get('epsilon', 1e-8))
        cw = stof(P.get('clip_weights', -1.0))
        gr = rescale * g + wd * w
        if clip >= 0:
            gr = _clip(gr, clip)
        om = one - gamma1
        if op == 'rmsprop_update':
            s[0] = om * (gr * gr) + gamma1 * s[0]
            r = w - lr * (gr / np.sqrt(s[0] + eps))
        else:
            s[0] = (om * gr) * gr + gamma1 * s[0]
            s[1] = om * gr + gamma1 * s[1]
            s[2] = gamma2 * s[2] - (lr * gr) / np.sqrt((s[0] - s[1] * s[1]) + eps)
            r = w + s[2]
        return (_clip(r, cw) if cw >= 0 else r), s
    if op == 'ftml_update':
        # 1205-1222; epsilon is a double field, t an int, clip field clip_grad
        beta1 = stof(P.get('beta1', 0.6))
        beta2 = stof(P.get('beta2', 0.999))
        eps = F(stod(str(P['epsilon']))) if 'epsilon' in P else F(np.float64(F(1e-8)))
        t = int(P['t'])
        clip = stof(P.get('clip_grad', -1.0))
        p1, p2 = powf(beta1, t), powf(beta2, t)
        gi = rescale * g + wd * w
        if clip >= 0:
            gi = _clip(gi, clip)
        s[1] = beta2 * s[1] + (one - beta2) * (gi * gi)
        dt = (one - p1) / lr * (np.sqrt(s[1] / (one - p2)) + eps)
        s[2] = (beta1 * s[2] + (one - beta1) * gi) - (dt - beta1 * s[0]) * w
        s[0] = dt
        return (-s[2]) / dt, s
    if op == 'ftrl_update':
        # 2133-2158: states z, n
        lamda1 = stof(P.get('lamda1', 0.01))
        beta = stof(P.get('beta', 1.0))
        gr = g * rescale
        if clip >= 0:
            gr = _clip(gr, clip)
        g2 = gr * gr
        s[0] = s[0] + (gr - ((np.sqrt(s[1] + g2) - np.sqrt(s[1])) * w) / lr)
        s[1] = s[1] + g2
        z = s[0]
        sgn = np.where(z < 0, F(-1), np.where(z > 0, one, F(0))).astype(F)
        gt = (np.abs(z) > lamda1).astype(F)
        return ((sgn * lamda1 - z) / ((beta + np.sqrt(s[1])) / lr + wd)) * gt, s
    raise ValueError(op)


# ------------------------------------------------------------------------------------ cases
SIZES = [1, 3, 4097, (1 << 20) + 5]

VARIANTS = {
    'nag_mom_update': {'plain': dict(lr=0.05, momentum=0.9, rescale_grad=0.125),
                       'clip_wd': dict(lr=0.05, momentum=0.9, wd=0.001, rescale_grad=1.0, clip_gradient=0.3)},
    'mp_nag_mom_update': {'plain': dict(lr=0.05, momentum=0.9, rescale_grad=0.125),
                          'clip_wd': dict(lr=0.05, momentum=0.9, wd=0.001, clip_gradient=0.3)},
    'signsgd_update': {'plain': dict(lr=0.01, rescale_grad=1.0),
                       'clip_wd': dict(lr=0.01, wd=0.01, rescale_grad=0.5, clip_gradient=0.1)},
    'signum_update': {'plain': dict(lr=0.01, momentum=0.9, rescale_grad=1.0),
                      'clip_wd': dict(lr=0.01, momentum=0.9, wd=0.001, rescale_grad=0.5, clip_gradient=0.3,
                                      wd_lh=0.01)},
    'rmsprop_update': {'plain': dict(lr=0.001, gamma1=0.9, epsilon=1e-08, rescale_grad=1.0),
                       'clip_wd': dict(lr=0.001, gamma1=0.9, epsilon=1e-08, wd=0.01, rescale_grad=2.0,
                                       clip_gradient=0.2, clip_weights=0.5)},
    'rmspropalex_update': {'plain': dict(lr=0.001, gamma1=0.9, gamma2=0.9, epsilon=1e-08, rescale_grad=1.0),
                           'clip_wd': dict(lr=0.001, gamma1=0.95, gamma2=0.8, epsilon=1e-08, wd=0.01,
                                           rescale_grad=2.0, clip_gradient=0.2, clip_weights=0.5)},
    'ftml_update': {'plain_t%d' % t: dict(lr=0.01, beta1=0.6, beta2=0.999, epsilon=1e-08, rescale_grad=1.0, t=t)
                    for t in (1, 2, 7)},
    'ftrl_update': {'plain': dict(lr=0.1, lamda1=0.01, beta=1, rescale_grad=1.0),
                    'clip_wd': dict(lr=0.1, lamda1=0.01, beta=1, wd=0.001, rescale_grad=0.5, clip_gradient=0.3)},
}
for _t in (1, 2, 7):
    VARIANTS['ftml_update']['clip_wd_t%d' % _t] = dict(lr=0.01, beta1=0.6, beta2=0.999, epsilon=1e-08, wd=0.001,
                                                       rescale_grad=0.5, clip_grad=0.3, t=_t)


def _cases():
    c = {}
    for op, variants in VARIANTS.items():
        dts = ['float16', 'bfloat16'] if op == 'mp_nag_mom_update' else ['float32']
        for dt in dts:
            for vname, params in variants.items():
                for n in SIZES:
                    name = '%s_%s%s_n%d' % (op, '' if dt == 'float32' else dt + '_', vname, n)
                    c[name] = dict(op=op, dtype=dt, n=n, params=params, distinct_out=False)
        # out as a separate array (kWriteTo): for nag the momentum then sees the old weight
        v0 = sorted(variants)[-1]
        name = '%s_%s_distinct_out_n4097' % (op, dts[0])
        c[name] = dict(op=op, dtype=dts[0], n=4097, params=variants[v0], distinct_out=True)
    return c


CASES = _cases()


def inputs(case):
    """[weight, grad, states...] of a case, regenerated from its name"""
    op, n = case['op'], case['n']
    rng = np.random.default_rng(zlib.crc32(('%s|%s|%d' % (op, case['dtype'], n)).encode()))
    u = lambda lo, hi: rng.uniform(lo, hi, n).astype(F)  # noqa: E731
    w, g = u(-1, 1), u(-1, 1)
    if op == 'nag_mom_update' or op == 'signum_update':
        st = [u(-0.5, 0.5)]
    elif op == 'mp_nag_mom_update':
        if case['dtype'] == 'bfloat16':
            wb, gb = to_bf16_bits(w), to_bf16_bits(g)
            return [wb, gb, u(-0.5, 0.5), bf16_bits_to_f32(wb).copy()]
        w16 = w.astype(np.float16)
        return [w16, g.astype(np.float16), u(-0.5, 0.5), w16.astype(F)]
    elif op == 'signsgd_update':
        g[::7] = 0                      # sign 0
        st = []
    elif op == 'rmsprop_update':
        st = [u(0, 1)]
    elif op == 'rmspropalex_update':
        gs = u(-0.5, 0.5)
        st = [gs * gs + u(0.01, 1), gs, u(-0.01, 0.01)]   # n - g*g stays positive
    elif op == 'ftml_update':
        st = [u(0.5, 50), u(0, 1), u(-1, 1)]
    else:                               # ftrl: z around +-lamda1 (incl. exact zeros), n >= 0, small g
        z = (u(-2, 2) * F(0.01)).astype(F)
        g = (g * F(0.004)).astype(F)
        z[::11] = 0
        g[::11] = 0
        st = [z, u(0, 0.5)]
    return [w, g] + st


def run_ref(case, ins=None):
    """the reference's own operator on a case: (out, states after)"""
    r = ref()
    assert r is not None and case['dtype'] != 'bfloat16'
    ins = [a.copy() for a in (ins if ins is not None else inputs(case))]
    out = np.zeros_like(ins[0]) if case['distinct_out'] else ins[0]
    r.op_invoke(case['op'], ins, [out], **case['params'])
    return out, ins[2:]


def run_restated(case, ins=None):
    ins = ins if ins is not None else inputs(case)
    return restate(case['op'], ins, case['params'], case['distinct_out'], case['dtype'])


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def fixture_entries(name, case, out, states):
    d = {}
    for tag, a in [('out', out)] + [('s%d' % i, s) for i, s in enumerate(states)]:
        a = np.ascontiguousarray(a)
        if case['n'] <= FULL_MAX:
            d['%s|%s' % (name, tag)] = a
        else:
            d['%s|%s|sha256' % (name, tag)] = digest(a)
            d['%s|%s|head' % (name, tag)] = a[:HEAD].copy()
    return d


def gen_update_ops():
    """tests/golden/update_ops.npz: outputs of the reference's own operators (bfloat16 mp_nag, which
    the reference's CPU type switch does not cover: the restatement, whose float32 part equals the
    reference's float16 cases and whose final rounding is round-to-nearest-even)"""
    d = {}
    for name, case in CASES.items():
        ins = inputs(case)
        out, st = run_restated(case, ins) if case['dtype'] == 'bfloat16' else run_ref(case, ins)
        d.update(fixture_entries(name, case, out, st))
    np.savez_compressed(os.path.join(GOLD, "update_ops.npz"), **d)


if __name__ == "__main__":
    build()
    assert ref() is not None, "build oracle/_ref/libmxref_update.so first: make -f oracle/update_ops.mk"
    gen_update_ops()
    if "--with-trajectories" in sys.argv:
        import ref_python_update
        ref_python_update.gen_trajectories()
