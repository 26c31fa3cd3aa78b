"""TEST INFRASTRUCTURE ONLY -- the NAG / Signum / RMSProp / FTML / Ftrl operators with a dense weight,
dense states and a row_sparse gradient, as the reference runs them: none of these operators registers
an FComputeEx for that storage pair, so imperative dispatch takes DispatchMode::kFComputeFallback
(src/imperative/imperative_utils.h:185-198). The fallback densifies the gradient with
CastStorageRspDnsImpl (src/operator/tensor/cast_storage-inl.h:139-163: the dense array is filled
with +0, then each stored row is copied to its row id) and runs the dense FCompute<cpu> over the
whole table. `densify` restates that cast in numpy (a zero fill and a row copy, no arithmetic);
each output is then the reference's own compiled dense operator (golden_update_ops.ref(), i.e.
oracle/_ref/libmxref_update.so) on the densified gradient.

Writes tests/golden/rsp_grad_update_ops.npz:

    make -f oracle/update_ops.mk && python oracle/golden_rsp_grad_update_ops.py

Inputs are regenerated from each case's seed wherever the fixture is read, so the fixture holds
outputs only: in full up to FULL_MAX elements, else a SHA-256 plus the first HEAD elements.
"""
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import golden_update_ops as GU  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
F = np.float32
OPS = [op for op in GU.OPS if op != 'mp_nag_mom_update']
FULL_MAX = 1024
HEAD = 16

# row_len 1 (rank 1), 5 (the scalar path), 64 and 512 (the 16-byte path), and a rank-3 weight
# (row_len 20) as in the reference's test_rms
SHAPES = {'r1': (37,), 'r5': (23, 5), 'r64': (40, 64), 'r512': (9, 512), 'rank3': (3, 4, 5)}
ROWSETS = ['some', 'none', 'all', 'ends']


def densify(shape, ids, vals):
    """CastStorageRspDnsImpl: +0.0f everywhere, then the stored rows copied to their ids"""
    d = np.zeros(shape, F)
    if len(ids):
        d[np.asarray(ids, np.int64)] = vals
    return d


def _cases():
    c = {}
    for op in OPS:
        variants = GU.VARIANTS[op]
        last = sorted(v for v in variants if v.startswith('clip_wd'))[-1]   # clip, rescale and wd
        for sname in SHAPES:
            for vname in sorted(variants):        # every hyper-parameter set on a partial row set
                c['%s_%s_%s_some' % (op, vname, sname)] = dict(op=op, shape=SHAPES[sname], rows='some',
                                                               params=variants[vname], distinct_out=False)
            for rows in ROWSETS[1:]:              # the edge row sets with clip, rescale and wd
                c['%s_%s_%s_%s' % (op, last, sname, rows)] = dict(op=op, shape=SHAPES[sname], rows=rows,
                                                                  params=variants[last], distinct_out=False)
        for sname in ('r5', 'r64'):               # out as a separate array
            c['%s_%s_%s_some_distinct_out' % (op, last, sname)] = dict(
                op=op, shape=SHAPES[sname], rows='some', params=variants[last], distinct_out=True)
    return c


CASES = _cases()


def inputs(case):
    """(weight, gradient ids, gradient rows, [states]) of a case, regenerated from its seed: the dense
    operands of golden_update_ops.inputs at the table's size, reshaped; the stored rows are the
    gradient's rows `ids` (ascending)"""
    shape = case['shape']
    n = int(np.prod(shape))
    ins = GU.inputs(dict(op=case['op'], dtype='float32', n=n))
    w, g = ins[0].reshape(shape), ins[1].reshape(shape)
    states = [s.reshape(shape) for s in ins[2:]]
    rows = shape[0]
    rng = np.random.default_rng(zlib.crc32(('%s|%s|%s' % (case['op'], shape, case['rows'])).encode()))
    if case['rows'] == 'none':
        ids = np.zeros(0, np.int64)
    elif case['rows'] == 'all':
        ids = np.arange(rows, dtype=np.int64)
    elif case['rows'] == 'ends':
        ids = np.unique([0, rows - 1]).astype(np.int64)
    else:
        ids = np.sort(rng.choice(rows, max(1, rows // 3), replace=False)).astype(np.int64)
    return w, ids, g[ids].copy(), states


def run_ref(case):
    """the reference's own dense operator on the densified gradient: (out, states after)"""
    w, ids, vals, states = inputs(case)
    ins = [w.reshape(-1), densify(case['shape'], ids, vals).reshape(-1)] + [s.reshape(-1) for s in states]
    out, st = GU.run_ref(dict(op=case['op'], dtype='float32', params=case['params'],
                              distinct_out=case['distinct_out']), ins)
    return out.reshape(case['shape']), [s.reshape(case['shape']) for s in st]


def run_restated(case):
    """golden_update_ops.restate on the densified gradient"""
    w, ids, vals, states = inputs(case)
    out, st = GU.restate(case['op'], [w, densify(case['shape'], ids, vals)] + states, case['params'],
                         case['distinct_out'])
    return out, st


def put(d, key, a):
    a = np.ascontiguousarray(a)
    if a.size <= FULL_MAX:
        d[key] = a
    else:
        d[key + '|sha256'] = GU.digest(a)
        d[key + '|head'] = a.reshape(-1)[:HEAD].copy()


def matches(gold, key, a):
    """a equals the fixture entry `key` bit for bit (in full, or by digest and head)"""
    want = {}
    put(want, key, a)
    return all(k in gold.files and np.array_equal(np.ascontiguousarray(v).view(np.uint8),
                                                  np.ascontiguousarray(gold[k]).view(np.uint8))
               for k, v in want.items())


def entries(name, out, states):
    d = {}
    put(d, '%s|out' % name, out)
    for i, s in enumerate(states):
        put(d, '%s|s%d' % (name, i), s)
    return d


def gen():
    d = {}
    for name, case in CASES.items():
        d.update(entries(name, *run_ref(case)))
    np.savez_compressed(os.path.join(GOLD, "rsp_grad_update_ops.npz"), **d)
    return d


if __name__ == "__main__":
    GU.build()
    assert GU.ref() is not None, "build oracle/_ref/libmxref_update.so first: make -f oracle/update_ops.mk"
    print(len(CASES), "cases,", len(gen()), "arrays")
