#!/usr/bin/env python
"""bench_sparse_grad.py -- a DENSE key with row_sparse gradients: the store step gluon.Trainer runs for
Embedding(sparse_grad=True). Table: dense (1 000 000, 512) fp32 key, 8 values of 10 000 seeded rows
each (bench_rsp.make_inputs), all on one GPU.

Legs:
  (a) update_on_kvstore=False: push, then pull into the 8 row_sparse gradients (ignore_sparse=False);
  (b) fused lazy SGD-momentum on the store: push, then pull into 8 dense weights.
Each leg first checks its result bit for bit against the CPU oracle.

Algorithmic bytes (every row and id read or written once, L = row length):
  (a) sum(nnr)*(4L+8) + union*(4L+8) for the push (sources read, merged value written), plus
      union*(4L+8)*(1+8) for the pull (value read once, written to 8 outs);
  (b) sum(nnr)*(4L+8) + union*16L for the push (sources read, weight and momentum rows read and
      written), plus table*4L*(1+8) for the pull (weight read once, written to 8 outs).
Prints one JSON line per leg with the fraction of 3.35 TB/s (H100 SXM HBM3 data sheet), and the
card name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from bench_rsp import ROWS, ROW_LEN, make_inputs, table_init  # noqa: E402

NVAL = 8
LR, MOM = 0.1, 0.9
PEAK_GBS = 3350.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as exc:  # noqa: BLE001
        return "unknown (%s)" % exc, "unknown"


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def timed(torch, fn, steps, mx):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    mx.nd.waitall()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    mx.nd.waitall()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def leg_a(mx, torch, w, idx, val, steps, warmup):
    import kvoracle as K
    shape = (ROWS, ROW_LEN)
    ctx = mx.gpu(0)
    kv = mx.kv.create('device')
    kv.init('emb', mx.nd.array(w, ctx))
    grads = [mx.nd.sparse.row_sparse_array((val[i], idx[i]), shape=shape, ctx=ctx) for i in range(NVAL)]
    outs = [mx.nd.sparse.zeros('row_sparse', shape, ctx) for _ in range(NVAL)]

    def step():
        kv.push('emb', grads)
        kv.pull('emb', out=outs, ignore_sparse=False)
    step()
    mx.nd.waitall()
    gi, gv = K.get_oracle().rsp_reduce(idx, val)
    ok = all(np.array_equal(o.indices.asnumpy(), gi) and eq(o.data.asnumpy().reshape(gv.shape), gv) for o in outs)
    for _ in range(warmup):
        step()
    ms = timed(torch, step, steps, mx)
    L = ROW_LEN
    nnr = sum(len(i) for i in idx)
    union = len(gi)
    alg = nnr * (4 * L + 8) + union * (4 * L + 8) + union * (4 * L + 8) * (1 + NVAL)
    return dict(leg="a: push + pull into %d row_sparse grads (update_on_kvstore=False)" % NVAL,
                ms=ms, union_rows=union, algorithmic_bytes=alg, parity_ok=bool(ok))


def leg_b(mx, torch, w, idx, val, steps, warmup):
    import kvoracle as K
    shape = (ROWS, ROW_LEN)
    ctx = mx.gpu(0)
    kv = mx.kv.create('device')
    kv.init('emb', mx.nd.array(w, ctx))
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=LR, momentum=MOM, rescale_grad=1.0 / NVAL))
    grads = [mx.nd.sparse.row_sparse_array((val[i], idx[i]), shape=shape, ctx=ctx) for i in range(NVAL)]
    outs = [mx.nd.empty(shape, ctx) for _ in range(NVAL)]

    def step():
        kv.push('emb', grads)
        kv.pull('emb', out=outs)
    step()
    mx.nd.waitall()
    o = K.get_oracle()
    gi, gv = o.rsp_reduce(idx, val)
    sub = np.ascontiguousarray(w[gi])        # the lazy update touches the union's rows only
    mom = np.zeros_like(sub)
    sp = K.scalar_param
    o.sgd_mom_rsp_update(sub, mom, np.arange(len(gi), dtype=np.int64), gv, sp(LR), sp(MOM), sp(0.0),
                         sp(1.0 / NVAL), None)
    ok = True
    for i in (0, NVAL - 1):                  # two outs in full (2 GB each), the others on the union rows
        got = outs[i].asnumpy()
        cold = np.ones(ROWS, bool)
        cold[gi] = False
        ok = ok and eq(got[gi], sub) and eq(got[cold], w[cold])
        del got
    for i in range(1, NVAL - 1):
        ok = ok and eq(outs[i].asnumpy()[gi], sub)
    for _ in range(warmup):
        step()
    ms = timed(torch, step, steps, mx)
    L = ROW_LEN
    nnr = sum(len(i) for i in idx)
    union = len(gi)
    alg = nnr * (4 * L + 8) + union * 16 * L + ROWS * 4 * L * (1 + NVAL)
    return dict(leg="b: push (fused lazy SGD-momentum) + pull into %d dense weights" % NVAL,
                ms=ms, union_rows=union, algorithmic_bytes=alg, parity_ok=bool(ok))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--legs", default="ab")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_sparse_grad.py needs a GPU")
    import anand_mxnet_b200 as mx
    name, power = card()
    w = table_init()
    idx, val, _ = make_inputs(NVAL)
    legs = {"a": leg_a, "b": leg_b}
    for k in args.legs:
        r = legs[k](mx, torch, w, idx, val, args.steps, args.warmup)
        gbs = r["algorithmic_bytes"] / (r["ms"] * 1e-3) / 1e9
        r.update(table=[ROWS, ROW_LEN], values=NVAL, rows_per_value=len(idx[0]), steps=args.steps,
                 achieved_gbs=gbs, frac_of_3350_gbs=gbs / PEAK_GBS, card=name, power_limit=power)
        print(json.dumps(r), flush=True)
        if not r["parity_ok"]:
            sys.exit("leg %s: result differs from the oracle" % k)


if __name__ == "__main__":
    main()
