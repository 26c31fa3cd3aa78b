#!/usr/bin/env python
"""bench_update_ops.py -- the single-tensor optimizer operators of the NAG / Signum / RMSProp / FTML /
Ftrl optimizers (update_kernels.cu) on one GPU.

For every operator:
  parity   the seeded 2^20 + 5 element case of oracle/golden_update_ops.py through mx.nd.<op>, bit for
           bit against the numpy restatement of the reference kernel (which tests hold to the
           reference's own code); the run fails if any operator differs
  flat     one call over one 64 M-element tensor (fp32; mp_nag: fp16 weight / grad, fp32 mom /
           weight32), CUDA events over --iters launches after --warmup
  r50      the ResNet-50 parameter set issued one call per key, as the store's updater callback
           does, time per whole set

Prints one JSON line per (operator, workload): algorithmic GB/s (bytes per element: signsgd 12;
signum, nag, mp_nag (fp16), rmsprop 20; ftrl 28; rmspropalex, ftml 36) and its fraction of the
3.35 TB/s H100 SXM data-sheet bandwidth (a data-sheet figure, not measured), with the card's name and
power limit.
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

HBM_DATASHEET_GBS = 3350.0
BYTES = {'signsgd_update': 12, 'signum_update': 20, 'nag_mom_update': 20, 'mp_nag_mom_update': 20,
         'rmsprop_update': 20, 'ftrl_update': 28, 'rmspropalex_update': 36, 'ftml_update': 36}
PARAMS = {'nag_mom_update': dict(lr=0.01, momentum=0.9, wd=1e-4),
          'mp_nag_mom_update': dict(lr=0.01, momentum=0.9, wd=1e-4),
          'signsgd_update': dict(lr=1e-4, wd=1e-4),
          'signum_update': dict(lr=1e-4, momentum=0.9, wd=1e-4),
          'rmsprop_update': dict(lr=1e-4, gamma1=0.9, epsilon=1e-8),
          'rmspropalex_update': dict(lr=1e-4, gamma1=0.95, gamma2=0.9, epsilon=1e-8),
          'ftml_update': dict(lr=0.01, beta1=0.6, beta2=0.999, epsilon=1e-8, t=3),
          'ftrl_update': dict(lr=0.1, lamda1=0.01, beta=1.0)}


def card():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, plim = (r.stdout.strip().split(", ") + ["?", "?"])[:2] if r.returncode == 0 else ("?", "?")
    return name, plim


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elems", type=int, default=64 << 20)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    import anand_mxnet_b200 as mx
    import golden_update_ops as GU
    from bench import resnet50_shapes
    name, plim = card()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    mx.base.set_stream(0, stream.cuda_stream)

    # ------------------------------------------------------------------------------- parity
    failed = []
    for op in GU.OPS:
        for cname, case in sorted(GU.CASES.items()):
            if case['op'] != op or case['n'] != (1 << 20) + 5 or case['dtype'] == 'bfloat16':
                continue
            ins = GU.inputs(case)
            nds = [mx.nd.array(a, mx.gpu(0), a.dtype) for a in ins]
            getattr(mx.nd, op)(*nds, out=nds[0], **case['params'])
            want_out, want_st = GU.run_restated(case, ins)
            ok = np.array_equal(nds[0].asnumpy().view(np.uint8), np.ascontiguousarray(want_out).view(np.uint8))
            ok = ok and all(np.array_equal(s.asnumpy().view(np.uint32), w.view(np.uint32))
                            for s, w in zip(nds[2:], want_st))
            print(json.dumps({"parity": cname, "bit_exact": bool(ok)}))
            if not ok:
                failed.append(cname)

    def timed(call, iters):
        for _ in range(args.warmup):
            call()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(iters):
            call()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    def emit(op, workload, ms, n, extra):
        gbs = BYTES[op] * n / (ms * 1e-3) / 1e9
        print(json.dumps({"metric": "update_op_GBps", "op": op, "workload": workload, "value": gbs,
                          "unit": "GB/s", "ms": ms, "elements": n, "bytes_per_elem": BYTES[op],
                          "frac_of_datasheet_hbm": gbs / HBM_DATASHEET_GBS,
                          "datasheet_hbm_gbs": HBM_DATASHEET_GBS, "datasheet": "not measured",
                          "gpu": name, "power_limit": plim, **extra}))

    def arrays(op, shapes, seed):
        """weight, grad, states as views of one torch buffer per operand"""
        nst = GU.N_STATES[op]
        half = op == 'mp_nag_mom_update'
        gen = torch.Generator(device='cuda').manual_seed(seed)
        total = sum(int(np.prod(s)) for s in shapes)
        out = []
        for i in range(2 + nst):
            dt = torch.float16 if (half and i < 2) else torch.float32
            buf = torch.empty(total + 128 * len(shapes), device='cuda', dtype=dt)
            buf.uniform_(0.0 if i >= 2 else -1.0, 1.0, generator=gen)
            if half and i == 3:
                buf.copy_(out[0][1].to(torch.float32))     # weight32 = weight
            views, off = [], 0
            for s in shapes:
                k = int(np.prod(s))
                views.append(mx.nd.from_torch(buf[off:off + k].view(*s)))
                off += k + ((-k) % 128)
            out.append((views, buf))
        return [[o[0][j] for o in out] for j in range(len(shapes))], out

    r50 = resnet50_shapes()
    r50_n = sum(int(np.prod(s)) for s in r50)
    for op in GU.OPS:
        f = getattr(mx.nd, op)
        p = PARAMS[op]
        sets, keep = arrays(op, [(args.elems,)], 1)
        a = sets[0]
        emit(op, "flat_64M", timed(lambda: f(*a, out=a[0], **p), args.iters), args.elems, {})
        del sets, keep, a
        sets, keep = arrays(op, r50, 2)

        def per_key():
            for a in sets:
                f(*a, out=a[0], **p)
        emit(op, "resnet50_per_key", timed(per_key, max(args.iters // 5, 10)), r50_n,
             {"calls_per_set": len(r50)})
        del sets, keep
        torch.cuda.empty_cache()
    if failed:
        print(json.dumps({"parity_failed": failed}))
        sys.exit(1)


if __name__ == "__main__":
    main()
