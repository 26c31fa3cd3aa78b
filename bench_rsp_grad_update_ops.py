#!/usr/bin/env python
"""bench_rsp_grad_update_ops.py -- nag_mom_update, signsgd_update, signum_update, rmsprop_update,
rmspropalex_update, ftml_update and ftrl_update with a dense weight, dense states and a row_sparse
gradient (update_kernels.cu: update_kernel<OP, float, true> after the row map of rowsparse_kernels.cu),
on one GPU, on an embedding table of --rows x --row-len float32 (default 1 M x 512), with 1 % of the
rows in the gradient (10 485 of 1 M) and with every row.

For each operator and density, timed with CUDA events over --iters calls after --warmup:
  a  rsp_pass   the operator on the row_sparse gradient: every row of the table moves, absent rows
                with g = +0.0f, without a dense gradient in memory
  b  densify    the reference's route: the gradient cast to a dense array on the GPU (copyto: a zero
                fill and a row scatter, CastStorageRspDnsImpl), then the dense operator
  c  dense      the dense operator on an already dense gradient
Before timing, (a) and (b) run once from the same inputs on separate copies, and every output (the
weight and each state) must be equal bit for bit; the run fails otherwise.

Byte model per table element (what the algorithm must move): the weight read (every operator here
reads it), out written, 8 B per state (read + write), and for
  a  + 4 B per stored gradient element, 8 B per stored id, and per table row 8 B of row map
     (memset, then read) + per stored row 4 B of scatter
  b  + 4 B of gradient read, + the cast: 4 B per table element of zero fill, 8 B per stored gradient
     element (read + write) and 8 B per stored id
  c  + 4 B of gradient read
One JSON line per operator, density and route: ms, algorithmic GB/s and its share of the 3.35 TB/s
H100 SXM data-sheet bandwidth (a bound that was not measured), with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

HBM_DATASHEET_GBS = 3350.0
# operator: (hyper-parameters, value range of each state)
OPS = {
    'nag_mom_update': (dict(lr=0.05, momentum=0.9, wd=1e-3, rescale_grad=1.0), [(-0.5, 0.5)]),
    'signsgd_update': (dict(lr=0.01, wd=1e-3), []),
    'signum_update': (dict(lr=0.01, momentum=0.9, wd=1e-3, wd_lh=0.01), [(-0.5, 0.5)]),
    'rmsprop_update': (dict(lr=0.001, gamma1=0.9, epsilon=1e-8, wd=1e-3), [(0, 1)]),
    'rmspropalex_update': (dict(lr=0.001, gamma1=0.95, gamma2=0.9, epsilon=1e-8, wd=1e-3),
                           [(1, 2), (-0.5, 0.5), (-0.01, 0.01)]),
    'ftml_update': (dict(lr=0.01, beta1=0.6, beta2=0.999, epsilon=1e-8, wd=1e-3, t=3),
                    [(0.5, 50), (0, 1), (-1, 1)]),
    'ftrl_update': (dict(lr=0.1, lamda1=0.01, beta=1, wd=1e-3), [(-0.02, 0.02), (0, 0.5)]),
}


def card():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, plim = (r.stdout.strip().split(", ") + ["?", "?"])[:2] if r.returncode == 0 else ("?", "?")
    return name, plim


def model_bytes(route, n, rows, nnr, row_len, nstates):
    dense = n * (4 + 4 + 8 * nstates)
    if route == 'rsp_pass':
        return dense + nnr * row_len * 4 + nnr * 8 + rows * 8 + nnr * 4
    if route == 'densify':
        return dense + n * 4 + n * 4 + nnr * row_len * 8 + nnr * 8
    return dense + n * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--row-len", type=int, default=512)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ops", default=",".join(OPS))
    args = ap.parse_args()
    import torch
    import anand_mxnet_b200 as mx
    name, plim = card()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    mx.base.set_stream(0, stream.cuda_stream)
    R, L = args.rows, args.row_len
    shape = (R, L)
    gen = torch.Generator(device='cuda').manual_seed(17)

    def uniform(lo, hi, *s):
        return torch.empty(*s, device='cuda').uniform_(lo, hi, generator=gen)

    def rsp(vals, idx):
        return mx.nd.sparse.row_sparse_array((mx.nd.from_torch(vals.contiguous()), mx.nd.from_torch(idx)),
                                             shape=shape, ctx=mx.gpu(0))

    def timed(call):
        for _ in range(args.warmup):
            call()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.iters):
            call()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.iters

    failed = []
    for nnr in (max(1, R // 100), R):
        ids = torch.randperm(R, device='cuda', generator=gen)[:nnr].sort().values
        g = rsp(uniform(-1, 1, nnr, L), ids)
        gd = mx.nd.empty(shape, mx.gpu(0))
        g.copyto(gd)
        for op in args.ops.split(','):
            params, ranges = OPS[op]
            f = getattr(mx.nd, op)
            init = [uniform(-1, 1, R, L)] + [uniform(lo, hi, R, L) for lo, hi in ranges]
            a = [mx.nd.from_torch(t.clone()) for t in init]
            b = [mx.nd.from_torch(t.clone()) for t in init]
            del init
            f(a[0], g, *a[1:], out=a[0], **params)
            g.copyto(gd)
            f(b[0], gd, *b[1:], out=b[0], **params)
            mx.nd.waitall()
            ok = all(torch.equal(mx.nd.to_torch(x).view(torch.int32), mx.nd.to_torch(y).view(torch.int32))
                     for x, y in zip(a, b))
            print(json.dumps({"parity": op, "rows_in_gradient": nnr, "rsp_pass_equals_densify": bool(ok)}),
                  flush=True)
            if not ok:
                failed.append((op, nnr))
            del b
            routes = {
                'rsp_pass': lambda: f(a[0], g, *a[1:], out=a[0], **params),
                'densify': lambda: (g.copyto(gd), f(a[0], gd, *a[1:], out=a[0], **params)),
                'dense': lambda: f(a[0], gd, *a[1:], out=a[0], **params),
            }
            for route, call in routes.items():
                ms = timed(call)
                nbytes = model_bytes(route, R * L, R, nnr, L, len(ranges))
                gbs = nbytes / (ms * 1e-3) / 1e9
                print(json.dumps({"metric": "rsp_grad_update_GBps", "op": op, "route": route, "ms": ms,
                                  "value": gbs, "unit": "GB/s", "table": [R, L], "rows_in_gradient": nnr,
                                  "bytes": nbytes, "bytes_per_elem": nbytes / (R * L),
                                  "frac_of_datasheet_hbm": gbs / HBM_DATASHEET_GBS,
                                  "datasheet_hbm_gbs": HBM_DATASHEET_GBS, "datasheet": "a bound, not measured",
                                  "gpu": name, "power_limit": plim}), flush=True)
            del a, routes
            torch.cuda.empty_cache()
        del g, gd
        torch.cuda.empty_cache()
    if failed:
        sys.exit("parity failed: %s" % failed)


if __name__ == "__main__":
    main()
