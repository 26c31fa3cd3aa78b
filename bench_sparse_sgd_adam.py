#!/usr/bin/env python
"""bench_sparse_sgd_adam.py -- sgd_mom_update and adam_update with a row_sparse gradient: the lazy
form on a row_sparse weight that holds every row and on a dense weight (rowsparse_kernels.cu:
rsp_row_update_kernel), and the standard form on a dense weight (update_rsp_grad_kernels.cu:
update_kernel<OP, float, true> after the row map), on one GPU, on an embedding table of
--rows x --row-len float32 (default 1 M x 512) with --nnr (default 1 % of the rows) seeded unique
gradient rows.

Workloads, each timed with CUDA events over --iters calls after --warmup:
  sgd_mom_rsp   sgd_mom_update, weight / grad / mom all row_sparse, lazy_update=True
  sgd_mom_dns   the same call on a dense weight and momentum: the same kernel, the same work
  sgd_mom_std   the dense-weight call with lazy_update=False: every row of the table moves, rows
                absent from the gradient with g = 0
  adam_rsp      adam_update, weight / grad / mean / var all row_sparse, lazy_update=True
  adam_dns      the same call on a dense weight, mean and var
  adam_std      the dense-weight call with lazy_update=False
  state_fill    the first-use fill of one row_sparse state that holds no rows: all rows allocated,
                zeroed and given ids 0..rows-1 (a sgd_mom_update with an empty gradient, which
                changes nothing else); timed per call including a fresh empty state each time

Before timing, the first call of every update workload is checked bit for bit against the C
restatement of the reference's kernels (oracle/kvoracle.c, which the tests hold to the reference's
own code) on the touched rows and on a sample of untouched rows (unchanged by the lazy form); the
fill is checked to leave every row zero. The run fails if any differs. One JSON line per workload:
time, algorithmic GB/s (bytes per touched element: SGD-momentum 20 = g 4 + w 8 + mom 8; Adam 28 =
g 4 + w 8 + mean 8 + var 8; plus 8 bytes of id per row. The standard form touches every table
element without reading a gradient there, 4 bytes fewer, and reads the gradient's rows once and
the row map, 8 bytes per table row and 4 per gradient row; the fill writes rows x (row_len x 4 +
8)) and its fraction of the 3.35 TB/s H100 SXM data-sheet bandwidth (a bound that was not
measured), with the card's name and power limit.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

HBM_DATASHEET_GBS = 3350.0
BYTES = {'sgd_mom': 20, 'adam': 28}
SGD_MOM = dict(lr=0.1, momentum=0.9, wd=1e-4, rescale_grad=1.0, lazy_update=True)
ADAM = dict(lr=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, wd=1e-4, rescale_grad=1.0, lazy_update=True)


def card():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, plim = (r.stdout.strip().split(", ") + ["?", "?"])[:2] if r.returncode == 0 else ("?", "?")
    return name, plim


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--row-len", type=int, default=512)
    ap.add_argument("--nnr", type=int, default=0, help="gradient rows (default: 1 %% of --rows)")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    import anand_mxnet_b200 as mx
    from anand_mxnet_b200.base import _LIB, check_call
    import kvoracle as K
    oracle = K.get_oracle()
    name, plim = card()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    mx.base.set_stream(0, stream.cuda_stream)
    R, L = args.rows, args.row_len
    N = args.nnr or max(1, R // 100)
    shape = (R, L)
    gen = torch.Generator(device='cuda').manual_seed(11)
    rng = np.random.default_rng(11)
    ids_np = np.sort(rng.choice(R, N, replace=False)).astype(np.int64)
    ids = torch.from_numpy(ids_np).cuda()
    cold = torch.from_numpy(np.setdiff1d(rng.choice(R, 4096, replace=False), ids_np)).cuda()

    def uniform(lo, hi, *s):
        return torch.empty(*s, device='cuda').uniform_(lo, hi, generator=gen)

    def rsp(vals, idx):
        out = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
        d, i = mx.nd.from_torch(vals.contiguous()), mx.nd.from_torch(idx.contiguous())
        check_call(_LIB.MXNDArraySyncCopyFromNDArray(out.handle, d.handle, ctypes.c_int(-1)))
        check_call(_LIB.MXNDArraySyncCopyFromNDArray(out.handle, i.handle, ctypes.c_int(0)))
        return out

    def tensor(a):
        return mx.nd.to_torch(a.data if a.stype == 'row_sparse' else a).view(R, L)

    def table(t, stype):
        return rsp(t, torch.arange(R, device='cuda')) if stype == 'row_sparse' else mx.nd.from_torch(t.clone())

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

    def emit(workload, nbytes, ms, extra=None):
        gbs = nbytes / (ms * 1e-3) / 1e9
        print(json.dumps({"metric": "sparse_sgd_adam_GBps", "workload": workload, "value": gbs, "unit": "GB/s",
                          "ms": ms, "table": [R, L], "rows_updated": N, "bytes": nbytes,
                          "frac_of_datasheet_hbm": gbs / HBM_DATASHEET_GBS,
                          "datasheet_hbm_gbs": HBM_DATASHEET_GBS, "datasheet": "a bound, not measured",
                          "gpu": name, "power_limit": plim, **(extra or {})}), flush=True)

    gvals = uniform(-1, 1, N, L)
    g = rsp(gvals, ids)
    g_np = gvals.cpu().numpy()
    for kind, lazy_params, nst in (('sgd_mom', SGD_MOM, 1), ('adam', ADAM, 2)):
        op = getattr(mx.nd.sparse, kind + '_update')
        for stype, lazy in (('row_sparse', True), ('default', True), ('default', False)):
            params = dict(lazy_params, lazy_update=lazy)
            w0 = uniform(-1, 1, R, L)
            s0 = [uniform(-0.1, 0.1, R, L), uniform(0, 0.01, R, L)][:nst]
            w = table(w0, stype)
            sts = [table(s, stype) for s in s0]
            # the standard form moves every row: the touched rows (first) and the untouched sample
            # form one sub-table for the oracle
            checked = ids if lazy else torch.cat([ids, cold])
            before = [t.index_select(0, checked).cpu().numpy() for t in [w0] + s0]
            op(w, g, *sts, out=w, **params)
            mx.nd.waitall()
            after = [tensor(a) for a in [w] + sts]
            kw = dict(lr=params['lr'], wd=params['wd'])
            if kind == 'sgd_mom':
                (oracle.sgd_mom_rsp_update if lazy else oracle.sgd_mom_std_rsp_update)(
                    before[0], before[1], np.arange(N), g_np, momentum=0.9, **kw)
            else:
                (oracle.adam_rsp_update if lazy else oracle.adam_std_rsp_update)(*before, np.arange(N), g_np, **kw)
            ok = all(np.array_equal(a.index_select(0, checked).cpu().numpy().view(np.uint32), b.view(np.uint32))
                     for a, b in zip(after, before))
            if lazy:
                ok = ok and all(torch.equal(a.index_select(0, cold).view(torch.int32),
                                            b.index_select(0, cold).view(torch.int32))
                                for a, b in zip(after, [w0] + s0))
            workload = "%s_%s" % (kind, 'std' if not lazy else 'rsp' if stype == 'row_sparse' else 'dns')
            print(json.dumps({"parity": workload, "bit_exact": bool(ok)}), flush=True)
            if not ok:
                failed.append(workload)
            ms = timed(lambda: op(w, g, *sts, out=w, **params))
            if lazy:
                nbytes = N * (BYTES[kind] * L + 8)
            else:
                nbytes = R * L * (BYTES[kind] - 4) + N * (L * 4 + 8 + 4) + R * 8
            emit(workload, nbytes, ms, {"weight_stype": stype, "lazy_update": lazy})
            del w, sts, after, w0, s0
            torch.cuda.empty_cache()
    # first-use fill of one row_sparse momentum that holds no rows
    w = table(uniform(-1, 1, R, L), 'row_sparse')
    empty_g = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
    m = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
    mx.nd.sparse.sgd_mom_update(w, empty_g, m, out=w, **SGD_MOM)
    mx.nd.waitall()
    ok = m.indices.shape[0] == R and bool((tensor(m) == 0).all()) and \
        torch.equal(mx.nd.to_torch(m.indices), torch.arange(R, device='cuda'))
    print(json.dumps({"parity": "state_fill", "ok": bool(ok)}), flush=True)
    if not ok:
        failed.append("state_fill")
    del m
    ms = timed(lambda: mx.nd.sparse.sgd_mom_update(w, empty_g, mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0)),
                                                   out=w, **SGD_MOM))
    emit("state_fill", R * (L * 4 + 8), ms, {"note": "one state, includes its allocation"})
    if failed:
        sys.exit("parity failed: %s" % failed)


if __name__ == "__main__":
    main()
