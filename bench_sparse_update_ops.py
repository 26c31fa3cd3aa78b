#!/usr/bin/env python
"""bench_sparse_update_ops.py -- the row_sparse forms of ftrl_update and _sparse_adagrad_update
(rowsparse_kernels.cu: rsp_row_update_kernel) and GroupAdaGrad's _contrib_group_adagrad_update
(rsp_group_adagrad_kernel) on one GPU, on an embedding table of --rows x --row-len
float32 (default 1 M x 512) with --nnr (default 80 000) seeded unique gradient rows.

Workloads, each timed with CUDA events over --iters launches after --warmup:
  ftrl_rsp           ftrl_update, weight / grad / z / n all row_sparse
  adagrad_rsp        _sparse_adagrad_update, (row_sparse, row_sparse, row_sparse)
  adagrad_dns        _sparse_adagrad_update, (dense, row_sparse, dense)
  store_ftrl_step    one step of a row_sparse key through the store's callback route with the
                     tests/compat Ftrl: a push of 8 values of nnr/8 rows each (disjoint row sets),
                     the merge, the updater's ftrl_update, and a row_sparse_pull of the nnr rows
  group_adagrad_rsp  _contrib_group_adagrad_update, (row_sparse, row_sparse, row_sparse), history
                     (rows, 1)
  group_adagrad_dns  _contrib_group_adagrad_update, (dense, row_sparse, dense)
  store_group_adagrad_step  store_ftrl_step with the tests/compat GroupAdaGrad

Before timing, the first call of every workload is checked bit for bit against the numpy
restatement of the reference kernel (oracle/golden_sparse_update_ops.py, which tests hold to the
reference's own code) on the touched rows, and a sample of untouched rows is checked unchanged; the
run fails if any differs. One JSON line per workload: time, algorithmic GB/s of the update (bytes per
touched element: Ftrl 28 = g 4 + w 4+4 + z 8 + n 8; AdaGrad 20 = g 4 + w 8 + h 8; GroupAdaGrad 12 =
g 4 + w 8; plus per row 8 bytes of id, and for GroupAdaGrad 8 more for its history value) and its
fraction of the 3.35 TB/s H100 SXM data-sheet bandwidth (a bound that was not measured), with the
card's name and power limit.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_DATASHEET_GBS = 3350.0
BYTES = {'ftrl': 28, 'adagrad': 20, 'group_adagrad': 12}
ROW_BYTES = {'ftrl': 8, 'adagrad': 8, 'group_adagrad': 16}
FTRL = dict(lr=0.1, lamda1=0.01, beta=1.0, wd=0.0, rescale_grad=1.0)
ADAGRAD = dict(lr=0.05, epsilon=1e-07, wd=0.0, rescale_grad=1.0)
GROUP_ADAGRAD = dict(lr=0.05, epsilon=1e-05, rescale_grad=1.0)


def card():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, plim = (r.stdout.strip().split(", ") + ["?", "?"])[:2] if r.returncode == 0 else ("?", "?")
    return name, plim


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--row-len", type=int, default=512)
    ap.add_argument("--nnr", type=int, default=80000)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    import anand_mxnet_b200 as mx
    from anand_mxnet_b200.base import _LIB, check_call
    import golden_sparse_update_ops as GS
    import golden_group_adagrad as GG
    name, plim = card()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    mx.base.set_stream(0, stream.cuda_stream)
    R, L, N = args.rows, args.row_len, args.nnr
    shape = (R, L)
    gen = torch.Generator(device='cuda').manual_seed(7)
    rng = np.random.default_rng(7)
    ids_np = np.sort(rng.choice(R, N, replace=False)).astype(np.int64)
    ids = torch.from_numpy(ids_np).cuda()
    cold = torch.from_numpy(np.setdiff1d(rng.choice(R, 4096, replace=False), ids_np)).cuda()

    def uniform(lo, hi, *s):
        return torch.empty(*s, device='cuda').uniform_(lo, hi, generator=gen)

    def rsp(vals, idx):
        """row_sparse array on cuda:0 with `vals` rows at ids `idx` (device copies)"""
        out = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
        d, i = mx.nd.from_torch(vals.contiguous()), mx.nd.from_torch(idx.contiguous())
        check_call(_LIB.MXNDArraySyncCopyFromNDArray(out.handle, d.handle, ctypes.c_int(-1)))
        check_call(_LIB.MXNDArraySyncCopyFromNDArray(out.handle, i.handle, ctypes.c_int(0)))
        return out

    def tensor(a):
        """the rows x row_len values of a table (row_sparse holding every row, or dense)"""
        return mx.nd.to_torch(a.data if a.stype == 'row_sparse' else a).view(R, L)

    def table(t, stype):
        return rsp(t, torch.arange(R, device='cuda')) if stype == 'row_sparse' else mx.nd.from_torch(t)

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

    def parity(workload, op, params, before, after, grad_vals, stypes):
        """before / after: [w, states...] torch tables; the restatement runs on the touched rows"""
        tabs = [t.index_select(0, ids).cpu().numpy() for t in before]
        nnr = [N if s == 'row_sparse' else 0 for s in stypes]
        st = [1 if s == 'row_sparse' else 0 for s in stypes]
        GS.restate(op, st[:1] + [1] + st[1:], [nnr[0], N] + nnr[1:],
                   [tabs[0], grad_vals.cpu().numpy()] + tabs[1:], np.arange(N), N, L, True, **params)
        ok = all(np.array_equal(a.index_select(0, ids).cpu().numpy().view(np.uint32), t.view(np.uint32))
                 for a, t in zip(after, tabs))
        ok = ok and all(torch.equal(a.index_select(0, cold).view(torch.int32), b.index_select(0, cold).view(torch.int32))
                        for a, b in zip(after, before))
        print(json.dumps({"parity": workload, "bit_exact": bool(ok)}))
        if not ok:
            failed.append(workload)

    def emit(workload, kind, ms, extra=None):
        nbytes = N * (BYTES[kind] * L + ROW_BYTES[kind])
        gbs = nbytes / (ms * 1e-3) / 1e9
        print(json.dumps({"metric": "sparse_update_GBps", "workload": workload, "value": gbs, "unit": "GB/s",
                          "ms": ms, "table": [R, L], "rows_updated": N, "bytes": nbytes,
                          "frac_of_datasheet_hbm": gbs / HBM_DATASHEET_GBS,
                          "datasheet_hbm_gbs": HBM_DATASHEET_GBS, "datasheet": "a bound, not measured",
                          "gpu": name, "power_limit": plim, **(extra or {})}))

    gvals = uniform(-1, 1, N, L)
    g = rsp(gvals, ids)
    # ------------------------------------------------------------------------------ operators
    for workload, kind, stypes in [('ftrl_rsp', 'ftrl', ['row_sparse'] * 3),
                                   ('adagrad_rsp', 'adagrad', ['row_sparse'] * 2),
                                   ('adagrad_dns', 'adagrad', ['default'] * 2)]:
        if kind == 'ftrl':
            init = [uniform(-1, 1, R, L), uniform(-0.02, 0.02, R, L), uniform(0, 0.5, R, L)]
            op, params, f = 'ftrl_update', FTRL, mx.nd.ftrl_update
            grad_vals = gvals * 0.004
            grad = rsp(grad_vals, ids)
        else:
            init = [uniform(-1, 1, R, L), uniform(0, 1, R, L)]
            op, params, f = '_sparse_adagrad_update', ADAGRAD, mx.nd.sparse.adagrad_update
            grad_vals, grad = gvals, g
        nds = [table(t, s) for t, s in zip(init, stypes)]
        before = [tensor(a).clone() for a in nds]
        del init
        f(nds[0], grad, *nds[1:], out=nds[0], **params)
        mx.nd.waitall()
        parity(workload, op, params, before, [tensor(a) for a in nds], grad_vals, stypes)
        del before
        emit(workload, kind, timed(lambda: f(nds[0], grad, *nds[1:], out=nds[0], **params)))
        del nds, grad
        torch.cuda.empty_cache()

    # --------------------------------------------------------------- one store step, callback route
    from compat import mxnet_optimizer_update as mxopt
    w0 = uniform(-1, 1, R, L)
    kv = mx.kv.create('device')
    kv.init(0, table(w0, 'row_sparse'))
    kv.set_optimizer(mxopt.Ftrl(learning_rate=FTRL['lr'], lamda1=FTRL['lamda1'], beta=FTRL['beta']))
    parts = np.array_split(rng.permutation(N), 8)
    small = gvals * 0.004
    vals = [rsp(small.index_select(0, torch.from_numpy(np.sort(p)).cuda()),
                ids.index_select(0, torch.from_numpy(np.sort(p)).cuda())) for p in parts]
    out = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
    row_ids = mx.nd.from_torch(ids)

    def store_step():
        kv.push(0, vals)
        kv.row_sparse_pull(0, out=out, row_ids=row_ids)
    store_step()
    mx.nd.waitall()
    z0 = torch.zeros(R, L, device='cuda')
    st = kv._updater.states[0]
    tabs = [w0.index_select(0, ids).cpu().numpy(), np.zeros((N, L), np.float32), np.zeros((N, L), np.float32)]
    GS.restate('ftrl_update', [1, 1, 1, 1], [N, N, N, N], [tabs[0], small.cpu().numpy()] + tabs[1:],
               np.arange(N), N, L, True, **FTRL)
    ok = np.array_equal(mx.nd.to_torch(out.data).view(N, L).cpu().numpy().view(np.uint32), tabs[0].view(np.uint32))
    ok = ok and all(np.array_equal(tensor(s).index_select(0, ids).cpu().numpy().view(np.uint32), t.view(np.uint32))
                    for s, t in zip(st, tabs[1:]))
    ok = ok and all(torch.equal(tensor(s).index_select(0, cold), z0.index_select(0, cold)) for s in st)
    print(json.dumps({"parity": "store_ftrl_step", "bit_exact": bool(ok)}))
    if not ok:
        failed.append("store_ftrl_step")
    del z0
    emit("store_ftrl_step", 'ftrl', timed(store_step),
         {"note": "whole step: push of 8 values + merge + callback ftrl_update + row_sparse_pull; "
                  "GB/s counts the update's bytes only"})
    del kv, vals, out, st
    torch.cuda.empty_cache()

    # ------------------------------------------------------------------------------ GroupAdaGrad
    def hist(t, stype):
        """a (rows, 1) history: row_sparse holding every row, or dense"""
        if stype == 'default':
            return mx.nd.from_torch(t)
        out = mx.nd.sparse.zeros('row_sparse', (R, 1), mx.gpu(0))
        d, i = mx.nd.from_torch(t), mx.nd.from_torch(torch.arange(R, device='cuda'))
        check_call(_LIB.MXNDArraySyncCopyFromNDArray(out.handle, d.handle, ctypes.c_int(-1)))
        check_call(_LIB.MXNDArraySyncCopyFromNDArray(out.handle, i.handle, ctypes.c_int(0)))
        return out

    def hvals(a):
        return mx.nd.to_torch(a.data if a.stype == 'row_sparse' else a).view(R, 1)

    def group_parity(workload, w_before, h_before, w, h, h_cold):
        """the restatement on the touched rows; sampled cold rows of w and h unchanged"""
        tw, th = w_before.index_select(0, ids).cpu().numpy(), h_before.index_select(0, ids).cpu().numpy()
        GG.restate(GG.OP, [1, 1, 1], [N, N, N], [tw, gvals.cpu().numpy(), th], np.arange(N), N, L, True,
                   **GROUP_ADAGRAD)
        ok = all(np.array_equal(a.index_select(0, ids).cpu().numpy().view(np.uint32), t.view(np.uint32))
                 for a, t in ((w, tw), (h, th)))
        ok = ok and torch.equal(w.index_select(0, cold).view(torch.int32),
                                w_before.index_select(0, cold).view(torch.int32))
        ok = ok and torch.equal(h.index_select(0, cold).view(torch.int32), h_cold.view(torch.int32))
        print(json.dumps({"parity": workload, "bit_exact": bool(ok)}))
        if not ok:
            failed.append(workload)

    f = mx.nd.contrib.group_adagrad_update
    for workload, stype in [('group_adagrad_rsp', 'row_sparse'), ('group_adagrad_dns', 'default')]:
        w0, h0 = uniform(-1, 1, R, L), uniform(0, 1, R, 1)
        w, h = table(w0, stype), hist(h0, stype)
        w_before, h_before = tensor(w).clone(), hvals(h).clone()
        del w0, h0
        f(w, g, h, out=w, **GROUP_ADAGRAD)
        mx.nd.waitall()
        group_parity(workload, w_before, h_before, tensor(w), hvals(h), h_before.index_select(0, cold))
        del w_before, h_before
        emit(workload, 'group_adagrad', timed(lambda: f(w, g, h, out=w, **GROUP_ADAGRAD)))
        del w, h
        torch.cuda.empty_cache()

    from compat import mxnet_optimizer_contrib as mxopt_contrib
    w0 = uniform(-1, 1, R, L)
    kv = mx.kv.create('device')
    kv.init(0, table(w0, 'row_sparse'))
    kv.set_optimizer(mxopt_contrib.GroupAdaGrad(learning_rate=GROUP_ADAGRAD['lr'],
                                                eps=GROUP_ADAGRAD['epsilon']))
    vals = [rsp(gvals.index_select(0, torch.from_numpy(np.sort(p)).cuda()),
                ids.index_select(0, torch.from_numpy(np.sort(p)).cuda())) for p in parts]
    out = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
    store_step()
    mx.nd.waitall()
    # the pulled rows and the history's touched rows against the restatement; cold history rows 0
    w_after = w0.clone()
    w_after.index_copy_(0, ids, mx.nd.to_torch(out.data).view(N, L))
    group_parity("store_group_adagrad_step", w0, torch.zeros(R, 1, device='cuda'), w_after,
                 hvals(kv._updater.states[0]), torch.zeros(len(cold), 1, device='cuda'))
    del w_after
    emit("store_group_adagrad_step", 'group_adagrad', timed(store_step),
         {"note": "whole step: push of 8 values + merge + callback group_adagrad_update + "
                  "row_sparse_pull; GB/s counts the update's bytes only"})
    if failed:
        print(json.dumps({"parity_failed": failed}))
        sys.exit(1)


if __name__ == "__main__":
    main()
