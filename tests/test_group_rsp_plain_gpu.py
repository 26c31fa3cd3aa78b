"""Rank-per-GPU store, the cases beside the fused dense / lazy-sparse hot path.

2-bit gradient compression (comm.h:552-596): every rank quantises its gradient with its own
residual, all ranks decode and sum every rank's words in rank order -- words, residual carry-over
and the SGD step on the merged gradient bit-exact against the oracle.

Row_sparse keys WITHOUT a fused lazy optimizer: plain assignment
(kvstore_local.h:237-243: stored = merged) and the standard -- non-lazy -- sparse update
(optimizer_op.cc:108-139, 291-320). Every rank builds the same merged gradient (union of all
ranks' rows, summed in rank order, peers read through IPC) and keeps a replica of the stored value.
Ids and rows bit-exact against the oracle. One process per GPU, gloo bootstrap on 127.0.0.1."""
import os
import socket

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [root, os.path.join(root, "oracle")]
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["LOCAL_RANK"] = str(rank)
    os.environ["B200KV_IPC_ARENA_MB"] = "512"
    os.environ["B200KV_NVLS"] = "0"
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    errors = []
    try:
        import kvoracle as K
        import anand_mxnet_b200 as mx
        mx.dist.init_peer_group(rank, symmetric_memory=False)
        ctx = mx.gpu(rank)
        o = K.get_oracle()
        sp = K.scalar_param
        shape = (1203, 24)

        def rsp_of(r, t):
            rg = np.random.default_rng(700 + 13 * r + t)
            n = 0 if (r == 1 and t == 1) else 90                # one rank pushes an all-zero gradient once
            idx = np.sort(rg.choice(shape[0], n, replace=False)).astype(np.int64)
            return idx, rg.uniform(-1, 1, (n, shape[1])).astype(np.float32)

        def push(kv, t):
            idx, val = rsp_of(rank, t)
            if len(idx):
                g = mx.nd.sparse.row_sparse_array((val, idx), shape=shape, ctx=ctx)
            else:
                g = mx.nd.sparse.zeros('row_sparse', shape, ctx)
            kv.push('emb', g)
            parts = [p for p in (rsp_of(r, t) for r in range(world)) if len(p[0])]
            return o.rsp_reduce([p[0] for p in parts], [p[1] for p in parts])

        def pull_all(kv):
            out = mx.nd.sparse.zeros('row_sparse', shape, ctx)
            kv.row_sparse_pull('emb', out=out, row_ids=mx.nd.array(np.arange(shape[0]), ctx, np.int64))
            return out.asnumpy()

        # ---- plain assignment: stored value = merged gradient of the last push
        kv = mx.kv.create('device')
        kv.init('emb', mx.nd.sparse.zeros('row_sparse', shape, ctx))
        for t in range(3):
            gi, gv = push(kv, t)
            want = np.zeros(shape, np.float32)
            want[gi] = gv
            got = pull_all(kv)
            if not np.array_equal(got.view(np.uint32), want.view(np.uint32)):
                errors.append("assign step %d" % t)
        # ---- standard (non-lazy) SGD with momentum: every row of the table moves each step
        w = np.random.default_rng(71).uniform(-1, 1, shape).astype(np.float32)
        m = np.zeros(shape, np.float32)
        kv = mx.kv.create('device')
        kv.init('emb', mx.nd.array(w, ctx).tostype('row_sparse'))
        kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9, wd=1e-3, rescale_grad=0.5,
                                          lazy_update=False))
        for t in range(3):
            gi, gv = push(kv, 10 + t)
            o.sgd_mom_std_rsp_update(w, m, gi, gv, sp(0.1), sp(0.9), sp(1e-3), sp(0.5), None)
            got = pull_all(kv)
            if not np.array_equal(got.view(np.uint32), w.view(np.uint32)):
                errors.append("std sgd step %d" % t)
        # ---- 2-bit gradient compression, several keys per call, SGD-momentum on the store
        shapes = [(1003,), (64, 33), (70001,), (5,)]
        thr = 0.25
        kv = mx.kv.create('device')
        kv.set_gradient_compression({'type': '2bit', 'threshold': thr})
        keys = list(range(len(shapes)))
        w0 = [np.random.default_rng(90 + k).uniform(-1, 1, s).astype(np.float32) for k, s in enumerate(shapes)]
        kv.init(keys, [mx.nd.array(x, ctx) for x in w0])
        kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9, wd=1e-4, rescale_grad=1.0 / world))
        model = K.LocalKVStoreModel('device')
        for k in keys:
            model.init(k, w0[k])
        model.set_optimizer('sgd', lr=0.1, momentum=0.9, wd=1e-4, rescale_grad=1.0 / world)
        res = [[np.zeros(int(np.prod(s)), np.float32) for _ in range(world)] for s in shapes]
        outs = [mx.nd.empty(s, ctx) for s in shapes]
        for step in range(4):
            def grad(r, k):
                return np.random.default_rng(4000 + 100 * step + 10 * r + k).uniform(-0.4, 0.4, shapes[k]).astype(np.float32)
            if step == 3:
                # a float16 value on the last key: every rank refuses the call before any key's
                # residual moves, so this step still follows the trajectory that never saw it
                bad = [mx.nd.array(grad(rank, k), ctx) for k in keys[:-1]]
                bad.append(mx.nd.array(grad(rank, keys[-1]).astype(np.float16), ctx, 'float16'))
                try:
                    kv.pushpull(keys, bad, out=outs)
                    errors.append("2bit: a float16 value on a float32 key was accepted")
                except mx.MXNetError as e:
                    if "push: dtype mismatch for key %d" % keys[-1] not in str(e):
                        errors.append("2bit: unexpected refusal %s" % e)
            kv.pushpull(keys, [mx.nd.array(grad(rank, k), ctx) for k in keys], out=outs)
            for k, s in enumerate(shapes):
                n = int(np.prod(s))
                deq = []
                for r in range(world):
                    comp = o.quantize_2bit(grad(r, k).ravel(), res[k][r], thr)
                    deq.append(o.dequantize_2bit(comp, n, thr))
                model.push(k, [o.reduce(deq, 'device').reshape(s)])     # the merged gradient, one value
                if not np.array_equal(outs[k].asnumpy().view(np.uint32), model.pull(k).view(np.uint32)):
                    errors.append("2bit step %d key %d" % (step, k))
        mx.nd.waitall()
        dist.barrier()
        mx.dist.destroy_peer_group()
    except Exception:  # noqa
        import traceback
        errors.append(traceback.format_exc())
    finally:
        q.put((rank, errors))
        dist.destroy_process_group()


def test_group_row_sparse_plain_and_compression():
    import torch
    import torch.multiprocessing as mp
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = []
    try:
        results = [q.get(timeout=300) for _ in procs]
    finally:
        for p in procs:
            p.join(timeout=30)
            if p.is_alive():
                p.kill()
    for rank, errors in results:
        assert not errors, (rank, errors[:3])
