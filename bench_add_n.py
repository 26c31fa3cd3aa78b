#!/usr/bin/env python
"""bench_add_n.py -- add_n on one GPU, against the same sum composed from chained elemwise_add calls.

Dense legs: 64 M elements, float32 at n = 2, 4 and 8 inputs and float16 at n = 8. add_n is one
add_n_kernel launch that reads every input once and writes out once; the chain is n - 1
elemwise_add calls (out = a0 + a1, then out = out + a_i), as a training loop without add_n sums.
Row_sparse leg: 8 inputs of 10 000 random rows each of a 1 M x 512 float32 table (the store's merge).

Parity first: each leg's outputs are checked bit for bit against the numpy restatement
(oracle/golden_add_n.py: the right-nested fold for 2-4 inputs, the left chain otherwise) before
anything is timed. Then add_n and the chain are timed alternately, `--rounds` times each, so both
see the same machine state:
  call_ms     CUDA events around `--iters` calls after a warm-up (ends with a device synchronise)
  kernel_ms   the mean duration of the call's kernels in a torch.profiler run of its own, times the
              kernels per call (add_n 1, the chain n - 1)
GB/s = (n + 1) x element size x elements / median kernel time (the bytes add_n has to move; the chain moves
about 3(n - 1) element sizes per element), and its share of the 3.35 TB/s HBM3 data-sheet figure
of the H100 SXM. The card's name and power limit are read in the same run. One JSON line per leg.

    python bench_add_n.py [--iters 50] [--rounds 3]
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

import golden_add_n as GAN  # noqa: E402

PEAK_GBS = 3350.0
N_DENSE = 64 * 1024 * 1024


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as exc:  # noqa: BLE001
        return "unknown (%s)" % exc, "unknown"


def call_ms(torch, mx, fn, iters):
    for _ in range(5):
        fn()
    mx.nd.waitall()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    mx.nd.waitall()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_ms(torch, mx, fn, iters, names, per_call):
    """the mean duration of the named kernels times the kernels one call launches (the profiler can
    drop an event at the end of its cycle, so the sum over the run is not used)"""
    mx.nd.waitall()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        mx.nd.waitall()
        torch.cuda.synchronize()
    durs = [e.device_time for e in prof.events() if any(k in e.name for k in names)]
    return float(np.mean(durs)) / 1e3 * per_call, len(durs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_add_n.py needs a GPU")
    import anand_mxnet_b200 as mx
    name, power = card()
    tdt = {"float16": torch.float16, "float32": torch.float32}
    for dtype, n in (("float32", 2), ("float32", 4), ("float32", 8), ("float16", 8)):
        gen = torch.Generator(device="cuda").manual_seed(0xADD + n)
        ts = [torch.empty(N_DENSE, dtype=tdt[dtype], device="cuda").uniform_(-4, 4, generator=gen) for _ in range(n)]
        torch.cuda.synchronize()
        arrays = [mx.nd.from_torch(t) for t in ts]
        out = mx.nd.empty((N_DENSE,), mx.gpu(0), dtype)
        chain_out = mx.nd.empty((N_DENSE,), mx.gpu(0), dtype)

        def add_n():
            mx.nd.add_n(*arrays, out=out)

        def chain():
            mx.nd._invoke('elemwise_add', [arrays[0], arrays[1]], out=chain_out)
            for a in arrays[2:]:
                mx.nd._invoke('elemwise_add', [chain_out, a], out=chain_out)

        # parity: both against the restatement on the same values
        raw = [t.cpu().numpy().view(GAN.RAW[dtype]) for t in ts]
        add_n()
        chain()
        assert np.array_equal(out.asnumpy().view(GAN.RAW[dtype]), GAN.fold(raw, dtype)), (dtype, n)
        want_chain = raw[0]
        for r in raw[1:]:
            want_chain = GAN.add(want_chain, r, dtype)
        assert np.array_equal(chain_out.asnumpy().view(GAN.RAW[dtype]), want_chain), (dtype, n)
        del raw, want_chain
        before = mx.base.kernel_launch_count()
        add_n()
        launches = mx.base.kernel_launch_count() - before
        res = {"add_n": [], "chain": []}
        for _ in range(args.rounds):
            for leg, fn, names, per_call in (("add_n", add_n, ["add_n_kernel"], launches),
                                             ("chain", chain, ["ew_kernel"], n - 1)):
                c = call_ms(torch, mx, fn, args.iters)
                k, nk = kernel_ms(torch, mx, fn, args.iters, names, per_call)
                res[leg].append((c, k, nk))
        nbytes = (n + 1) * ts[0].element_size() * N_DENSE
        line = dict(bench="add_n", leg="dense", dtype=dtype, n=n, elements=N_DENSE, bytes=nbytes,
                    launches_per_call=launches, iters=args.iters, parity="ok", card=name, power_limit=power)
        for leg in ("add_n", "chain"):
            calls = [c for c, _, _ in res[leg]]
            kerns = [k for _, k, _ in res[leg]]
            med = float(np.median(kerns))
            line[leg] = dict(call_ms=[round(c, 4) for c in calls], kernel_ms=[round(k, 4) for k in kerns],
                             kernels_profiled=[nk for _, _, nk in res[leg]],
                             gbs=round(nbytes / (med * 1e-3) / 1e9, 1),
                             frac_of_3350_gbs=round(nbytes / (med * 1e-3) / 1e9 / PEAK_GBS, 3))
        line["chain_over_add_n"] = round(float(np.median([k for _, k, _ in res["chain"]]) /
                                               np.median([k for _, k, _ in res["add_n"]])), 2)
        print(json.dumps(line), flush=True)
        del arrays, ts, out, chain_out
        mx.nd.waitall()
        torch.cuda.empty_cache()

    # row_sparse: 8 x 10 000 rows of a 1 M x 512 table
    rng = np.random.default_rng(0xADD)
    shape = (1_000_000, 512)
    ins = [(np.sort(rng.choice(shape[0], 10_000, replace=False)).astype(np.int64),
            rng.standard_normal((10_000, 512)).astype(np.float32)) for _ in range(8)]
    arrays = [mx.nd.sparse.row_sparse_array((rows, ids), shape=shape, ctx=mx.gpu(0)) for ids, rows in ins]
    out = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
    case = dict(dtype='float32', stypes=['row_sparse'] * 8, shape=shape)
    ids, rows = GAN.restate(case, ins)
    mx.nd.sparse.add_n(*arrays, out=out)
    assert np.array_equal(out.indices.asnumpy(), ids)
    assert np.array_equal(out.data.asnumpy().view(np.uint32), rows.view(np.uint32))
    calls = [call_ms(torch, mx, lambda: mx.nd.sparse.add_n(*arrays, out=out), args.iters) for _ in range(args.rounds)]
    nbytes = (80_000 + len(ids)) * 512 * 4
    print(json.dumps(dict(bench="add_n", leg="row_sparse", n=8, rows_per_input=10_000, table=list(shape),
                          union_rows=int(len(ids)), row_bytes=nbytes, call_ms=[round(c, 4) for c in calls],
                          row_gbs=round(nbytes / (float(np.median(calls)) * 1e-3) / 1e9, 1), parity="ok", card=name,
                          power_limit=power)), flush=True)


if __name__ == "__main__":
    main()
