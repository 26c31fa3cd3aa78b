"""Measures the GPU normal sampler (_random_normal) and one SGLD step, on one GPU.

    python bench_random.py [--iters 50]

Prints one JSON line per measurement: _random_normal float32 at 64 M, 1 M and 10 K elements (ms per
call, GB/s of writes, share of the 3.35 TB/s HBM3 data-sheet figure), the same launch with the
reference's per-thread store order (each thread storing as it draws), and one SGLD step over the
ResNet-50 parameter set through a local updater. Before timing, the staged and per-thread orders
are checked to write the same bits from the same generator state. Times are a host clock
around `iters` back-to-back calls that ends in a device synchronise, after a warm-up; the card's name and power limit are
printed with them."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import anand_mxnet_b200 as mx  # noqa: E402
from bench import resnet50_shapes  # noqa: E402

DATASHEET_BPS = 3.35e12


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        return "unknown"


def sync():
    mx.nd.waitall()


def timed(fn, iters):
    """ms per call: a host clock around `iters` calls that ends in a device synchronise"""
    fn()
    sync()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    sync()
    return (time.perf_counter() - t0) * 1e3 / iters


def into(out, staged):
    mx.base.check_call(mx.base._LIB.B200KVRandomNormalInto(out.handle, ctypes.c_float(0.0),
                                                            ctypes.c_float(1.0), ctypes.c_int(staged)))


def same_bits(n):
    """the staged and per-thread orders write the same numbers from the same state"""
    a = mx.nd.empty((n,), mx.gpu(0))
    b = mx.nd.empty((n,), mx.gpu(0))
    mx.random.seed(5)
    into(a, 1)
    mx.random.seed(5)
    into(b, 0)
    return np.array_equal(a.asnumpy().view(np.uint32), b.asnumpy().view(np.uint32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    gpu = card()
    for n in (64 << 20, 1 << 20, 10_000):
        assert same_bits(n), "staged and per-thread store orders differ at n=%d" % n
        out = mx.nd.empty((n,), mx.gpu(0))
        iters = args.iters if n > (1 << 20) else args.iters * 20
        for staged, label in ((1, "staged"), (0, "per_thread")):
            ms = timed(lambda: into(out, staged), iters)
            gbs = n * 4 / (ms * 1e-3) / 1e9
            print(json.dumps({"bench": "_random_normal", "dtype": "float32", "n": n, "store": label,
                              "ms": round(ms, 4), "write_GBps": round(gbs, 1),
                              "of_datasheet": round(gbs * 1e9 / DATASHEET_BPS, 3), "gpu": gpu}))
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    from compat import mxnet_optimizer_sgld as mxopt
    shapes = resnet50_shapes()
    rng = np.random.default_rng(0)
    ws = [mx.nd.array(rng.uniform(-1, 1, s).astype(np.float32), mx.gpu(0)) for s in shapes]
    gs = [mx.nd.array(rng.uniform(-1, 1, s).astype(np.float32), mx.gpu(0)) for s in shapes]
    upd = mxopt.get_updater(mxopt.SGLD(learning_rate=0.01, rescale_grad=1 / 64, clip_gradient=0.005, wd=1e-4))

    def step():
        for k in range(len(shapes)):
            upd(k, gs[k], ws[k])
    ms = timed(step, max(args.iters // 5, 3))
    n = sum(int(np.prod(s)) for s in shapes)
    print(json.dumps({"bench": "sgld_step_local_updater", "workload": "resnet50", "arrays": len(shapes),
                      "elements": n, "ms": round(ms, 3), "gpu": gpu}))


if __name__ == "__main__":
    main()
