#!/usr/bin/env python
"""bench_sample_params.py -- sampling with NDArray parameters (_sample_uniform, _sample_normal,
_sample_gamma, _sample_exponential) on one GPU, beside the reference's own launch of the same
multi-sample sampler.

Each distribution writes 64 M float32 outputs from float32 parameters in three layouts:
  64M x ()      64 M parameter sets, one sample each (nBatch 1: every element reads its own)
  1M x (64,)    1 M parameter sets, 64 samples each
  1 x (64M,)    one parameter set; shown beside the scalar operator (_random_*) over the same 64 M
gamma runs at alpha 1, beta 2; uniform low -2, high 3; normal mu 0.5, sigma 2; exponential lam 2.
  kernel_ms   the mean duration of param_draw_kernel (the scalar leg: the scalar operator's kernel)
              in a torch.profiler run of its own
  ref_ms      the reference's LaunchRNG launch of the same sampler and layout
              (oracle/_ref/libmxref_sample_params_gpu.so), CUDA events around its launches only
GB/s = (outputs written + parameters read) / kernel_ms. The card's name and power limit are read in
the same run. One JSON line per leg.

    python bench_sample_params.py [--iters 20]
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

import golden_sample_params as GP  # noqa: E402

N = 64 << 20
LAYOUTS = [("64Mx()", N, ()), ("1Mx(64,)", 1 << 20, (64,)), ("1x(64M,)", 1, (N,))]
# (distribution, parameters, the scalar operator's call into out, its kernel's name)
DISTS = [
    ("uniform", (-2.0, 3.0), lambda mx, o: mx.random.uniform(-2.0, 3.0, out=o), "sample_kernel"),
    ("normal", (0.5, 2.0), lambda mx, o: mx.random.normal(0.5, 2.0, out=o), "normal_kernel"),
    ("gamma", (1.0, 2.0), lambda mx, o: mx.random.gamma(1.0, 2.0, out=o), "sample_kernel"),
    ("exponential", (2.0, 0.0), lambda mx, o: mx.random.exponential(0.5, out=o), "sample_kernel"),
]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as exc:  # noqa: BLE001
        return "unknown (%s)" % exc, "unknown"


def kernel_ms(torch, mx, fn, iters, kernel):
    for _ in range(3):
        fn()
    mx.nd.waitall()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        mx.nd.waitall()
        torch.cuda.synchronize()
    durs = [e.device_time for e in prof.events() if kernel in e.name]
    return float(np.mean(durs)) / 1e3 if durs else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import torch
    import anand_mxnet_b200 as mx
    name, power = card()
    have_ref = GP.available()
    gpu = mx.gpu(0)
    for dist, (p0, p1), scalar, scalar_kernel in DISTS:
        for label, nparm, shape in LAYOUTS:
            a = mx.nd.array(np.full(nparm, p0, np.float32), gpu)
            b = mx.nd.array(np.full(nparm, p1, np.float32), gpu)
            o = mx.nd.empty((nparm,) + shape, gpu)
            ins = [a] if dist == "exponential" else [a, b]
            fn = getattr(mx.nd, "sample_" + dist)
            kms = kernel_ms(torch, mx, lambda: fn(*ins, shape=shape, out=o), args.iters, "param_draw_kernel")
            ref_ms = (GP.time_ref(dist, nparm, N, p0, p1, np.float32, "float32", 3, args.iters)
                      if have_ref else None)
            nbytes = N * 4 + nparm * 4 * len(ins)
            row = {"bench": "_sample_" + dist, "layout": label, "n": N, "kernel_ms": round(kms, 4),
                   "ref_ms": None if ref_ms is None else round(ref_ms, 4),
                   "GBps": round(nbytes / (kms * 1e-3) / 1e9, 1), "gpu": name, "power_limit": power}
            if nparm == 1:
                flat = mx.nd.empty((N,), gpu)
                sms = kernel_ms(torch, mx, lambda: scalar(mx, flat), args.iters, scalar_kernel)
                row["scalar_op_kernel_ms"] = round(sms, 4)
            print(json.dumps(row), flush=True)
            del a, b, o


if __name__ == "__main__":
    main()
