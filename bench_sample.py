#!/usr/bin/env python
"""bench_sample.py -- the GPU samplers _random_uniform, _random_exponential, _random_gamma and
_random_randint on one GPU, beside the reference's own launch of the same sampler.

Legs: each sampler into a float32 array (randint: int32 and int64) of 64 M, 1 M and 10 K elements;
gamma at alpha 0.5, 1 and 9 (alpha < 1 takes one more uniform per element; larger alpha rejects
less often). Before timing, the 1 M leg of each is checked bit for bit against the reference's
sampler (oracle/golden_sample.py) from the same generator state.
  call_ms     CUDA events around `--iters` calls after a warm-up (ends with a device synchronise)
  kernel_ms   the mean duration of sample_kernel in a torch.profiler run of its own
  ref_ms      the reference's LaunchRNG launch of the same sampler (oracle/_ref/libmxref_sample_gpu.so),
              CUDA events around its launches only, its states on the device
GB/s = bytes written / kernel_ms, and its share of the 3.35 TB/s HBM3 data-sheet figure of the H100
SXM. The card's name and power limit are read in the same run. One JSON line per leg.

    python bench_sample.py [--iters 50]
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

import golden_sample as GS  # noqa: E402

PEAK_GBS = 3350.0
SIZES = (64 << 20, 1 << 20, 10_000)
# (label, sampler, python call, parameters for the reference arm, dtype)
LEGS = [
    ("uniform", "uniform", lambda mx, o: mx.random.uniform(-2.0, 3.0, out=o), (-2.0, 3.0), "float32"),
    ("exponential", "exponential", lambda mx, o: mx.random.exponential(0.5, out=o), (2.0, 0.0), "float32"),
    ("gamma_a0.5", "gamma", lambda mx, o: mx.random.gamma(0.5, 2.0, out=o), (0.5, 2.0), "float32"),
    ("gamma_a1", "gamma", lambda mx, o: mx.random.gamma(1.0, 2.0, out=o), (1.0, 2.0), "float32"),
    ("gamma_a9", "gamma", lambda mx, o: mx.random.gamma(9.0, 2.0, out=o), (9.0, 2.0), "float32"),
    ("randint", "randint", lambda mx, o: mx.random.randint(-1000, 1 << 40, out=o), (-1000, 1 << 40), "int32"),
    ("randint", "randint", lambda mx, o: mx.random.randint(-1000, 1 << 40, out=o), (-1000, 1 << 40), "int64"),
]


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


def kernel_ms(torch, mx, fn, iters):
    mx.nd.waitall()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        mx.nd.waitall()
        torch.cuda.synchronize()
    durs = [e.device_time for e in prof.events() if "sample_kernel" in e.name]
    return float(np.mean(durs)) / 1e3 if durs else float("nan")


def parity(mx, dist, fn, params, dtype):
    """the 1 M leg equals the reference's draw from the same seeded state"""
    n = 1 << 20
    mx.random.seed(11)
    ref = GS.SampleGenerators(0, 11)
    o = mx.nd.empty((n,), mx.gpu(0), dtype=dtype)
    fn(mx, o)
    if dist == "exponential":
        want = ref.exponential(n, float(np.float32(1.0 / 0.5)), dtype)
    else:
        want = getattr(ref, dist)(n, *[p if dist == "randint" else float(np.float32(p)) for p in params], dtype)
    return np.array_equal(o.asnumpy().view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    import torch
    import anand_mxnet_b200 as mx
    name, power = card()
    have_ref = GS.available()
    for label, dist, fn, params, dtype in LEGS:
        ok = parity(mx, dist, fn, params, dtype) if have_ref else None
        for n in SIZES:
            o = mx.nd.empty((n,), mx.gpu(0), dtype=dtype)
            iters = args.iters if n > (1 << 20) else args.iters * 20
            ms = call_ms(torch, mx, lambda: fn(mx, o), iters)
            kms = kernel_ms(torch, mx, lambda: fn(mx, o), min(iters, 200))
            ref_ms = GS.time_ref(dist, n, params[0], params[1], dtype, 10, iters) if have_ref else None
            nbytes = n * np.dtype(dtype).itemsize
            gbs = nbytes / (kms * 1e-3) / 1e9
            print(json.dumps({"bench": "_random_" + dist, "leg": label, "dtype": dtype, "n": n,
                              "bit_exact_vs_reference": ok, "call_ms": round(ms, 4), "kernel_ms": round(kms, 4),
                              "ref_ms": None if ref_ms is None else round(ref_ms, 4),
                              "write_GBps": round(gbs, 1), "of_datasheet": round(gbs / PEAK_GBS, 3),
                              "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
