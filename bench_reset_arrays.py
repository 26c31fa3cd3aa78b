#!/usr/bin/env python
"""bench_reset_arrays.py -- reset_arrays, the bulk gradient reset of ParameterDict.zero_grad, on one GPU.

Legs:
  r50_fp32    the ResNet-50 gradient set (bench.resnet50_shapes(): 157 arrays, 102 MB in float32)
  bert_fp16   the BERT-base set (bench.bert_base_shapes(): 199 arrays, 219 MB in float16)
  flat_fp32   one 512 MB float32 tensor
Each leg compares, alternating in one process:
  reset       one reset_arrays call over every array
  zeros_like  one zeros_like(g, out=g) per array, the only way to zero them before reset_arrays
  torch       torch.Tensor.zero_() on one torch tensor of the flat leg's size: a write-rate yardstick
              on the same card (the same on every leg)

Parity first: every array is filled with random bits, zeroed by each path in turn, and every byte is
checked against zero on the device.

Bytes written = every byte of every array once. Kernel time is the mean duration of
reset_arrays_kernel (and of torch's fill kernel for the yardstick) in a torch.profiler run of its own;
call time is CUDA events around many calls on the stream the library is given (torch's current
stream), so it includes the host's enqueue whenever that is slower than the device. Prints one JSON
line per leg with GB/s over kernel time and its fraction of 3.35 TB/s (H100 SXM HBM3 data sheet),
with the card's name and power limit read in the same run.

    python bench_reset_arrays.py [--iters N] [--rounds R]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import bert_base_shapes, resnet50_shapes  # noqa: E402

PEAK_GBS = 3350.0
FLAT = (128 * 1024 * 1024,)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as exc:  # noqa: BLE001
        return "unknown (%s)" % exc, "unknown"


def legs():
    return [("r50_fp32", "float32", resnet50_shapes()), ("bert_fp16", "float16", bert_base_shapes()),
            ("flat_fp32", "float32", [FLAT])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_reset_arrays.py needs a GPU")
    import anand_mxnet_b200 as mx
    name, power = card()
    tdt = {"float16": torch.float16, "float32": torch.float32}
    yard = torch.empty(FLAT, dtype=torch.float32, device="cuda")
    mx.base.set_stream(0, torch.cuda.current_stream().cuda_stream)

    def timed(fn, iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / iters

    def kernel_us(fn, iters, kernel):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                fn()
            torch.cuda.synchronize()
        durs = [e.device_time for e in prof.events() if kernel(e.name)]
        return (float(np.mean(durs)) if durs else float("nan")), len(durs)

    for leg, dtype, shapes in legs():
        gen = torch.Generator(device="cuda").manual_seed(0xB200)
        ts = [torch.empty(int(np.prod(s)), dtype=tdt[dtype], device="cuda") for s in shapes]
        arrays = [mx.nd.from_torch(t) for t in ts]
        nbytes = sum(t.numel() * t.element_size() for t in ts)

        def reset():
            mx.nd.reset_arrays(*arrays, num_arrays=len(arrays))

        def per_array():
            for a in arrays:
                mx.nd.zeros_like(a, out=a)

        def fill():
            for t in ts:
                t.view(torch.uint8).random_(1, 256, generator=gen)

        # parity: random bits everywhere, then every byte zero after each path
        for fn in (reset, per_array):
            fill()
            assert all(torch.count_nonzero(t.view(torch.uint8)).item() == t.numel() * t.element_size() for t in ts)
            fn()
            assert all(torch.count_nonzero(t.view(torch.uint8)).item() == 0 for t in ts), (leg, fn.__name__)
        before = mx.base.kernel_launch_count()
        reset()
        launches = mx.base.kernel_launch_count() - before
        assert launches == math.ceil(len(arrays) / 200), (leg, launches)
        for fn in (reset, per_array, yard.zero_):   # warm-up
            for _ in range(5):
                fn()
        torch.cuda.synchronize()
        calls = {"reset": [], "zeros_like": [], "torch": []}
        for _ in range(args.rounds):   # alternating, one window per path per round
            calls["reset"].append(timed(reset, args.iters))
            calls["zeros_like"].append(timed(per_array, args.iters))
            calls["torch"].append(timed(yard.zero_, args.iters))
        k_us, k_n = kernel_us(reset, args.iters, lambda n: "reset_arrays_kernel" in n)
        t_us, _ = kernel_us(yard.zero_, args.iters, lambda n: "fill" in n.lower() or "zero" in n.lower())
        gbs = nbytes / (k_us * 1e-6) / 1e9
        t_gbs = yard.numel() * 4 / (t_us * 1e-6) / 1e9
        print(json.dumps(dict(
            bench="reset_arrays", leg=leg, dtype=dtype, arrays=len(arrays), bytes=nbytes,
            launches_per_call=launches, kernel_us=round(k_us, 2), kernels_profiled=k_n,
            achieved_gbs=round(gbs, 1), frac_of_3350_gbs=round(gbs / PEAK_GBS, 3),
            call_us_reset=[round(x, 1) for x in calls["reset"]],
            call_us_zeros_like_per_array=[round(x, 1) for x in calls["zeros_like"]],
            call_us_torch_zero_flat=[round(x, 1) for x in calls["torch"]],
            torch_zero_flat_kernel_us=round(t_us, 2), torch_zero_flat_gbs=round(t_gbs, 1),
            parity="ok", card=name, power_limit=power)), flush=True)
        del arrays
        mx.nd.waitall()
    mx.base.set_stream(0, None)


if __name__ == "__main__":
    main()
