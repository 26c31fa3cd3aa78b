#!/usr/bin/env python
"""bench_clip_global_norm.py -- gluon.utils.clip_global_norm (one _b200kv_clip_global_norm call) on
one GPU, float32.

Legs:
  r50_fp32    the ResNet-50 gradient set (bench.resnet50_shapes(): 157 arrays, 102 MB)
  bert_fp32   the BERT-base set (bench.bert_base_shapes(): 199 arrays, 438 MB)
  flat_fp32   one 512 MB tensor
each with a max_norm that clips (from 1e-3 down)
and one that never does (1e30). Once clipped, a set's norm equals max_norm and the next call would
not clip, so the clipped variant lowers max_norm by 0.05 % from call to call, in both arms: every
timed call reads, scales and writes.

Parity first: on the same seeded values the norm is within 1e-5 of a float64 sum and every array is
bit-equal to oracle/golden_clip_global_norm.restate on the norm the GPU returned, before anything is
timed. A missing GPU is an error.

Baseline, in the same process and alternating with the new call: what the package offered before
this operator -- multi_sum_sq in groups of 64, a host read of the sums, the fold, sqrt and factor on
the host, then one _mul_scalar launch per array when the factor is below 1.

Per leg and variant, one JSON line: launches per call; the mean duration of each kernel
(clip_norm_partial / _fold / _scale) over 50 calls in a torch.profiler run of its own; call time from CUDA
events over alternating rounds that fill about a second per arm; bytes = 4 B/element when not
clipped (every gradient read once; the scaling kernel returns before reading), 12 B/element when
clipped (read, read, write); GB/s over the summed kernel time and its fraction of 3.35 TB/s, the
H100 SXM HBM3 data-sheet figure; the card's name and power limit read in the same run. The 50 MB L2
can serve part of the ResNet-50 set's second pass (102 MB); flat_fp32 is the bandwidth leg.

    python bench_clip_global_norm.py [--seconds S]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from bench import bert_base_shapes, resnet50_shapes  # noqa: E402
import golden_clip_global_norm as G  # noqa: E402

PEAK_GBS = 3350.0
KERNELS = ("clip_norm_partial", "clip_norm_fold", "clip_norm_scale")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as exc:  # noqa: BLE001
        return "unknown (%s)" % exc, "unknown"


def legs():
    return [("r50_fp32", resnet50_shapes()), ("bert_fp32", bert_base_shapes()),
            ("flat_fp32", [(128 * 1024 * 1024,)])]


def baseline(mx, arrays, max_norm):
    """clip_global_norm composed from multi_sum_sq, a host read and _mul_scalar"""
    sums = [mx.nd.multi_sum_sq(*arrays[i:i + 64], num_arrays=len(arrays[i:i + 64]))
            for i in range(0, len(arrays), 64)]
    ss = np.float32(0)
    for s in sums:
        ss = np.float32(ss + s.asnumpy().sum(dtype=np.float32))
    norm = np.sqrt(ss)
    scale = min(np.float32(max_norm) / (norm + np.float32(1e-8)), np.float32(1.0))
    if scale < 1:
        for a in arrays:
            a *= float(scale)
    return norm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0, help="timed work per arm and variant")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip_global_norm.py needs a GPU")
    import anand_mxnet_b200 as mx
    name, power = card()
    for leg, shapes in legs():
        gen = torch.Generator(device="cuda").manual_seed(0xB200)
        sizes = [int(np.prod(s)) for s in shapes]
        ts = [torch.empty(n, dtype=torch.float32, device="cuda").normal_(0, 0.02, generator=gen) for n in sizes]
        torch.cuda.synchronize()
        arrays = [mx.nd.from_torch(t) for t in ts]
        n_elem = sum(sizes)
        for variant, max_norm in (("clipped", 1e-3), ("not_clipped", 1e30)):
            bound = [max_norm]

            def next_bound():
                if variant == "clipped":
                    bound[0] *= 0.9995
                return bound[0]

            def call():
                return mx.gluon.utils.clip_global_norm(arrays, next_bound(), check_isfinite=False)
            # parity on the values as they stand (the clipped variant runs first and scales them)
            before_h = [t.cpu().numpy() for t in ts]
            exact = float(np.sqrt(sum(float(np.sum(x.astype(np.float64) ** 2)) for x in before_h)))
            norm = call().asnumpy()[0]
            assert abs(float(norm) - exact) <= 1e-5 * exact, (leg, variant, norm, exact)
            for x, t in zip(before_h, ts):
                assert t.cpu().numpy().tobytes() == G.restate(norm, bound[0], x).tobytes(), (leg, variant)
            del before_h
            count0 = mx.base.kernel_launch_count()
            call()
            launches = mx.base.kernel_launch_count() - count0
            count0 = mx.base.kernel_launch_count()
            baseline(mx, arrays, next_bound())
            base_launches = mx.base.kernel_launch_count() - count0
            for _ in range(5):   # warm-up of both arms
                call()
                baseline(mx, arrays, next_bound())
            mx.nd.waitall()
            # size the rounds: five alternating rounds per arm, `seconds` in all
            t0 = time.perf_counter()
            call()
            mx.nd.waitall()
            t_new = time.perf_counter() - t0
            t0 = time.perf_counter()
            baseline(mx, arrays, next_bound())
            mx.nd.waitall()
            t_base = time.perf_counter() - t0
            rounds = 5
            k_new = max(3, int(args.seconds / rounds / t_new))
            k_base = max(3, int(args.seconds / rounds / t_base))
            new_ms, base_ms = [], []
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(rounds):
                torch.cuda.synchronize()
                e0.record()
                for _ in range(k_new):
                    call()
                mx.nd.waitall()
                e1.record()
                torch.cuda.synchronize()
                new_ms.append(e0.elapsed_time(e1) / k_new)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(k_base):
                    baseline(mx, arrays, next_bound())
                mx.nd.waitall()
                base_ms.append((time.perf_counter() - t0) * 1e3 / k_base)
            # kernel time: each kernel's own durations, in a profiled run of its own
            n_prof = 50
            groups = (len(arrays) + 199) // 200
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(n_prof):
                    call()
                mx.nd.waitall()
                torch.cuda.synchronize()
            kernel_us = {}
            for k in KERNELS:
                durs = [e.device_time for e in prof.events() if k + "_kernel" in e.name]
                per_call = 1 if k == "clip_norm_fold" else groups
                assert len(durs) == n_prof * per_call, (k, len(durs))   # no profiler event was dropped
                kernel_us[k] = round(float(np.mean(durs)) * per_call, 2)
            total_us = sum(kernel_us.values())
            nbytes = n_elem * (12 if variant == "clipped" else 4)
            gbs = nbytes / (total_us * 1e-6) / 1e9
            print(json.dumps(dict(
                bench="clip_global_norm", leg=leg, variant=variant, max_norm_start=max_norm, arrays=len(arrays),
                elements=n_elem, bytes=nbytes, launches_per_call=launches, kernel_us_per_call=kernel_us,
                kernel_us_total=round(total_us, 2), call_us=round(float(np.median(new_ms)) * 1e3, 2),
                call_us_rounds=[round(v * 1e3, 1) for v in new_ms], calls_per_round=k_new,
                achieved_gbs=round(gbs, 1), frac_of_3350_gbs_datasheet=round(gbs / PEAK_GBS, 3),
                baseline_launches_per_call=base_launches, baseline_call_us=round(float(np.median(base_ms)) * 1e3, 2),
                baseline_call_us_rounds=[round(v * 1e3, 1) for v in base_ms], baseline_calls_per_round=k_base,
                parity="ok", card=name, power_limit=power)), flush=True)
        del arrays, ts
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
