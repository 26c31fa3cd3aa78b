"""One optimizer step of the reference's Adamax, Nadam and AdaDelta classes (the tests/compat mirror
over this package's NDArray) on the ResNet-50 and BERT-base gradient sets, through a local updater
(update_on_kvstore=False: one `update` per key, each a chain of elementwise operators).

    python bench_arith_optimizers.py [--steps 10] [--warmup 3]

One JSON line per (workload, optimizer):
- `ms_per_step`: CUDA events on the library's stream around `steps` steps after `warmup` steps;
- `launches_per_step`: the library's kernel launch counter (B200KVGetKernelLaunchCount) over one step;
- `bytes_per_step`: algorithmic bytes of the operators the step issues, each counted once as the
  bytes it must read and write (every input and the output, in their dtypes);
- `GBps` and `frac_of_datasheet_hbm`: bytes_per_step over ms_per_step, and that rate over the
  H100 SXM data-sheet 3.35 TB/s (a data-sheet figure, not a measured ceiling);
- the card's name and power limit, read by nvidia-smi in the same run.
fp32 weights and gradients, default hyper-parameters with wd=1e-4. Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_DATASHEET_GBS = 3350.0
ITEMSIZE = {'float16': 2, 'bfloat16': 2, 'float32': 4, 'float64': 8, 'int32': 4, 'int64': 8}


def card():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, plim = (r.stdout.strip().split(", ") + ["?", "?"])[:2] if r.returncode == 0 else ("?", "?")
    return name, plim


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import anand_mxnet_b200 as mx
    import anand_mxnet_b200.ndarray as ndmod
    from bench import resnet50_shapes, bert_base_shapes
    from compat import mxnet_optimizer_arith as mxopt
    if not torch.cuda.is_available():
        sys.exit("bench_arith_optimizers.py needs a GPU")
    name, plim = card()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    mx.base.set_stream(0, stream.cuda_stream)

    invoke = ndmod._invoke
    issued = []

    def counting_invoke(op_name, inputs, out=None, **kwargs):
        res = invoke(op_name, inputs, out=out, **kwargs)
        o = out if out is not None else res
        o = o[0] if isinstance(o, (list, tuple)) else o
        dt = o.dtype if isinstance(o.dtype, str) else np.dtype(o.dtype).name
        nbytes = o.size * ITEMSIZE[dt]
        in_bytes = sum(a.size * ITEMSIZE[a.dtype if isinstance(a.dtype, str) else np.dtype(a.dtype).name]
                       for a in inputs)
        issued.append((op_name, in_bytes + nbytes))
        return res

    def step_bytes(step):
        """(launches, bytes, operators) of one step"""
        issued[:] = []
        ndmod._invoke = counting_invoke
        try:
            mx.nd.waitall()
            before = mx.base.kernel_launch_count()
            step()
            mx.nd.waitall()
            launches = mx.base.kernel_launch_count() - before
        finally:
            ndmod._invoke = invoke
        return launches, sum(b for _, b in issued), len(issued)

    def timed(step):
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        mx.nd.waitall()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            step()
        e1.record(stream)
        mx.nd.waitall()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    rng = np.random.default_rng(0)
    for workload, shapes in (("resnet50", resnet50_shapes()), ("bert_base", bert_base_shapes())):
        n = sum(int(np.prod(s)) for s in shapes)
        weights = [mx.nd.array(rng.uniform(-1, 1, s).astype(np.float32), mx.gpu(0)) for s in shapes]
        grads = [mx.nd.array(rng.uniform(-1, 1, s).astype(np.float32), mx.gpu(0)) for s in shapes]
        for cls in ('Adamax', 'Nadam', 'AdaDelta'):
            upd = mxopt.get_updater(getattr(mxopt, cls)(wd=1e-4))

            def step():
                for k in range(len(shapes)):
                    upd(k, grads[k], weights[k])
            step()                                    # creates the states
            launches, nbytes, nops = step_bytes(step)
            ms = timed(step)
            gbs = nbytes / (ms * 1e-3) / 1e9
            print(json.dumps({"metric": "arith_optimizer_step", "workload": workload, "optimizer": cls,
                              "tensors": len(shapes), "elements": n, "ms_per_step": ms,
                              "launches_per_step": launches, "operators_per_step": nops,
                              "bytes_per_step": nbytes, "GBps": gbs,
                              "frac_of_datasheet_hbm": gbs / HBM_DATASHEET_GBS,
                              "datasheet_hbm_gbs": HBM_DATASHEET_GBS, "steps": args.steps,
                              "warmup": args.warmup, "gpu": name, "power_limit": plim}), flush=True)
            del upd
        del weights, grads
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
