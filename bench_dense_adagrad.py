"""The trailing-axis mean kernel alone, and one step of the reference's AdaGrad and GroupAdaGrad
classes with dense gradients (the tests/compat mirror over this package's NDArray) through a local
updater.

    python bench_dense_adagrad.py [--steps 20] [--warmup 3]

One JSON line per measurement, each with the card's name and power limit read by nvidia-smi in the
same run:
- `row_mean`: float32 `mean(x, axis=-1)` over R x C. `ms` is CUDA events on the library's stream
  around `steps` calls after `warmup` calls; `bytes` is R*C*4 + R*4 (the input read once, the
  output written once); `frac_of_datasheet_hbm` is bytes / ms over the H100 SXM data-sheet 3.35 TB/s
  (a data-sheet figure, not a measured ceiling). Every output is checked bit for bit against the
  numpy restatement (oracle/golden_dense_adagrad.py) before it is timed.
- `dense_adagrad_step`: AdaGrad over the fp32 ResNet-50 and BERT-base gradient sets, GroupAdaGrad
  over BERT-base's 2-D weights and over a 1M x 512 table: `ms_per_step` (CUDA events, as above) and
  `launches_per_step` (the library's kernel launch counter over one step).
Needs a GPU."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from bench_arith_optimizers import HBM_DATASHEET_GBS, card  # noqa: E402

MEAN_SHAPES = [(1 << 20, 512), (4 << 20, 16), (32 << 10, 4096), (768, 768)]
TABLE = (1 << 20, 512)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import anand_mxnet_b200 as mx
    import golden_dense_adagrad as GD
    from bench import resnet50_shapes, bert_base_shapes
    from compat import mxnet_optimizer_dense_adagrad as mxopt
    if not torch.cuda.is_available():
        sys.exit("bench_dense_adagrad.py needs a GPU")
    name, plim = card()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    mx.base.set_stream(0, stream.cuda_stream)

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        mx.nd.waitall()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            fn()
        e1.record(stream)
        mx.nd.waitall()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    def launches(fn):
        mx.nd.waitall()
        before = mx.base.kernel_launch_count()
        fn()
        mx.nd.waitall()
        return mx.base.kernel_launch_count() - before

    gen = torch.Generator(device='cuda').manual_seed(0)
    for R, C in MEAN_SHAPES:
        t = torch.rand((R, C), generator=gen, device='cuda', dtype=torch.float32) * 2 - 1
        X = mx.nd.from_torch(t)
        O = mx.nd.empty((R,), mx.gpu(0))
        call = lambda: mx.nd.mean(X, axis=-1, out=O)  # noqa: E731
        call()
        got, want = O.asnumpy(), GD.mean_rows(t.cpu().numpy(), 'float32')
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), "row_mean %dx%d differs" % (R, C)
        ms = timed(call)
        nbytes = R * C * 4 + R * 4
        gbs = nbytes / (ms * 1e-3) / 1e9
        print(json.dumps({"metric": "row_mean", "rows": R, "cols": C, "dtype": "float32", "ms": ms,
                          "bytes": nbytes, "GBps": gbs, "frac_of_datasheet_hbm": gbs / HBM_DATASHEET_GBS,
                          "datasheet_hbm_gbs": HBM_DATASHEET_GBS, "checked": True, "steps": args.steps,
                          "warmup": args.warmup, "gpu": name, "power_limit": plim}), flush=True)
        del X, O, t
        torch.cuda.empty_cache()

    bert2d = [s for s in bert_base_shapes() if len(s) == 2]
    runs = [("resnet50", "AdaGrad", resnet50_shapes()), ("bert_base", "AdaGrad", bert_base_shapes()),
            ("bert_base_2d", "GroupAdaGrad", bert2d), ("table_1Mx512", "GroupAdaGrad", [TABLE])]
    for workload, cls, shapes in runs:
        n = sum(int(np.prod(s)) for s in shapes)
        weights = [mx.nd.from_torch(torch.rand(s, generator=gen, device='cuda') * 2 - 1) for s in shapes]
        grads = [mx.nd.from_torch(torch.rand(s, generator=gen, device='cuda') * 2 - 1) for s in shapes]
        upd = mxopt.get_updater(getattr(mxopt, cls)(learning_rate=0.01, **({'wd': 1e-4} if cls == 'AdaGrad' else {})))

        def step():
            for k in range(len(shapes)):
                upd(k, grads[k], weights[k])
        step()                                    # creates the states
        nl = launches(step)
        ms = timed(step)
        print(json.dumps({"metric": "dense_adagrad_step", "workload": workload, "optimizer": cls,
                          "tensors": len(shapes), "elements": n, "ms_per_step": ms, "launches_per_step": nl,
                          "steps": args.steps, "warmup": args.warmup, "gpu": name, "power_limit": plim}),
              flush=True)
        del upd, weights, grads
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
