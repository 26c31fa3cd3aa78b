"""mx.random (python/mxnet/random.py, ndarray/random.py): seeding and normal sampling on the GPU, in
the reference's GPU Philox streams. Each GPU holds 4 copies of 32768 curand Philox states; every
sampling call takes the next copy in turn, so a seed followed by the same calls gives the same
numbers as the reference's GPU build. CPU sampling is refused: the reference's CPU generator is a
different stream."""
import ctypes

import numpy as np

from .base import _LIB, check_call
from .context import Context, current_context
from .ndarray import NDArray, _invoke


def seed(seed_state, ctx="all"):
    """Seeds the random number generators. With ctx="all" every GPU's generators are reseeded from
    seed_state and the device id (and the seed is kept for GPUs first used later); with a context
    only that device's generators are reseeded, without the device id, so two GPUs seeded this way
    draw the same numbers."""
    if not isinstance(seed_state, int):
        raise ValueError('seed_state must be int')
    seed_state = ctypes.c_int(int(seed_state))
    if ctx == "all":
        check_call(_LIB.MXRandomSeed(seed_state))
    else:
        ctx = Context(ctx)
        check_call(_LIB.MXRandomSeedContext(seed_state, ctx.device_typeid, ctx.device_id))


def _dtype_name(dtype):
    return 'bfloat16' if isinstance(dtype, str) and dtype == 'bfloat16' else np.dtype(dtype).name


def normal(loc=0, scale=1, shape=None, dtype=None, ctx=None, out=None, **kwargs):
    """Draws samples from N(loc, scale**2) into a new array of `shape` (default (1,)) on `ctx`, or
    into `out` (whose context, shape and dtype then decide). dtype: float16, float32 (default),
    float64, or bfloat16 (an extension; the float32 draw rounded once). loc and scale are numbers;
    scale must be positive."""
    if isinstance(loc, NDArray) or isinstance(scale, NDArray):
        raise ValueError("normal with NDArray parameters (_sample_normal) is not available; "
                         "loc and scale must be numbers")
    if ctx is None:
        ctx = current_context()
    if shape is None and out is None:
        shape = 1
    if shape is not None:
        kwargs['shape'] = (shape,) if isinstance(shape, int) else tuple(shape)
    if dtype is not None:
        kwargs['dtype'] = _dtype_name(dtype)
    return _invoke('_random_normal', [], out=out, loc=loc, scale=scale, ctx=ctx, **kwargs)
