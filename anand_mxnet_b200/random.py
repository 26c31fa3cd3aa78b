"""mx.random (python/mxnet/random.py, ndarray/random.py): seeding, and uniform, normal, exponential,
gamma and randint sampling on the GPU, in the reference's GPU Philox streams. Each GPU holds 4
copies of 32768 curand Philox states; every sampling call, whichever its distribution, takes the
next copy in turn, so a seed followed by the same calls gives the same numbers as the reference's
GPU build. CPU sampling is refused: the reference's CPU generator is a different stream.

The _like forms (uniform_like, normal_like, exponential_like, gamma_like) take shape, context and
dtype from an array; mx.nd.random exposes them beside the functions here."""
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


def _sample(op, name, params, shape, dtype, ctx, out, kwargs):
    """the reference's _random_helper for number parameters: shape (1,) when neither shape nor out
    is given, the current context when ctx is None"""
    if any(isinstance(v, NDArray) for v in params.values()):
        raise ValueError("%s with NDArray parameters (_sample_%s) is not available; %s must be numbers"
                         % (name, name, " and ".join(params)))
    if ctx is None:
        ctx = current_context()
    if shape is None and out is None:
        shape = 1
    if shape is not None:
        kwargs['shape'] = (shape,) if isinstance(shape, int) else tuple(shape)
    if dtype is not None:
        kwargs['dtype'] = _dtype_name(dtype)
    kwargs.update(params)
    return _invoke(op, [], out=out, ctx=ctx, **kwargs)


def uniform(low=0, high=1, shape=None, dtype=None, ctx=None, out=None, **kwargs):
    """Draws samples from U[low, high) into a new array of `shape` (default (1,)) on `ctx`, or into
    `out` (whose context, shape and dtype then decide). dtype: float16, float32 (default), float64,
    or bfloat16 (an extension; the float32 draw rounded once). high must not be below low."""
    return _sample('_random_uniform', 'uniform', {'low': low, 'high': high}, shape, dtype, ctx, out, kwargs)


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


def randn(*shape, **kwargs):
    """normal(loc, scale, shape) with the shape given as positional arguments: randn(2, 3, loc=1)"""
    loc = kwargs.pop('loc', 0)
    scale = kwargs.pop('scale', 1)
    dtype = kwargs.pop('dtype', None)
    ctx = kwargs.pop('ctx', None)
    out = kwargs.pop('out', None)
    return normal(loc, scale, shape if shape else None, dtype, ctx, out, **kwargs)


def exponential(scale=1, shape=None, dtype=None, ctx=None, out=None, **kwargs):
    """Draws samples from the exponential distribution of mean `scale` (the operator's lam is
    1.0 / scale), as uniform does. scale must be positive."""
    if isinstance(scale, NDArray):
        raise ValueError("exponential with NDArray parameters (_sample_exponential) is not available; "
                         "scale must be a number")
    return _sample('_random_exponential', 'exponential', {'lam': 1.0 / scale}, shape, dtype, ctx, out, kwargs)


def gamma(alpha=1, beta=1, shape=None, dtype=None, ctx=None, out=None, **kwargs):
    """Draws samples from the gamma distribution of shape `alpha` and scale `beta`, as uniform does.
    alpha and beta must be positive."""
    return _sample('_random_gamma', 'gamma', {'alpha': alpha, 'beta': beta}, shape, dtype, ctx, out, kwargs)


def randint(low, high, shape=None, dtype=None, ctx=None, out=None, **kwargs):
    """Draws integers uniformly from [low, high) (int64 bounds) into a new array of `shape` (default
    (1,)) on `ctx`, or into `out`. dtype: int32 (default; a value outside int32 wraps) or int64.
    high must be greater than low."""
    return _sample('_random_randint', 'randint', {'low': low, 'high': high}, shape, dtype, ctx, out, kwargs)


def _like(op, data, params, out, kwargs):
    if any(isinstance(v, NDArray) for v in params.values()):
        raise ValueError("%s takes number parameters only" % op)
    kwargs.update(params)
    return _invoke(op, [data], out=out, **kwargs)


def uniform_like(data, low=0, high=1, out=None, **kwargs):
    """uniform(low, high) with data's shape, context and dtype (_random_uniform_like); data's values
    are not read, so out may be data"""
    return _like('_random_uniform_like', data, {'low': low, 'high': high}, out, kwargs)


def normal_like(data, loc=0, scale=1, out=None, **kwargs):
    """normal(loc, scale) with data's shape, context and dtype (_random_normal_like)"""
    return _like('_random_normal_like', data, {'loc': loc, 'scale': scale}, out, kwargs)


def exponential_like(data, lam=1, out=None, **kwargs):
    """the exponential distribution of rate lam with data's shape, context and dtype
    (_random_exponential_like; the operator takes lam, not scale)"""
    return _like('_random_exponential_like', data, {'lam': lam}, out, kwargs)


def gamma_like(data, alpha=1, beta=1, out=None, **kwargs):
    """gamma(alpha, beta) with data's shape, context and dtype (_random_gamma_like)"""
    return _like('_random_gamma_like', data, {'alpha': alpha, 'beta': beta}, out, kwargs)
