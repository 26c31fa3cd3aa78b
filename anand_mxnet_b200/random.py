"""mx.random (python/mxnet/random.py, ndarray/random.py): seeding, and uniform, normal, exponential,
gamma and randint sampling on the GPU, in the reference's GPU Philox streams. Each GPU holds 4
copies of 32768 curand Philox states; every sampling call, whichever its distribution, takes the
next copy in turn, so a seed followed by the same calls gives the same numbers as the reference's
GPU build. CPU sampling is refused: the reference's CPU generator is a different stream.

uniform, normal, randn, gamma and exponential also take NDArray parameters, as the reference's
_random_helper does: with every parameter an NDArray they call the multi-sample operators
(_sample_uniform, _sample_normal, _sample_gamma, _sample_exponential), whose output has the
parameters' shape followed by `shape`, each parameter set drawing its own samples.

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


def _shape_arg(shape):
    return (shape,) if isinstance(shape, int) else tuple(shape)


def _sample_params(name, params, shape, dtype, out, kwargs):
    """_random_helper with NDArray parameters: _sample_<name> over the arrays, shape and dtype passed
    only when given, ctx ignored"""
    if shape is not None:
        kwargs['shape'] = _shape_arg(shape)
    if dtype is not None:
        kwargs['dtype'] = _dtype_name(dtype)
    return _invoke('_sample_' + name, list(params.values()), out=out, **kwargs)


def _array_params(name, params):
    """True when every parameter is an NDArray, False when none is; a mix is refused"""
    arrays = [isinstance(v, NDArray) for v in params.values()]
    if any(arrays) and not all(arrays):
        raise ValueError("%s: NDArray parameters must all be NDArrays (%s); got a mix of NDArrays and "
                         "numbers" % (name, " and ".join(params)))
    return all(arrays)


def _sample(op, name, params, shape, dtype, ctx, out, kwargs):
    """the reference's _random_helper: NDArray parameters go to _sample_<name>; for number
    parameters, shape (1,) when neither shape nor out is given, the current context when ctx is None"""
    if name != 'randint' and _array_params(name, params):
        return _sample_params(name, params, shape, dtype, out, kwargs)
    if any(isinstance(v, NDArray) for v in params.values()):
        raise ValueError("%s with NDArray parameters is not available; %s must be numbers"
                         % (name, " and ".join(params)))
    if ctx is None:
        ctx = current_context()
    if shape is None and out is None:
        shape = 1
    if shape is not None:
        kwargs['shape'] = _shape_arg(shape)
    if dtype is not None:
        kwargs['dtype'] = _dtype_name(dtype)
    kwargs.update(params)
    return _invoke(op, [], out=out, ctx=ctx, **kwargs)


def uniform(low=0, high=1, shape=None, dtype=None, ctx=None, out=None, **kwargs):
    """Draws samples from U[low, high) into a new array of `shape` (default (1,)) on `ctx`, or into
    `out` (whose context, shape and dtype then decide). dtype: float16, float32 (default), float64,
    or bfloat16 (an extension; the float32 draw rounded once). high must not be below low.

    With NDArray low and high (one shape and dtype, float16 / float32 / float64, on one GPU): an
    array of shape low.shape + shape (shape default ()), each (low, high) pair drawing its own
    samples (_sample_uniform); dtype float16, float32 (default) or float64; ctx is ignored."""
    return _sample('_random_uniform', 'uniform', {'low': low, 'high': high}, shape, dtype, ctx, out, kwargs)


def normal(loc=0, scale=1, shape=None, dtype=None, ctx=None, out=None, **kwargs):
    """Draws samples from N(loc, scale**2) into a new array of `shape` (default (1,)) on `ctx`, or
    into `out` (whose context, shape and dtype then decide). dtype: float16, float32 (default),
    float64, or bfloat16 (an extension; the float32 draw rounded once). Number loc and scale: scale
    must be positive. NDArray loc and scale draw as uniform's NDArray form does (_sample_normal)."""
    if _array_params('normal', {'loc': loc, 'scale': scale}):
        return _sample_params('normal', {'mu': loc, 'sigma': scale}, shape, dtype, out, kwargs)
    if ctx is None:
        ctx = current_context()
    if shape is None and out is None:
        shape = 1
    if shape is not None:
        kwargs['shape'] = _shape_arg(shape)
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
    1.0 / scale), as uniform does. A number scale must be positive; an NDArray scale passes
    lam = 1.0 / scale (_rdiv_scalar) to _sample_exponential."""
    return _sample('_random_exponential', 'exponential', {'lam': 1.0 / scale}, shape, dtype, ctx, out, kwargs)


def gamma(alpha=1, beta=1, shape=None, dtype=None, ctx=None, out=None, **kwargs):
    """Draws samples from the gamma distribution of shape `alpha` and scale `beta`, as uniform does.
    Numbers: alpha and beta must be positive and alpha finite. NDArrays (_sample_gamma) are not
    checked, as in the reference; an element whose draw cannot end (alpha NaN, +-inf or <= -2/3) is
    NaN."""
    return _sample('_random_gamma', 'gamma', {'alpha': alpha, 'beta': beta}, shape, dtype, ctx, out, kwargs)


def randint(low, high, shape=None, dtype=None, ctx=None, out=None, **kwargs):
    """Draws integers uniformly from [low, high) (int64 bounds) into a new array of `shape` (default
    (1,)) on `ctx`, or into `out`. dtype: int32 (default; a value outside int32 wraps) or int64.
    high must be greater than low. low and high are numbers: the reference has no _sample_randint."""
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
