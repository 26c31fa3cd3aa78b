"""TEST INFRASTRUCTURE -- a mirror of the reference's amp.unscale
(python/mxnet/contrib/amp/amp.py:331-352) for this package's NDArray: the per-gradient
`g[:] *= trainer._scale` becomes one bulk `contrib.multi_scale` call per device, which multiplies
by the same float32 factor. It is NOT part of the product: anand_mxnet_b200/ never imports it.
"""
from anand_mxnet_b200 import ndarray as nd
from anand_mxnet_b200 import optimizer as fused

from . import mxnet_optimizer as opt


def unscale(optimizer_or_trainer):
    """Check and unscale the gradients manually. This function should only be used
    if accessing gradients is necessary, e.g. for gradient clipping.

    A trainer is anything with `_params` (each with `_grad`, the per-device gradient list or None)
    and `_scale`, which is what the reference reads of a gluon Trainer."""
    if hasattr(optimizer_or_trainer, '_params') and hasattr(optimizer_or_trainer, '_scale'):
        valid_grads = [p._grad for p in optimizer_or_trainer._params if p._grad is not None]
        n_dev = max((len(grads) for grads in valid_grads), default=0)
        for d in range(n_dev):
            per_dev = [grads[d] for grads in valid_grads if len(grads) > d]
            nd.contrib.multi_scale(*per_dev, scalar=optimizer_or_trainer._scale)
        optimizer_or_trainer._scale = 1.
    elif isinstance(optimizer_or_trainer, (opt.Optimizer, fused.FusedOptimizer)):
        raise TypeError("AMP is currently only compatible with Gluon Trainer")
    else:
        raise TypeError("optimizer_or_trainer should be a Gluon Trainer or "
                        "an optimizer, instead is %s" % type(optimizer_or_trainer))
