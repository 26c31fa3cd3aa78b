"""TEST INFRASTRUCTURE -- the SGLD optimizer of the reference's Python front-end
(python/mxnet/optimizer/optimizer.py:1510-1537) for this package's NDArray, on top of the Optimizer
base class and Updater of tests/compat/mxnet_optimizer.py. Its update composes `_mul_scalar`, clip,
`_plus` and one `_random_normal` per call, in the reference's order and with the reference's
scalars. Like its siblings this is NOT part of the product: in a real integration the reference's
own file plays this role unchanged.
"""
import math

from anand_mxnet_b200.ndarray import NDArray, clip
from anand_mxnet_b200.random import normal
from compat.mxnet_optimizer import Optimizer, register, get_updater  # noqa: F401  (get_updater re-exported)

__all__ = ['SGLD', 'get_updater']


@register
class SGLD(Optimizer):
    """Stochastic Gradient Langevin Dynamics: half an SGD step, plus N(0, lr) noise. No state."""

    def __init__(self, **kwargs):
        super(SGLD, self).__init__(**kwargs)

    def create_state(self, index, weight):
        return None

    def update(self, index, weight, grad, state):
        assert isinstance(weight, NDArray)
        assert isinstance(grad, NDArray)
        self._update_count(index)
        lr = self._get_lr(index)
        wd = self._get_wd(index)

        grad = grad * self.rescale_grad
        if self.clip_gradient is not None:
            grad = clip(grad, -self.clip_gradient, self.clip_gradient)
        weight[:] += - lr/2 * (grad + wd * weight)
        weight[:] += normal(0, math.sqrt(lr), shape=weight.shape,
                            dtype=weight.dtype, ctx=weight.context)
