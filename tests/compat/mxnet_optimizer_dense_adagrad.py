"""TEST INFRASTRUCTURE -- the reference's AdaGrad (python/mxnet/optimizer/optimizer.py:1632-1688) and
GroupAdaGrad (optimizer/contrib.py:30-100) for this package's NDArray, with their dense-gradient
branches. The classes extend the row_sparse-only mirrors of tests/compat/mxnet_optimizer_sparse.py
and tests/compat/mxnet_optimizer_contrib.py: a row_sparse gradient still goes to the fused
row_sparse operator there, a dense gradient runs the NDArray arithmetic here (square, mean over the
last axis, clip, sqrt, the row broadcast of `/`), one library operator per operation. The operator
sequence, every parameter string and the states are those of the reference's classes
(tests/test_dense_adagrad_host.py holds them to it). They are not registered: the names AdaGrad and
GroupAdaGrad stay the row_sparse mirrors' in the registry. Like its siblings this is NOT part of the
product: in a real integration the reference's own files play this role unchanged.
"""
from anand_mxnet_b200.ndarray import NDArray, clip, sqrt, square, mean
from compat import mxnet_optimizer_contrib as _contrib
from compat import mxnet_optimizer_sparse as _sparse
from compat.mxnet_optimizer import get_updater  # noqa: F401  (re-exported)

__all__ = ['AdaGrad', 'GroupAdaGrad', 'get_updater']


def _scaled_clipped(opt, grad):
    """grad * rescale_grad, clipped to +-clip_gradient whenever one is set, 0 included"""
    grad = grad * opt.rescale_grad
    if opt.clip_gradient is not None:
        grad = clip(grad, -opt.clip_gradient, opt.clip_gradient)
    return grad


class AdaGrad(_sparse.AdaGrad):
    """history += grad^2; weight -= lr * (grad / sqrt(history + eps) + wd * weight)"""

    def update(self, index, weight, grad, state):
        if grad.stype == 'row_sparse':
            return super(AdaGrad, self).update(index, weight, grad, state)
        assert isinstance(weight, NDArray) and isinstance(grad, NDArray)
        self._update_count(index)
        lr = self._get_lr(index)
        wd = self._get_wd(index)
        history = state
        g = _scaled_clipped(self, grad)
        history[:] += square(g)
        step = g / sqrt(history + self.float_stable_eps)
        weight[:] += (step + weight * wd) * -lr


class GroupAdaGrad(_contrib.GroupAdaGrad):
    """one history value per row: history += mean(grad^2 over the row); weight -= lr * grad /
    sqrt(history + eps), the history broadcast along each row"""

    def update(self, index, weight, grad, state):
        if grad.stype == 'row_sparse':
            return super(GroupAdaGrad, self).update(index, weight, grad, state)
        assert isinstance(weight, NDArray) and isinstance(grad, NDArray)
        self._update_count(index)
        lr = self._get_lr(index)
        wd = self._get_wd(index)
        assert wd == 0, 'Weight decay is not supported for GroupAdaGrad'
        g = _scaled_clipped(self, grad)
        state[:] += mean(square(g), axis=1, keepdims=True)
        weight[:] -= lr * g / sqrt(state + self.float_stable_eps)
