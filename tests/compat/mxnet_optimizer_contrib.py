"""TEST INFRASTRUCTURE -- mirror of the reference's GroupAdaGrad optimizer (python/mxnet/optimizer/
contrib.py:30-100) for this package's NDArray, on top of the Optimizer base class and Updater of
tests/compat/mxnet_optimizer.py. GroupAdaGrad trains embedding tables with one AdaGrad history value
per row: its row_sparse branch calls contrib.group_adagrad_update (_contrib_group_adagrad_update),
on a row_sparse table (the store's per-key updater callback) or on a dense table with a row_sparse
gradient (a local updater). Like its siblings this is NOT part of the product: in a real
integration the reference's own file plays this role unchanged.
"""
from anand_mxnet_b200.ndarray import NDArray, zeros, contrib
from compat.mxnet_optimizer import Optimizer, register, get_updater  # noqa: F401  (get_updater re-exported)

__all__ = ['GroupAdaGrad', 'get_updater']


@register
class GroupAdaGrad(Optimizer):
    """contrib.py:30-100: history of shape (rows, 1) in the weight's storage type; a row_sparse
    gradient goes to contrib.group_adagrad_update. The dense-gradient branch is Python NDArray
    arithmetic (mean, square, clip, sqrt) that this package does not serve."""

    def __init__(self, eps=1e-5, **kwargs):
        super(GroupAdaGrad, self).__init__(**kwargs)
        self.float_stable_eps = eps

    def create_state(self, index, weight):
        assert len(weight.shape) == 2
        history = zeros(
            (weight.shape[0], 1), weight.context, stype=weight.stype)
        return history

    def update(self, index, weight, grad, state):
        assert (isinstance(weight, NDArray))
        assert (isinstance(grad, NDArray))
        self._update_count(index)
        lr = self._get_lr(index)
        wd = self._get_wd(index)
        assert wd == 0, 'Weight decay is not supported for GroupAdaGrad'

        is_sparse = grad.stype == 'row_sparse'
        if is_sparse:
            kwargs = {
                'epsilon': self.float_stable_eps,
                'rescale_grad': self.rescale_grad
            }
            if self.clip_gradient:
                kwargs['clip_gradient'] = self.clip_gradient
            contrib.group_adagrad_update(
                weight,
                grad,
                state,
                out=weight,
                lr=lr,
                **kwargs)
        else:
            raise NotImplementedError(
                "GroupAdaGrad with a dense gradient needs the mean / square / clip / sqrt NDArray "
                "operators, which this package does not serve; push row_sparse gradients")
