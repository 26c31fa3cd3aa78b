"""TEST INFRASTRUCTURE -- mirror of the reference's AdaGrad optimizer (python/mxnet/optimizer/
optimizer.py:1632-1688) for this package's NDArray, on top of the Optimizer base class and Updater of
tests/compat/mxnet_optimizer.py. Together with the Ftrl of tests/compat/mxnet_optimizer_update.py
(re-exported here) these are the two optimizers that train row_sparse embedding tables through the
store's per-key updater callback: Ftrl's states take the weight's storage type, so a row_sparse table
reaches the row_sparse form of ftrl_update; AdaGrad's row_sparse branch calls sparse.adagrad_update
(_sparse_adagrad_update). Like its siblings this is NOT part of the product: in a real integration the
reference's own file plays this role unchanged.
"""
from anand_mxnet_b200.ndarray import NDArray, zeros, sparse
from compat.mxnet_optimizer import Optimizer, register, get_updater  # noqa: F401  (get_updater re-exported)
from compat.mxnet_optimizer_update import Ftrl  # noqa: F401  (re-exported)

__all__ = ['AdaGrad', 'Ftrl', 'get_updater']


@register
class AdaGrad(Optimizer):
    """optimizer.py:1632-1688: state history; a row_sparse gradient goes to sparse.adagrad_update.
    The dense-gradient branch is Python NDArray arithmetic (square, clip, division) that this package
    does not serve."""

    def __init__(self, eps=1e-7, **kwargs):
        super(AdaGrad, self).__init__(**kwargs)
        self.float_stable_eps = eps

    def create_state(self, index, weight):
        return zeros(weight.shape, weight.context, stype=weight.stype)  # history

    def update(self, index, weight, grad, state):
        assert(isinstance(weight, NDArray))
        assert(isinstance(grad, NDArray))
        self._update_count(index)
        lr = self._get_lr(index)
        wd = self._get_wd(index)

        is_sparse = grad.stype == 'row_sparse'
        history = state

        if is_sparse:
            kwargs = {'epsilon': self.float_stable_eps,
                      'rescale_grad': self.rescale_grad}
            if self.clip_gradient:
                kwargs['clip_gradient'] = self.clip_gradient
            sparse.adagrad_update(weight, grad, history, out=weight, lr=lr, wd=wd, **kwargs)
        else:
            raise NotImplementedError(
                "AdaGrad with a dense gradient needs the square / clip / division NDArray "
                "operators, which this package does not serve; push row_sparse gradients")
