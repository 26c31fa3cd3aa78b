"""TEST INFRASTRUCTURE -- mirror of the reference's NAG, Signum, RMSProp, FTML and Ftrl optimizers
(python/mxnet/optimizer/optimizer.py :673-737 Signum, :740-795 FTML, :1433-1507 NAG, :1691-1766
RMSProp, :1829-1901 Ftrl) for this package's NDArray, on top of the Optimizer base class and Updater
of tests/compat/mxnet_optimizer.py. Their update rules are the library's single-tensor operators
(nag_mom_update, signum_update, rmsprop_update, ...); the store runs them through the per-key
updater callback. Like its sibling this is NOT part of the product: in a real integration the
reference's own file plays this role unchanged.
"""
import warnings

import numpy

from anand_mxnet_b200.ndarray import (NDArray, zeros, sgd_update, mp_sgd_update, nag_mom_update,
                                      mp_nag_mom_update, signsgd_update, signum_update, rmsprop_update,
                                      rmspropalex_update, ftml_update, ftrl_update)
from compat.mxnet_optimizer import Optimizer, register, get_updater  # noqa: F401  (get_updater re-exported)

__all__ = ['NAG', 'Signum', 'RMSProp', 'FTML', 'Ftrl', 'get_updater']


@register
class Signum(Optimizer):
    """optimizer.py:673-737: signum_update with a momentum state, signsgd_update without"""

    def __init__(self, learning_rate=0.01, momentum=0.9, wd_lh=0.0, **kwargs):
        super(Signum, self).__init__(learning_rate=learning_rate, **kwargs)
        self.momentum = momentum
        self.wd_lh = wd_lh

    def create_state(self, index, weight):
        momentum = None
        if self.momentum != 0.0:
            momentum = zeros(weight.shape, weight.context, dtype=weight.dtype, stype=weight.stype)
        return momentum

    def _update_impl(self, index, weight, grad, state):
        assert(isinstance(weight, NDArray))
        assert(isinstance(grad, NDArray))
        self._update_count(index)
        lr = self._get_lr(index)
        wd = self._get_wd(index)
        kwargs = {'rescale_grad': self.rescale_grad}
        if self.momentum > 0:
            kwargs['momentum'] = self.momentum
        if self.clip_gradient:
            kwargs['clip_gradient'] = self.clip_gradient
        if self.wd_lh:
            kwargs['wd_lh'] = self.wd_lh
        if state is not None:
            signum_update(weight, grad, state, out=weight, lr=lr, wd=wd, **kwargs)
        else:
            signsgd_update(weight, grad, out=weight, lr=lr, wd=wd, **kwargs)

    def update(self, index, weight, grad, state):
        self._update_impl(index, weight, grad, state)


@register
class FTML(Optimizer):
    """optimizer.py:740-795: states (d, v, z); t is the index's update count"""

    def __init__(self, beta1=0.6, beta2=0.999, epsilon=1e-8, **kwargs):
        super(FTML, self).__init__(**kwargs)
        self.beta1 = beta1
        self.beta2 = beta2
        self.epsilon = epsilon

    def create_state(self, index, weight):
        return (zeros(weight.shape, weight.context, dtype=weight.dtype),   # d_0
                zeros(weight.shape, weight.context, dtype=weight.dtype),   # v_0
                zeros(weight.shape, weight.context, dtype=weight.dtype))   # z_0

    def update(self, index, weight, grad, state):
        assert(isinstance(weight, NDArray))
        assert(isinstance(grad, NDArray))
        self._update_count(index)
        lr = self._get_lr(index)
        wd = self._get_wd(index)
        t = self._index_update_count[index]
        kwargs = {'beta1': self.beta1, 'beta2': self.beta2, 'epsilon': self.epsilon,
                  'rescale_grad': self.rescale_grad, 't': t}
        if self.clip_gradient:
            kwargs['clip_grad'] = self.clip_gradient
        prev_d, prev_v, prev_z = state
        ftml_update(weight, grad, prev_d, prev_v, prev_z, out=weight, lr=lr, wd=wd, **kwargs)


@register
class NAG(Optimizer):
    """optimizer.py:1433-1507: nag_mom_update / mp_nag_mom_update; sgd_update / mp_sgd_update when
    momentum is 0. Its multi-precision state is (momentum, weight32)."""

    def __init__(self, momentum=0.0, **kwargs):
        super(NAG, self).__init__(**kwargs)
        self.momentum = momentum

    def create_state_multi_precision(self, index, weight):
        weight_master_copy = None
        if self.multi_precision and weight.dtype == numpy.float16:
            weight_master_copy = weight.astype(numpy.float32)
            return (self.create_state(index, weight_master_copy), weight_master_copy)
        if weight.dtype == numpy.float16 and not self.multi_precision:
            warnings.warn("Accumulating with float16 in optimizer can lead to poor accuracy or slow "
                          "convergence. Consider using multi_precision=True option of the NAG optimizer")
        return self.create_state(index, weight)

    def create_state(self, index, weight):
        momentum = None
        if self.momentum != 0.0:
            momentum = zeros(weight.shape, weight.context, dtype=weight.dtype)
        return momentum

    def _update_impl(self, index, weight, grad, state, multi_precision=False):
        assert(isinstance(weight, NDArray))
        assert(isinstance(grad, NDArray))
        self._update_count(index)
        lr = self._get_lr(index)
        wd = self._get_wd(index)
        kwargs = {'rescale_grad': self.rescale_grad}
        if self.momentum > 0:
            kwargs['momentum'] = self.momentum
        if self.clip_gradient:
            kwargs['clip_gradient'] = self.clip_gradient
        if not multi_precision:
            if state is not None:
                nag_mom_update(weight, grad, state, out=weight, lr=lr, wd=wd, **kwargs)
            else:
                sgd_update(weight, grad, out=weight, lr=lr, wd=wd, **kwargs)
        else:
            if state[0] is not None:
                mp_nag_mom_update(weight, grad, state[0], state[1], out=weight, lr=lr, wd=wd, **kwargs)
            else:
                mp_sgd_update(weight, grad, state[1], out=weight, lr=lr, wd=wd, **kwargs)

    def update(self, index, weight, grad, state):
        self._update_impl(index, weight, grad, state, multi_precision=False)

    def update_multi_precision(self, index, weight, grad, state):
        use_multi_precision = self.multi_precision and weight.dtype == numpy.float16 \
            and isinstance(state, (tuple, list))
        self._update_impl(index, weight, grad, state, multi_precision=use_multi_precision)


@register
class RMSProp(Optimizer):
    """optimizer.py:1691-1766: rmsprop_update (state n), or rmspropalex_update (states n, g, delta)
    when centered"""

    def __init__(self, learning_rate=0.001, gamma1=0.9, gamma2=0.9, epsilon=1e-8, centered=False,
                 clip_weights=None, **kwargs):
        super(RMSProp, self).__init__(learning_rate=learning_rate, **kwargs)
        self.gamma1 = gamma1
        self.gamma2 = gamma2
        self.centered = centered
        self.epsilon = epsilon
        self.clip_weights = clip_weights

    def create_state(self, index, weight):
        if self.centered:
            return (zeros(weight.shape, weight.context, stype=weight.stype),   # n
                    zeros(weight.shape, weight.context, stype=weight.stype),   # g
                    zeros(weight.shape, weight.context, stype=weight.stype))   # delta
        return (zeros(weight.shape, weight.context, stype=weight.stype),)      # n

    def update(self, index, weight, grad, state):
        assert(isinstance(weight, NDArray))
        assert(isinstance(grad, NDArray))
        self._update_count(index)
        lr = self._get_lr(index)
        wd = self._get_wd(index)
        kwargs = {'gamma1': self.gamma1, 'epsilon': self.epsilon, 'rescale_grad': self.rescale_grad}
        if self.centered:
            kwargs['gamma2'] = self.gamma2
        if self.clip_gradient:
            kwargs['clip_gradient'] = self.clip_gradient
        if self.clip_weights:
            kwargs['clip_weights'] = self.clip_weights
        if not self.centered:
            (n, ) = state
            rmsprop_update(weight, grad, n, out=weight, lr=lr, wd=wd, **kwargs)
        else:
            n, g, delta = state
            rmspropalex_update(weight, grad, n, g, delta, out=weight, lr=lr, wd=wd, **kwargs)


@register
class Ftrl(Optimizer):
    """optimizer.py:1829-1901: states (z, n); the learning rate is set after the base class"""

    def __init__(self, lamda1=0.01, learning_rate=0.1, beta=1, **kwargs):
        super(Ftrl, self).__init__(**kwargs)
        self.lamda1 = lamda1
        self.beta = beta
        self.lr = learning_rate

    def create_state(self, index, weight):
        return (zeros(weight.shape, weight.context, stype=weight.stype),   # z
                zeros(weight.shape, weight.context, stype=weight.stype))   # n

    def update(self, index, weight, grad, state):
        assert(isinstance(weight, NDArray))
        assert(isinstance(grad, NDArray))
        self._update_count(index)
        wd = self._get_wd(index)
        lr = self._get_lr(index)
        kwargs = {'lamda1': self.lamda1, 'beta': self.beta, 'rescale_grad': self.rescale_grad}
        if self.clip_gradient:
            kwargs['clip_gradient'] = self.clip_gradient
        z, n = state
        ftrl_update(weight, grad, z, n, out=weight, lr=lr, wd=wd, **kwargs)
