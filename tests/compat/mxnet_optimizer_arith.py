"""TEST INFRASTRUCTURE -- the Adamax, Nadam and AdaDelta optimizers of the reference's Python
front-end (python/mxnet/optimizer/optimizer.py:1768-1825 AdaDelta, :1904-1959 Adamax, :1962-2029
Nadam) for this package's NDArray, on top of the Optimizer base class and Updater of
tests/compat/mxnet_optimizer.py. Their update rules compose NDArray arithmetic (`+ - * /` of arrays
and scalars, `x[:] op= y`, clip, maximum, abs, sqrt); each operation is one library operator. The
operator sequence, every scalar each one receives and the states are those of the reference's
classes (tests/test_arith_ops_host.py holds them to it). Like its siblings this is NOT part of the
product: in a real integration the reference's own file plays this role unchanged.
"""
from anand_mxnet_b200.ndarray import NDArray, zeros, clip, sqrt, maximum, abs as NDabs
from compat.mxnet_optimizer import Optimizer, register, get_updater  # noqa: F401  (get_updater re-exported)

__all__ = ['Adamax', 'Nadam', 'AdaDelta', 'get_updater']


def _clipped(opt, grad):
    """the gradient clipped to +-clip_gradient whenever one is set, 0 included"""
    if opt.clip_gradient is None:
        return grad
    return clip(grad, -opt.clip_gradient, opt.clip_gradient)


@register
class Adamax(Optimizer):
    """Adam under the infinity norm (Kingma & Ba, section 7). States: the first moment and the
    running maximum of |grad|, in the weight's dtype."""

    def __init__(self, learning_rate=0.002, beta1=0.9, beta2=0.999, **kwargs):
        super(Adamax, self).__init__(learning_rate=learning_rate, **kwargs)
        self.beta1 = beta1
        self.beta2 = beta2

    def create_state(self, index, weight):
        return tuple(zeros(weight.shape, weight.context, dtype=weight.dtype) for _ in range(2))

    def update(self, index, weight, grad, state):
        assert isinstance(weight, NDArray) and isinstance(grad, NDArray)
        self._update_count(index)
        lr = self._get_lr(index)
        wd = self._get_wd(index)
        lr /= (1. - self.beta1 ** self._index_update_count[index])
        g = _clipped(self, grad * self.rescale_grad + wd * weight)
        mean, peak = state
        mean[:] *= self.beta1
        mean[:] += (1. - self.beta1) * g
        peak[:] = maximum(self.beta2 * peak, NDabs(g))
        weight[:] -= lr * mean / peak


@register
class Nadam(Optimizer):
    """Adam with Nesterov momentum and a warming momentum schedule. `m_schedule`, the product of
    every momentum used so far, belongs to the optimizer: it advances once per key update."""

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8,
                 schedule_decay=0.004, **kwargs):
        super(Nadam, self).__init__(learning_rate=learning_rate, **kwargs)
        self.beta1 = beta1
        self.beta2 = beta2
        self.epsilon = epsilon
        self.schedule_decay = schedule_decay
        self.m_schedule = 1.

    def create_state(self, index, weight):
        return tuple(zeros(weight.shape, weight.context, dtype=weight.dtype) for _ in range(2))

    def _momentum(self, t):
        return self.beta1 * (1. - 0.5 * (0.96 ** (t * self.schedule_decay)))

    def update(self, index, weight, grad, state):
        assert isinstance(weight, NDArray) and isinstance(grad, NDArray)
        self._update_count(index)
        lr = self._get_lr(index)
        wd = self._get_wd(index)
        t = self._index_update_count[index]
        g = _clipped(self, grad * self.rescale_grad + wd * weight)
        mom_now, mom_next = self._momentum(t), self._momentum(t + 1)
        self.m_schedule = self.m_schedule * mom_now
        schedule_next = self.m_schedule * mom_next
        mean, var = state
        mean[:] *= self.beta1
        mean[:] += (1. - self.beta1) * g
        var[:] *= self.beta2
        var[:] += (1. - self.beta2) * g * g
        g_hat = g / (1. - self.m_schedule)
        mean_hat = mean / (1. - schedule_next)
        var_hat = var / (1. - self.beta2 ** t)
        mean_bar = (1. - mom_now) * g_hat + mom_next * mean_hat
        weight[:] -= lr * mean_bar / (sqrt(var_hat) + self.epsilon)


@register
class AdaDelta(Optimizer):
    """AdaDelta (Zeiler, 2012): no learning rate. States: the running averages of squared gradients
    and of squared steps, float32. The gradient is rescaled in place, so the caller's array holds
    grad * rescale_grad afterwards."""

    def __init__(self, rho=0.90, epsilon=1e-5, **kwargs):
        super(AdaDelta, self).__init__(**kwargs)
        self.rho = rho
        self.epsilon = epsilon

    def create_state(self, index, weight):
        return tuple(zeros(weight.shape, weight.context) for _ in range(2))

    def update(self, index, weight, grad, state):
        assert isinstance(weight, NDArray) and isinstance(grad, NDArray)
        wd = self._get_wd(index)
        self._update_count(index)
        grad *= self.rescale_grad
        g = _clipped(self, grad)
        sq_grad, sq_step = state
        sq_grad[:] *= self.rho
        sq_grad[:] += (1. - self.rho) * g * g
        step = sqrt(sq_step + self.epsilon) / sqrt(sq_grad + self.epsilon) * g
        sq_step[:] *= self.rho
        sq_step[:] += (1. - self.rho) * step * step
        weight[:] -= step + wd * weight
