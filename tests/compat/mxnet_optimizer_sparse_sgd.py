"""TEST INFRASTRUCTURE -- the reference's SGD, ccSGD and Adam (python/mxnet/optimizer/optimizer.py:
526-669, 1542-1546, 1547-1629) for this package's NDArray, with the reference's state storage rule:
a state takes the weight's storage type when lazy_update is set, else it is dense (optimizer.py:
596-601, 1603-1608). A row_sparse table therefore reaches the row_sparse-weight forms of
sgd_update / sgd_mom_update / adam_update: lazy with row_sparse states that hold no rows yet, or
standard with dense states. The classes extend the mirrors of tests/compat/mxnet_optimizer.py, whose
states are always dense, and change nothing else; tests/test_sparse_sgd_adam_host.py holds their
operator calls, parameter strings and signatures to the reference's classes. They are not
registered: the registry keeps the names SGD and Adam for the existing mirrors, and ccSGD is not in
it. Like its siblings this is NOT part of the product: in a real integration the reference's own
file plays this role unchanged.
"""
from anand_mxnet_b200.ndarray import zeros
from compat import mxnet_optimizer as _base
from compat.mxnet_optimizer import get_updater  # noqa: F401  (re-exported)

__all__ = ['SGD', 'ccSGD', 'Adam', 'get_updater']


class SGD(_base.SGD):
    """optimizer.py:526-669; momentum takes the weight's stype when lazy_update is set"""

    def create_state(self, index, weight):
        momentum = None
        if self.momentum != 0.0:
            stype = weight.stype if self.lazy_update else 'default'
            momentum = zeros(weight.shape, weight.context, dtype=weight.dtype, stype=stype)
        return momentum


class ccSGD(SGD):  # noqa: N801  (the reference's name)
    """[DEPRECATED] Same as `SGD`. Left here for backward compatibility (optimizer.py:1542-1546).
    Its class name is not one the store runs in its fused step, so kv.set_optimizer(ccSGD(...))
    calls it back per key."""

    def __init__(self, *args, **kwargs):
        super(ccSGD, self).__init__(*args, **kwargs)


class Adam(_base.Adam):
    """optimizer.py:1547-1629; mean and var take the weight's stype when lazy_update is set"""

    def create_state(self, index, weight):
        stype = weight.stype if self.lazy_update else 'default'
        return (zeros(weight.shape, weight.context, dtype=weight.dtype, stype=stype),  # mean
                zeros(weight.shape, weight.context, dtype=weight.dtype, stype=stype))  # variance
