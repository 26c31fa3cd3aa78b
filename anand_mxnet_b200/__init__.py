"""anand_mxnet_b200 -- H100-native KVStore hot path (reduce + optimizer + broadcast) behind the
reference's own interfaces.

    import anand_mxnet_b200 as mx
    kv = mx.kv.create('device')
    kv.init(3, mx.nd.ones((2, 3), mx.gpu(0)))
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9))
    kv.pushpull(3, [g0, g1], out=[w0, w1])

Only the KVStore path exists here (see DESIGN.md); importing this package loads libb200kv.so and
fails when the CUDA library cannot be built/loaded.
"""
from . import base
from .base import MXNetError
from .context import Context, cpu, gpu, cpu_pinned
from . import ndarray
from . import ndarray as nd
from . import random
from . import optimizer
from . import gluon
from . import kvstore
from . import kvstore as kv
from . import dist
from .kvstore import KVStore, KVStoreBase, create as _create_kvstore

__version__ = "0.1.0"
