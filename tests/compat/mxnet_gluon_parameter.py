"""TEST INFRASTRUCTURE -- a mirror of the reference's ParameterDict.zero_grad
(python/mxnet/gluon/parameter.py:889-911) for this package's NDArray: per context, the dense
gradients go to one `reset_arrays` call and each row_sparse gradient to `zeros_like(g, out=g)`, in
the reference's order. The numpy-mode branch (`ele[()] = 0`) is not mirrored. It is NOT part of the
product: anand_mxnet_b200/ never imports it.
"""
from collections import defaultdict

from anand_mxnet_b200 import ndarray


def zero_grad(params):
    """Sets all Parameters' gradient buffer to 0.

    `params` is anything with `values()` giving parameters, each with `grad_req`, `_grad` (None
    when uninitialised) and `list_grad()`, which is what the reference reads of a ParameterDict."""
    arrays = defaultdict(list)
    for p in params.values():
        if p.grad_req == 'null' or p._grad is None:
            continue
        for g in p.list_grad():
            if g.stype == 'row_sparse':
                ndarray.zeros_like(g, out=g)
            else:
                arrays[g.ctx].append(g)

    if len(arrays) == 0:
        return

    for arr in arrays.values():
        ndarray.reset_arrays(*arr, num_arrays=len(arr))
