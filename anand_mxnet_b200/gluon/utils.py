"""gluon.utils.clip_global_norm (python/mxnet/gluon/utils.py:118-157) as one operator call."""
import warnings

import numpy as np

from .. import ndarray

__all__ = ['clip_global_norm']


def clip_global_norm(arrays, max_norm, check_isfinite=True):
    """Rescales NDArrays so that the sum of their 2-norm is smaller than `max_norm`.

    The arrays (float32, dense or row_sparse, all on one GPU) are scaled in place by
    min(max_norm / (total_norm + 1e-8), 1) in one `_b200kv_clip_global_norm` call that never waits on
    the host. When the total norm is inf or nan the arrays are left as they are.

    Parameters
    ----------
    arrays : list of NDArray
    max_norm : float
    check_isfinite : bool, default True
         If True, check that the total_norm is finite (not nan or inf). This
         requires a blocking .asscalar() call.

    Returns
    -------
    NDArray or float
      Total norm. Return type is NDArray of shape (1,) if check_isfinite is
      False. Otherwise a float is returned.
    """
    assert len(arrays) > 0
    total_norm = ndarray._invoke('_b200kv_clip_global_norm', list(arrays), num_arrays=len(arrays),
                                 max_norm=max_norm)
    if check_isfinite:
        norm = float(total_norm.asscalar())
        if not np.isfinite(norm):
            warnings.warn(
                UserWarning('nan or inf is detected. '
                            'Clipping results will be undefined.'), stacklevel=2)
        return norm
    return total_norm
