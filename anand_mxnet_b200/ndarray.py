"""NDArray / RowSparseNDArray front-end over the C ABI (the slice of python/mxnet/ndarray/ that the
KVStore path and its tests need): creation, host copies, waits, DLPack interop with torch, the
optimizer operators and the few elementwise operators custom updaters use.

Arithmetic runs on the GPU through MXImperativeInvokeEx; CPU-context arrays are containers only
(create / copy / asnumpy) -- they exist so host-resident gradients can be pushed, as with the
reference's kvstore('local').
"""
import ctypes
import operator
from array import array as _pyarray

import numpy as np

from .base import _LIB, check_call, c_str_array, NDArrayHandle, OpHandle, MXNetError
from .context import Context, cpu, gpu

_DTYPE_NP_TO_MX = {np.dtype(np.float32): 0, np.dtype(np.float64): 1, np.dtype(np.float16): 2,
                   np.dtype(np.uint8): 3, np.dtype(np.int32): 4, np.dtype(np.int8): 5,
                   np.dtype(np.int64): 6}
_DTYPE_MX_TO_NP = {v: k for k, v in _DTYPE_NP_TO_MX.items()}
BFLOAT16 = 12
_STYPE_STR = {0: 'default', 1: 'row_sparse', 2: 'csr', -1: 'undefined'}


def _mx_dtype(dtype):
    if dtype is None:
        return 0
    if isinstance(dtype, str) and dtype == 'bfloat16':
        return BFLOAT16
    return _DTYPE_NP_TO_MX[np.dtype(dtype)]


_op_cache = {}


def _op_handle(name):
    h = _op_cache.get(name)
    if h is None:
        h = OpHandle()
        check_call(_LIB.NNGetOpHandle(name.encode(), ctypes.byref(h)))
        _op_cache[name] = h
    return h


_HV = operator.attrgetter('_hv')
_NULL_OUT = ctypes.POINTER(ctypes.c_void_p)()


def _invoke(op_name, inputs, out=None, **kwargs):
    """MXImperativeInvokeEx the way python/mxnet/_ctypes/ndarray.py:_imperative_invoke does:
    every keyword is formatted with str() and parsed by the operator's parameter struct.
    Handle lists are marshalled through array('Q') buffers, several times cheaper than per-element
    ctypes conversions for a multi-tensor call of hundreds of operands."""
    h = _op_handle(op_name)
    n_in = len(inputs)
    ibuf = _pyarray('Q', map(_HV, inputs))
    in_arr = (ctypes.c_void_p * n_in).from_buffer(ibuf) if n_in else None
    keys = list(kwargs.keys())
    vals = [str(kwargs[k]) for k in keys]
    if out is not None:
        outs = out if isinstance(out, (list, tuple)) else [out]
        n_out = ctypes.c_int(len(outs))
        obuf = _pyarray('Q', map(_HV, outs))
        out_arr = (ctypes.c_void_p * len(outs)).from_buffer(obuf)
        out_ptr = ctypes.cast(out_arr, ctypes.POINTER(ctypes.c_void_p))
    else:
        n_out = ctypes.c_int(0)
        out_ptr = ctypes.POINTER(ctypes.c_void_p)()
    stypes = ctypes.POINTER(ctypes.c_int)()
    check_call(_LIB.MXImperativeInvokeEx(h, ctypes.c_int(n_in), in_arr, ctypes.byref(n_out),
                                         ctypes.byref(out_ptr), ctypes.c_int(len(keys)),
                                         c_str_array(keys), c_str_array(vals), ctypes.byref(stypes)))
    if out is not None:
        return out
    res = [_wrap(NDArrayHandle(out_ptr[i])) for i in range(n_out.value)]
    return res[0] if len(res) == 1 else res


class NDArray(object):
    __slots__ = ['handle', '_hv', '_keepalive', '__weakref__']

    def __init__(self, handle):
        assert isinstance(handle, ctypes.c_void_p)
        self.handle = handle
        self._hv = handle.value      # plain int: list marshalling reads it without ctypes hops
        self._keepalive = None

    def __del__(self):
        try:
            _LIB.MXNDArrayFree(self.handle)
        except Exception:  # interpreter shutdown
            pass

    # ---- metadata
    @property
    def shape(self):
        ndim = ctypes.c_int()
        pdata = ctypes.POINTER(ctypes.c_int)()
        check_call(_LIB.MXNDArrayGetShapeEx(self.handle, ctypes.byref(ndim), ctypes.byref(pdata)))
        return tuple(pdata[i] for i in range(ndim.value))

    @property
    def size(self):
        n = 1
        for d in self.shape:
            n *= d
        return n

    @property
    def _mx_dtype(self):
        t = ctypes.c_int()
        check_call(_LIB.MXNDArrayGetDType(self.handle, ctypes.byref(t)))
        return t.value

    @property
    def dtype(self):
        t = self._mx_dtype
        return 'bfloat16' if t == BFLOAT16 else _DTYPE_MX_TO_NP[t].type

    @property
    def context(self):
        dt, di = ctypes.c_int(), ctypes.c_int()
        check_call(_LIB.MXNDArrayGetContext(self.handle, ctypes.byref(dt), ctypes.byref(di)))
        return Context(Context.devtype2str[dt.value], di.value)

    ctx = context

    @property
    def stype(self):
        s = ctypes.c_int()
        check_call(_LIB.MXNDArrayGetStorageType(self.handle, ctypes.byref(s)))
        return _STYPE_STR[s.value]

    # ---- synchronisation
    def wait_to_read(self):
        check_call(_LIB.MXNDArrayWaitToRead(self.handle))

    def wait_to_write(self):
        check_call(_LIB.MXNDArrayWaitToWrite(self.handle))

    # ---- host copies
    def asnumpy(self):
        t = self._mx_dtype
        if t == BFLOAT16:
            raw = np.empty(self.shape, dtype=np.uint16)
            check_call(_LIB.MXNDArraySyncCopyToCPU(self.handle, raw.ctypes.data_as(ctypes.c_void_p),
                                                   ctypes.c_size_t(raw.size)))
            return (raw.astype(np.uint32) << 16).view(np.float32)
        out = np.empty(self.shape, dtype=_DTYPE_MX_TO_NP[t])
        check_call(_LIB.MXNDArraySyncCopyToCPU(self.handle, out.ctypes.data_as(ctypes.c_void_p),
                                               ctypes.c_size_t(out.size)))
        return out

    def asscalar(self):
        assert self.size == 1
        return self.asnumpy().reshape(-1)[0]

    def _sync_copyfrom(self, src):
        t = self._mx_dtype
        if t == BFLOAT16:
            f = np.ascontiguousarray(src, dtype=np.float32)
            x = f.view(np.uint32).astype(np.uint64)
            src = ((x + 0x7fff + ((x >> 16) & 1)) >> 16).astype(np.uint16)
        else:
            src = np.ascontiguousarray(src, dtype=_DTYPE_MX_TO_NP[t])
        if src.shape != self.shape:
            src = np.broadcast_to(src, self.shape).copy()
        check_call(_LIB.MXNDArraySyncCopyFromCPU(self.handle, src.ctypes.data_as(ctypes.c_void_p),
                                                 ctypes.c_size_t(src.size)))

    def copyto(self, other):
        if isinstance(other, NDArray):
            if other.handle.value == self.handle.value:
                return other
            return _invoke('_copyto', [self], out=other)
        if isinstance(other, Context):
            out = empty(self.shape, other, self.dtype) if self.stype == 'default' else \
                sparse_zeros('row_sparse', self.shape, other, self.dtype)
            return _invoke('_copyto', [self], out=out)
        raise TypeError('copyto does not support type ' + str(type(other)))

    def copy(self):
        return self.copyto(self.context)

    def as_in_context(self, context):
        return self if self.context == context else self.copyto(context)

    def astype(self, dtype):
        name = dtype if isinstance(dtype, str) else np.dtype(dtype).name
        return _invoke('cast', [self], dtype=name)

    def reshape(self, shape):
        # metadata-only view through DLPack of the same memory (dense, contiguous)
        arr = self.asnumpy().reshape(shape)
        return array(arr, self.context, self.dtype)

    def tostype(self, stype):
        if stype == self.stype:
            return self
        if stype == 'row_sparse':
            dense = self.asnumpy()
            rows = np.nonzero(dense.reshape(dense.shape[0], -1).any(axis=1))[0].astype(np.int64)
            return row_sparse_array((dense[rows], rows), shape=self.shape, ctx=self.context,
                                    dtype=self.dtype)
        raise MXNetError('tostype(%s) is not on the KVStore path' % stype)

    # ---- DLPack / torch interop (zero copy)
    def to_dlpack_for_read(self):
        self.wait_to_read()
        return _to_dlpack(self)

    to_dlpack_for_write = to_dlpack_for_read

    # ---- the few operators updaters use (GPU only)
    def _binary(self, other, op_nd, op_scalar, out=None):
        if isinstance(other, NDArray):
            return _invoke(op_nd, [self, other], out=out)
        return _invoke(op_scalar, [self], out=out, scalar=float(other))

    def __add__(self, other):
        return self._binary(other, '_plus', '_plus_scalar')

    __radd__ = __add__

    def __iadd__(self, other):
        return self._binary(other, '_plus', '_plus_scalar', out=self)

    def __sub__(self, other):
        if isinstance(other, NDArray):
            return _invoke('_minus', [self, other])
        return _invoke('_plus_scalar', [self], scalar=-float(other))

    def __isub__(self, other):
        if isinstance(other, NDArray):
            return _invoke('_minus', [self, other], out=self)
        return _invoke('_plus_scalar', [self], out=self, scalar=-float(other))

    def __mul__(self, other):
        return self._binary(other, '_mul', '_mul_scalar')

    __rmul__ = __mul__

    def __imul__(self, other):
        return self._binary(other, '_mul', '_mul_scalar', out=self)

    def __truediv__(self, other):
        return self._binary(other, 'broadcast_div', '_div_scalar')

    def __itruediv__(self, other):
        return self._binary(other, 'broadcast_div', '_div_scalar', out=self)

    def __rtruediv__(self, other):
        """scalar / array (_rdiv_scalar), floating dtypes only"""
        return _invoke('_rdiv_scalar', [self], scalar=float(other))

    __rdiv__ = __rtruediv__

    def __getitem__(self, key):
        """a[b:e] on the first axis: a view sharing memory (MXNDArraySlice, ndarray.py:_slice)"""
        if isinstance(key, int):
            key = slice(key, key + 1)
        if not isinstance(key, slice) or key.step not in (None, 1):
            raise MXNetError('only contiguous slices of the first axis are supported')
        begin, end, _ = key.indices(self.shape[0])
        h = NDArrayHandle()
        check_call(_LIB.MXNDArraySlice(self.handle, ctypes.c_uint(begin), ctypes.c_uint(end),
                                       ctypes.byref(h)))
        return NDArray(h)

    def norm(self):
        return norm(self)

    def mean(self, axis=None, keepdims=False, exclude=False, out=None):
        return mean(self, axis=axis, keepdims=keepdims, exclude=exclude, out=out)

    def __setitem__(self, key, value):
        if not (isinstance(key, slice) and key == slice(None)):
            raise MXNetError('only full-slice assignment (a[:] = v) is supported')
        if isinstance(value, NDArray):
            if value.handle.value != self.handle.value:
                value.copyto(self)
        elif isinstance(value, (int, float, np.generic)):
            if self.context.device_type == 'gpu':
                # the reference's _full (ndarray.py:504): value=float(value), cast to the dtype
                _invoke('_full', [], out=self, value=float(value))
            else:
                self._sync_copyfrom(np.full(self.shape, value))
        else:
            self._sync_copyfrom(np.asarray(value))

    def __repr__(self):
        return '\n%s\n<%s %s @%s>' % (str(self.asnumpy()), self.__class__.__name__,
                                      'x'.join(str(x) for x in self.shape), self.context)

    # pickling (optimizer-state checkpoints, optimizer.py:2143-2161): the state is the array's
    # NDArray::Save bytes under the key 'handle', exactly as python/mxnet/ndarray/ndarray.py does
    def __getstate__(self):
        length = ctypes.c_size_t()
        cptr = ctypes.POINTER(ctypes.c_char)()
        check_call(_LIB.MXNDArraySaveRawBytes(self.handle, ctypes.byref(length), ctypes.byref(cptr)))
        return {'handle': bytearray(ctypes.string_at(cptr, length.value))}

    def __setstate__(self, state):
        if 'handle' in state:
            buf = state['handle']
            raw = (ctypes.c_char * len(buf)).from_buffer(buf if isinstance(buf, bytearray) else bytearray(buf))
            h = NDArrayHandle()
            check_call(_LIB.MXNDArrayLoadFromRawBytes(raw, ctypes.c_size_t(len(buf)), ctypes.byref(h)))
        else:  # states written by earlier versions of this package
            a = array(state['np'], Context(*state['ctx']), state['dtype'])
            h, a.handle = a.handle, ctypes.c_void_p(None)
        self.handle = h
        self._hv = h.value
        self._keepalive = None
        st = ctypes.c_int()
        check_call(_LIB.MXNDArrayGetStorageType(h, ctypes.byref(st)))
        if st.value == 1 and type(self) is NDArray:
            self.__class__ = RowSparseNDArray


class RowSparseNDArray(NDArray):
    """row_sparse array: `indices` (int64, ascending) + `data` rows (python/mxnet/ndarray/sparse.py)."""
    __slots__ = []

    @property
    def indices(self):
        h = NDArrayHandle()
        check_call(_LIB.MXNDArrayGetAuxNDArray(self.handle, ctypes.c_uint(0), ctypes.byref(h)))
        return NDArray(h)

    @property
    def data(self):
        h = NDArrayHandle()
        check_call(_LIB.MXNDArrayGetDataNDArray(self.handle, ctypes.byref(h)))
        return NDArray(h)

    def asnumpy(self):
        self.wait_to_read()
        out = np.zeros(self.shape, dtype=_DTYPE_MX_TO_NP[self._mx_dtype])
        idx = self.indices
        if idx.shape[0] > 0:
            out[idx.asnumpy()] = self.data.asnumpy()
        return out

    def tostype(self, stype):
        if stype == 'row_sparse':
            return self
        if stype == 'default':
            return array(self.asnumpy(), self.context, self.dtype)
        raise MXNetError('tostype(%s) is not on the KVStore path' % stype)

    def copyto(self, other):
        if isinstance(other, Context):
            out = sparse_zeros('row_sparse', self.shape, other, self.dtype)
            return _invoke('_copyto', [self], out=out)
        return _invoke('_copyto', [self], out=other)


def _wrap(handle):
    s = ctypes.c_int()
    check_call(_LIB.MXNDArrayGetStorageType(handle, ctypes.byref(s)))
    return RowSparseNDArray(handle) if s.value == 1 else NDArray(handle)


_ndarray_cls = _wrap


def _ctx(ctx):
    return ctx if ctx is not None else cpu()


def empty(shape, ctx=None, dtype=None):
    if isinstance(shape, int):
        shape = (shape,)
    ctx = _ctx(ctx)
    h = NDArrayHandle()
    arr = (ctypes.c_uint32 * len(shape))(*shape)
    check_call(_LIB.MXNDArrayCreateEx(arr, ctypes.c_uint32(len(shape)), ctypes.c_int(ctx.device_typeid),
                                      ctypes.c_int(ctx.device_id), ctypes.c_int(0),
                                      ctypes.c_int(_mx_dtype(dtype)), ctypes.byref(h)))
    return NDArray(h)


def array(source, ctx=None, dtype=None):
    if isinstance(source, NDArray):
        source = source.asnumpy()
    src = np.asarray(source)
    if dtype is None:
        dtype = np.float32 if src.dtype.kind == 'f' or not isinstance(source, np.ndarray) else src.dtype
    out = empty(src.shape, ctx, dtype)
    out._sync_copyfrom(src)
    return out


def zeros(shape, ctx=None, dtype=None, stype=None):
    if stype in ('row_sparse',):
        return sparse_zeros(stype, shape, ctx, dtype)
    if isinstance(shape, int):
        shape = (shape,)
    return array(np.zeros(shape, dtype=np.float32), ctx, dtype or np.float32)


def ones(shape, ctx=None, dtype=None):
    if isinstance(shape, int):
        shape = (shape,)
    return array(np.ones(shape, dtype=np.float32), ctx, dtype or np.float32)


def full(shape, val, ctx=None, dtype=None):
    if isinstance(shape, int):
        shape = (shape,)
    return array(np.full(shape, val, dtype=np.float32), ctx, dtype or np.float32)


def sparse_zeros(stype, shape, ctx=None, dtype=None):
    assert stype == 'row_sparse', 'only row_sparse is on the KVStore path'
    ctx = _ctx(ctx)
    h = NDArrayHandle()
    arr = (ctypes.c_uint32 * len(shape))(*shape)
    aux_type = (ctypes.c_int * 1)(6)
    aux_ndims = (ctypes.c_uint32 * 1)(1)
    aux_shape = (ctypes.c_uint32 * 1)(0)
    check_call(_LIB.MXNDArrayCreateSparseEx(ctypes.c_int(1), arr, ctypes.c_uint32(len(shape)),
                                            ctypes.c_int(ctx.device_typeid), ctypes.c_int(ctx.device_id),
                                            ctypes.c_int(1), ctypes.c_int(_mx_dtype(dtype)),
                                            ctypes.c_uint32(1), aux_type, aux_ndims, aux_shape,
                                            ctypes.byref(h)))
    return RowSparseNDArray(h)


def row_sparse_array(arg1, shape=None, ctx=None, dtype=None):
    """row_sparse_array((data, indices), shape=...) as python/mxnet/ndarray/sparse.py:1014-1130."""
    if isinstance(arg1, RowSparseNDArray):
        return arg1.copyto(_ctx(ctx))
    if isinstance(arg1, tuple) and len(arg1) == 2:
        data, indices = arg1
        data = data.asnumpy() if isinstance(data, NDArray) else np.asarray(data)
        indices = indices.asnumpy() if isinstance(indices, NDArray) else np.asarray(indices)
        dtype = dtype or (data.dtype if data.dtype.kind == 'f' and data.dtype != np.float64 else np.float32)
        assert shape is not None and len(indices) == data.shape[0]
        assert np.all(np.diff(indices) > 0), 'row indices must be ascending and unique'
        out = sparse_zeros('row_sparse', shape, ctx, dtype)
        if len(indices) > 0:
            d = array(data.reshape((len(indices),) + tuple(shape[1:])), _ctx(ctx), dtype)
            i = array(indices.astype(np.int64), _ctx(ctx), np.int64)
            check_call(_LIB.MXNDArraySyncCopyFromNDArray(out.handle, d.handle, ctypes.c_int(-1)))
            check_call(_LIB.MXNDArraySyncCopyFromNDArray(out.handle, i.handle, ctypes.c_int(0)))
        return out
    dense = np.asarray(arg1)
    return array(dense, ctx, dtype).tostype('row_sparse')


class _Sparse(object):
    zeros = staticmethod(sparse_zeros)
    row_sparse_array = staticmethod(row_sparse_array)
    RowSparseNDArray = RowSparseNDArray


sparse = _Sparse()


def save(fname, data):
    """mx.nd.save (python/mxnet/ndarray/utils.py:222-273): a list of arrays or a dict name -> array"""
    if isinstance(data, NDArray):
        data = [data]
    if isinstance(data, dict):
        keys, arrs = list(data.keys()), list(data.values())
        ckeys = c_str_array(keys)
    else:
        arrs, ckeys = list(data), None
    handles = (ctypes.c_void_p * len(arrs))(*[a.handle.value for a in arrs])
    check_call(_LIB.MXNDArraySave(fname.encode(), ctypes.c_uint(len(arrs)), handles, ckeys))


def load(fname):
    """mx.nd.load (utils.py:149-182): list, or dict when the file holds names"""
    n, nn = ctypes.c_uint(), ctypes.c_uint()
    harr = ctypes.POINTER(ctypes.c_void_p)()
    names = ctypes.POINTER(ctypes.c_char_p)()
    check_call(_LIB.MXNDArrayLoad(fname.encode(), ctypes.byref(n), ctypes.byref(harr), ctypes.byref(nn),
                                  ctypes.byref(names)))
    arrs = [_wrap(NDArrayHandle(harr[i])) for i in range(n.value)]
    if nn.value == 0:
        return arrs
    return {names[i].decode(): arrs[i] for i in range(n.value)}


def waitall():
    check_call(_LIB.MXNDArrayWaitAll())


# ------------------------------------------------------------------------------------------ DLPack
_c_str_dltensor = b'dltensor'
_c_str_used_dltensor = b'used_dltensor'
ctypes.pythonapi.PyCapsule_GetPointer.restype = ctypes.c_void_p
ctypes.pythonapi.PyCapsule_GetPointer.argtypes = [ctypes.py_object, ctypes.c_char_p]
ctypes.pythonapi.PyCapsule_IsValid.restype = ctypes.c_int
ctypes.pythonapi.PyCapsule_IsValid.argtypes = [ctypes.py_object, ctypes.c_char_p]
ctypes.pythonapi.PyCapsule_SetName.argtypes = [ctypes.py_object, ctypes.c_char_p]
ctypes.pythonapi.PyCapsule_New.restype = ctypes.py_object
ctypes.pythonapi.PyCapsule_New.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p]


def from_dlpack(capsule):
    """Zero-copy NDArray over a DLPack capsule (python/mxnet/dlpack.py ndarray_from_dlpack)."""
    assert ctypes.pythonapi.PyCapsule_IsValid(capsule, _c_str_dltensor), \
        'Invalid DLPack Tensor. DLTensor capsules can be consumed only once.'
    ptr = ctypes.pythonapi.PyCapsule_GetPointer(capsule, _c_str_dltensor)
    h = NDArrayHandle()
    check_call(_LIB.MXNDArrayFromDLPackEx(ctypes.c_void_p(ptr), ctypes.c_bool(False), ctypes.byref(h)))
    ctypes.pythonapi.PyCapsule_SetName(capsule, _c_str_used_dltensor)
    return NDArray(h)


def from_torch(t):
    """Zero-copy view of a contiguous torch tensor; the tensor is kept alive by the NDArray."""
    import torch.utils.dlpack as tdl
    nd = from_dlpack(tdl.to_dlpack(t))
    nd._keepalive = t
    return nd


def _to_dlpack(nd):
    p = ctypes.c_void_p()
    check_call(_LIB.MXNDArrayToDLPack(nd.handle, ctypes.byref(p)))
    return ctypes.pythonapi.PyCapsule_New(p, _c_str_dltensor, None)


def to_torch(nd):
    import torch.utils.dlpack as tdl
    return tdl.from_dlpack(nd.to_dlpack_for_read())


# ------------------------------------------------------------------------------------------ operators
def _op(name):
    def f(*args, **kwargs):
        out = kwargs.pop('out', None)
        return _invoke(name, list(args), out=out, **kwargs)
    f.__name__ = name
    return f


sgd_update = _op('sgd_update')
# the multi-sample operators under the reference's generated names: sample_uniform(low, high,
# shape=(), dtype=None, out=None) and likewise sample_normal(mu, sigma), sample_gamma(alpha, beta),
# sample_exponential(lam)
sample_uniform = _op('sample_uniform')
sample_normal = _op('sample_normal')
sample_gamma = _op('sample_gamma')
sample_exponential = _op('sample_exponential')
sgd_mom_update = _op('sgd_mom_update')
mp_sgd_update = _op('mp_sgd_update')
mp_sgd_mom_update = _op('mp_sgd_mom_update')
multi_sgd_update = _op('multi_sgd_update')
multi_sgd_mom_update = _op('multi_sgd_mom_update')
multi_mp_sgd_update = _op('multi_mp_sgd_update')
multi_mp_sgd_mom_update = _op('multi_mp_sgd_mom_update')
adam_update = _op('adam_update')
# the operators of the reference's NAG / Signum / RMSProp / FTML / Ftrl optimizers (dense float32;
# mp_nag_mom_update: float16 / bfloat16 weights with float32 mom and weight32)
nag_mom_update = _op('nag_mom_update')
mp_nag_mom_update = _op('mp_nag_mom_update')
signsgd_update = _op('signsgd_update')
signum_update = _op('signum_update')
rmsprop_update = _op('rmsprop_update')
rmspropalex_update = _op('rmspropalex_update')
ftml_update = _op('ftml_update')
ftrl_update = _op('ftrl_update')
# mx.nd.sparse.*: row updates driven by a row_sparse gradient (float32, out must be the weight):
# ftrl_update on row_sparse weight / grad / z / n (mx.nd.ftrl_update takes the same form from its
# operands' storage types), adagrad_update on (row_sparse, row_sparse, row_sparse) or (dense,
# row_sparse, dense) with wd = 0. sgd_update, sgd_mom_update and adam_update are the operators of
# mx.nd under their sparse names: on a row_sparse weight that holds every row, lazy_update=True
# moves the gradient's rows and lazy_update=False every row; their states are row_sparse (every
# row, or none yet: zero-filled first) or dense (the standard form)
_Sparse.ftrl_update = staticmethod(_op('_sparse_ftrl_update'))
_Sparse.adagrad_update = staticmethod(_op('_sparse_adagrad_update'))
_Sparse.sgd_update = staticmethod(_op('sgd_update'))
_Sparse.sgd_mom_update = staticmethod(_op('sgd_mom_update'))
_Sparse.adam_update = staticmethod(_op('adam_update'))
# mx.nd.sparse.zeros_like: the _sparse_zeros_like alias of zeros_like (init_op.cc:153-154)
_Sparse.zeros_like = staticmethod(_op('_sparse_zeros_like'))
cast = _op('cast')
multi_sum_sq = _op('multi_sum_sq')
multi_lars = _op('multi_lars')
# AMP's gradient overflow check: out (a (1,) float32 array, created on the inputs' GPU when not
# given) is set to 1 when init_output (default True), then to 0 if any element of any input is
# inf or nan. multi_all_finite(*arrays, num_arrays=len(arrays), init_output=..., out=...)
all_finite = _op('all_finite')
multi_all_finite = _op('multi_all_finite')
# ParameterDict.zero_grad's bulk reset: every input (float16 / bfloat16 / float32 / float64, one GPU)
# zeroed in place, one launch per 200 dense arrays; row_sparse inputs end with no stored rows.
# reset_arrays(*arrays, num_arrays=len(arrays)); no output
reset_arrays = _op('reset_arrays')
# zeros of data's shape and dtype; a row_sparse data or out gives a row_sparse array with no rows
zeros_like = _op('zeros_like')


def _sum_op(name):
    """add_n(*arrays, out=None): the element-wise sum of arrays of one shape and dtype on one GPU.
    num_args is len(arrays) unless given, as the reference's generated function fills it in. Dense
    inputs give a dense sum in the reference's association; row_sparse (float32) inputs a row_sparse
    sum; a mix a dense one. out may be the first input itself."""
    def f(*arrays, **kwargs):
        out = kwargs.pop('out', None)
        kwargs.setdefault('num_args', len(arrays))
        return _invoke(name, list(arrays), out=out, **kwargs)
    f.__name__ = name
    return f


add_n = _sum_op('add_n')
ElementWiseSum = _sum_op('ElementWiseSum')
_Sparse.add_n = staticmethod(_sum_op('_sparse_add_n'))
preloaded_multi_sgd_update = _op('preloaded_multi_sgd_update')
preloaded_multi_sgd_mom_update = _op('preloaded_multi_sgd_mom_update')
preloaded_multi_mp_sgd_update = _op('preloaded_multi_mp_sgd_update')
preloaded_multi_mp_sgd_mom_update = _op('preloaded_multi_mp_sgd_mom_update')
lamb_update_phase1 = _op('lamb_update_phase1')
lamb_update_phase2 = _op('lamb_update_phase2')
mp_lamb_update_phase1 = _op('mp_lamb_update_phase1')
mp_lamb_update_phase2 = _op('mp_lamb_update_phase2')
sqrt = _op('sqrt')
# the arithmetic of the reference's Adamax, Nadam and AdaDelta optimizers (GPU arrays of one shape;
# no broadcasting): maximum(lhs, rhs) of two arrays, abs(data), clip(data, a_min, a_max)
maximum = _op('broadcast_maximum')
abs = _op('abs')  # noqa: A001  (mx.nd.abs, as the reference names it)


def clip(data, a_min, a_max, out=None):
    return _invoke('clip', [data], out=out, a_min=a_min, a_max=a_max)


# the two operators the dense-gradient branches of the reference's AdaGrad and GroupAdaGrad add:
# square(data) on every dtype, and the mean over the last axis of a float array of rank 2 or more
# (axis=-1 or its positive index; any other axis is refused)
square = _op('square')


def mean(data, axis=None, keepdims=False, exclude=False, out=None):
    return _invoke('mean', [data], out=out, axis=axis, keepdims=keepdims, exclude=exclude)


def norm(data, out=None):
    """L2 norm of the whole array as a (1,) float32 array (mx.nd.norm with its defaults, the form
    the LAMB optimizer uses: optimizer.py:1304-1305, 1314-1315)."""
    return _invoke('sqrt', [multi_sum_sq(data, num_arrays=1)], out=out)


class _Internal(object):
    _adamw_update = staticmethod(_op('_adamw_update'))
    _mp_adamw_update = staticmethod(_op('_mp_adamw_update'))
    _multi_adamw_update = staticmethod(_op('_multi_adamw_update'))
    _multi_mp_adamw_update = staticmethod(_op('_multi_mp_adamw_update'))
    _multi_lamb_update = staticmethod(_op('_multi_lamb_update'))
    _multi_mp_lamb_update = staticmethod(_op('_multi_mp_lamb_update'))


_internal = _Internal()


def _flatten_list(nested_list):
    return [item for sublist in nested_list for item in sublist]


class _Contrib(object):
    """python/mxnet/ndarray/contrib.py:557-680: argument marshalling of the AdamW / LAMB operators
    (rescale_grad travels as an NDArray so that a dynamic loss scale never forces a host sync)."""

    @staticmethod
    def _rescale(rescale_grad, like):
        if isinstance(rescale_grad, NDArray):
            return rescale_grad
        return full((1,), rescale_grad, ctx=like.context)

    @staticmethod
    def adamw_update(weight, grad, mean, var, rescale_grad, lr, eta, beta1=0.9, beta2=0.999,
                     epsilon=1e-8, wd=0, clip_gradient=-1, out=None, **kwargs):
        rs = _Contrib._rescale(rescale_grad, weight)
        return _internal._adamw_update(weight, grad, mean, var, rs, out=out, lr=lr, eta=eta,
                                       beta1=beta1, beta2=beta2, epsilon=epsilon, wd=wd,
                                       clip_gradient=clip_gradient, **kwargs)

    @staticmethod
    def mp_adamw_update(weight, grad, mean, var, weight32, rescale_grad, lr, eta, beta1=0.9,
                        beta2=0.999, epsilon=1e-8, wd=0, clip_gradient=-1, out=None, **kwargs):
        rs = _Contrib._rescale(rescale_grad, weight32)
        return _internal._mp_adamw_update(weight, grad, mean, var, weight32, rs, out=out, lr=lr,
                                          eta=eta, beta1=beta1, beta2=beta2, epsilon=epsilon, wd=wd,
                                          clip_gradient=clip_gradient, **kwargs)

    @staticmethod
    def multi_adamw_update(weights, grads, mean, var, rescale_grad, lrs, wds, etas, out=None,
                           size=0, **kwargs):
        if not size:
            size = len(weights)
        rs = _Contrib._rescale(rescale_grad, weights[0])
        temp_list = _flatten_list(zip(weights, grads, mean, var)) + [rs]
        return _internal._multi_adamw_update(*temp_list, out=out, num_weights=size, lrs=lrs,
                                             wds=wds, etas=etas, **kwargs)

    @staticmethod
    def multi_mp_adamw_update(weights, grads, mean, var, weights32, rescale_grad, lrs, wds, etas,
                              out=None, size=0, **kwargs):
        if not size:
            size = len(weights)
        rs = _Contrib._rescale(rescale_grad, weights32[0])
        temp_list = _flatten_list(zip(weights, grads, mean, var, weights32)) + [rs]
        return _internal._multi_mp_adamw_update(*temp_list, out=out, num_weights=size, lrs=lrs,
                                                wds=wds, etas=etas, **kwargs)

    @staticmethod
    def multi_lamb_update(weights, grads, mean, var, step_count, lrs, wds, out=None,
                          num_tensors=0, **kwargs):
        if not num_tensors:
            num_tensors = len(weights)
        temp_list = _flatten_list(zip(weights, grads, mean, var))
        return _internal._multi_lamb_update(*temp_list, out=out, num_tensors=num_tensors,
                                            step_count=step_count, learning_rates=lrs, wds=wds,
                                            **kwargs)

    @staticmethod
    def multi_mp_lamb_update(weights, grads, mean, var, weights32, step_count, lrs, wds, out=None,
                             num_tensors=0, **kwargs):
        if not num_tensors:
            num_tensors = len(weights)
        temp_list = _flatten_list(zip(weights, grads, mean, var, weights32))
        return _internal._multi_mp_lamb_update(*temp_list, out=out, num_tensors=num_tensors,
                                               step_count=step_count, learning_rates=lrs, wds=wds,
                                               **kwargs)

    # GroupAdaGrad's lazy row update (float32, out must be the weight): (row_sparse, row_sparse,
    # row_sparse) or (dense, row_sparse, dense), history of shape (rows, 1); no wd parameter
    group_adagrad_update = staticmethod(_op('_contrib_group_adagrad_update'))

    @staticmethod
    def multi_scale(*arrays, scalar):
        """x *= float32(scalar) in place for every array (float32, dense or row_sparse, one GPU) in
        one launch per 200 arrays: the bulk form of amp.unscale's `g[:] *= scale`. The scalar is
        parsed as `_mul_scalar` parses its own in the reference (std::stod, then rounded to float)."""
        _invoke('_b200kv_multi_scale', list(arrays), num_arrays=len(arrays), scalar=scalar)


contrib = _Contrib()


class _Random(object):
    """mx.nd.random: the samplers of mx.random (random.py), and the _like operators, which the
    reference's op module places here"""
    _NAMES = ('uniform', 'normal', 'randn', 'exponential', 'gamma', 'randint',
              'uniform_like', 'normal_like', 'exponential_like', 'gamma_like')

    def __getattr__(self, name):
        if name not in _Random._NAMES:
            raise AttributeError("mx.nd.random has no attribute '%s'" % name)
        from . import random as _random
        return getattr(_random, name)


random = _Random()
