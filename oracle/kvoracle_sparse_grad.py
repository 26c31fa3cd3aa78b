"""kvoracle_sparse_grad -- TEST INFRASTRUCTURE: LocalKVStoreModel (kvoracle.py) extended to row_sparse
values pushed to dense keys, the store step gluon.Trainer runs for a dense weight with a sparse
gradient (Embedding(sparse_grad=True); python/mxnet/gluon/trainer.py:141-160, 193-226, 375-388).

Row_sparse values (``Rsp``) are merged by ReduceRowSparse (comm.h:478-501, ElementwiseSumRsp,
ndarray_function.cc:155-176). Without an optimizer the stored value becomes the merged row_sparse
array (kvstore_local.h:237-243: ``local = merged.Copy(local.ctx())``), so the value's storage type
follows the last push; a dense push makes it dense again. With one, the stored dense weight is updated
by the (dense weight, row_sparse grad) kernels the reference's operators dispatch to
(src/operator/optimizer_op-inl.h): lazy SGDDnsRspKernel :453-475, SGDMomDnsRspDnsKernel :749-773,
AdamDnsRspDnsKernel :1350-1380, and with lazy_update=False the standard forms that update every row
(SGDStdUpdateDnsRspDnsImpl :505-528 and the momentum / Adam counterparts). They run from
oracle/_ref/libmxref.so when it is built, else from kvoracle's restatement of them. Hyper-parameters
reach them as scalar parameters (sgd_update / sgd_mom_update / adam_update: python/mxnet/optimizer/
optimizer.py:603-659, 1610-1629); the update counts and states are the ones dense pushes use.
"""
import numpy as np

import kvoracle as K


class Rsp(object):
    """A row_sparse value: ascending unique ids and their rows, in a table of `shape`."""

    def __init__(self, idx, val, shape=None):
        self.idx = np.ascontiguousarray(idx, dtype=np.int64)
        val = K._f32(val)
        self.val = val.reshape(self.idx.size, int(np.prod(val.shape[1:])))
        self.shape = shape


class DenseKeySparseGradModel(K.LocalKVStoreModel):
    """LocalKVStoreModel whose dense keys also take row_sparse values; ``stype[key]`` is the storage
    type of the key's current value."""

    def __init__(self, order="local"):
        super(DenseKeySparseGradModel, self).__init__(order)
        self.stype = {}
        self.lazy = True

    def init(self, key, value):
        super(DenseKeySparseGradModel, self).init(key, value)
        self.stype[key] = 'default'

    def set_optimizer(self, kind, lazy_update=True, **kw):
        super(DenseKeySparseGradModel, self).set_optimizer(kind, **kw)
        self.lazy = lazy_update

    def shape(self, key):
        return self.store[key].shape

    def _densify(self, key):
        if self.stype[key] == 'row_sparse':
            self.store[key] = self.pull(key)
            self.stype[key] = 'default'
        return self.store[key]

    def _kernels(self):
        r = K.ref()
        return r if r is not None and r.has_sparse() else self.o

    def push(self, key, values):
        values = values if isinstance(values, (list, tuple)) else [values]
        if isinstance(values[0], Rsp):
            return self._push_rsp(key, values)
        self._densify(key)
        super(DenseKeySparseGradModel, self).push(key, values)

    def _push_rsp(self, key, values):
        shape = self.shape(key)
        kern = self._kernels()
        gidx, gval = kern.rsp_reduce([v.idx for v in values], [v.val for v in values])
        if self.opt is None:
            self.store[key] = Rsp(gidx, gval, shape)
            self.stype[key] = 'row_sparse'
            return
        p = self.opt
        w = self._densify(key)
        w2 = w.reshape(shape[0], -1)
        gval = np.ascontiguousarray(gval.reshape(gidx.size, w2.shape[1]))
        self.count[key] = self.count.get(key, 0) + 1
        lr = p['lr'] * p['lr_mult'].get(key, 1.0)
        wd = p['wd'] * p['wd_mult'].get(key, 1.0)
        sp = K.scalar_param
        clip = sp(p['clip']) if p['clip'] else None
        if p['kind'] == 'sgd':
            if p['momentum'] != 0.0:
                mom = self.state.setdefault(key, np.zeros_like(w)).reshape(w2.shape)
                f = kern.sgd_mom_rsp_update if self.lazy else kern.sgd_mom_std_rsp_update
                f(w2, mom, gidx, gval, sp(lr), sp(p['momentum']) if p['momentum'] > 0 else 0.0, sp(wd),
                  sp(p['rescale']), clip)
            else:
                f = kern.sgd_rsp_update if self.lazy else kern.sgd_std_rsp_update
                f(w2, gidx, gval, sp(lr), sp(wd), sp(p['rescale']), clip)
        elif p['kind'] == 'adam':
            m, v = self.state.setdefault(key, (np.zeros_like(w), np.zeros_like(w)))
            lr_t = K.adam_lr(lr, p['beta1'], p['beta2'], self.count[key])
            f = kern.adam_rsp_update if self.lazy else kern.adam_std_rsp_update
            f(w2, m.reshape(w2.shape), v.reshape(w2.shape), gidx, gval, sp(lr_t), sp(p['beta1']),
              sp(p['beta2']), sp(p['eps']), sp(wd), sp(p['rescale']), clip)
        else:
            raise ValueError("row_sparse values take sgd or adam: %s" % p['kind'])

    def pull(self, key):
        """the stored value, dense: a row_sparse value is zeros plus its rows (CastStorageRspDnsImpl)"""
        v = self.store[key]
        if self.stype[key] == 'default':
            return v.copy()
        d = np.zeros(v.shape, np.float32)
        d.reshape(d.shape[0], -1)[v.idx] = v.val
        return d

    def pull_rsp(self, key):
        """(ids, rows) of a row_sparse value, as a pull into a row_sparse out with
        ignore_sparse=False returns them (CopyFromToRspImpl, ndarray.cc:1076-1093)"""
        assert self.stype[key] == 'row_sparse'
        v = self.store[key]
        return v.idx.copy(), v.val.reshape((v.idx.size,) + tuple(v.shape[1:])).copy()
