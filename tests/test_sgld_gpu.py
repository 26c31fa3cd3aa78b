"""The reference's SGLD optimizer (tests/compat/mxnet_optimizer_sgld.py) on the GPU, five steps, bit
for bit: through a local updater and through the 'device' store's updater callback
(kv.set_optimizer), with rescale_grad, clip_gradient and wd, on the ResNet-50 and BERT-base float32
parameter sets and one float16 set with multi_precision=True. The expected weights are the same
steps restated: the NDArray arithmetic from the existing oracle (golden_ndarray_ops,
golden_arith_ops) and the noise from the reference's own GPU sampler (golden_random), drawn from the
generator copies in the reference's round robin, one call per key and step in key order."""
import math
import zlib

import numpy as np
import pytest

import golden_arith_ops as GA
import golden_ndarray_ops as G
import golden_random as GR
import kvoracle as K

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(GR.ref() is None, reason="needs oracle/_ref/libmxref_random_gpu.so")]
STEPS = 5
OPT = dict(learning_rate=0.01, rescale_grad=1.0 / 64, clip_gradient=0.005, wd=1e-4)
SEED = 17
NP = {'float16': np.float16, 'float32': np.float32}


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def shapes(name):
    import bench
    if name == 'resnet50':
        return bench.resnet50_shapes()
    if name == 'bert':
        return bench.bert_base_shapes()
    return [(64, 3, 7, 7), (1000,), (3,), (257, 129)]


def weights0(name, dt):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    return [rng.uniform(-1, 1, s).astype(NP[dt]) for s in shapes(name)]


def gradients(name, dt, step):
    """|g| in [0.25, 1]: halving one for the store's two pushed values is exact in float16 too"""
    rng = np.random.default_rng(zlib.crc32(('%s|%d' % (name, step)).encode()))
    return [(rng.uniform(0.25, 1, s) * rng.choice([-1.0, 1.0], s)).astype(NP[dt]) for s in shapes(name)]


class Restated(object):
    """the compat class's steps in numpy: the weights after each step"""

    def __init__(self, w0, dt, mp):
        self.ref = GR.RefGenerators(0, SEED)
        self.dt, self.mp = dt, mp
        self.cdt = 'float32' if mp else dt
        self.ws = [G.cast(w, dt, 'float32') if mp else w.copy() for w in w0]

    def step(self, gs):
        lr, c, wd, cdt = OPT['learning_rate'], OPT['clip_gradient'], OPT['wd'], self.cdt
        scale = float(K.dmlc_stof(str(math.sqrt(lr))))
        for k, g in enumerate(gs):
            g = G.cast(g, self.dt, 'float32') if self.mp else g
            g = G.binary_scalar('mul', g, repr(float(OPT['rescale_grad'])), cdt)
            g = GA.clip(g, repr(-float(c)), repr(float(c)), cdt)
            t = G.binary('plus', g, G.binary_scalar('mul', self.ws[k], repr(float(wd)), cdt), cdt)
            t = G.binary_scalar('mul', t, repr(-lr / 2), cdt)
            w = G.binary('plus', self.ws[k], t, cdt)
            noise = self.ref.normal(w.size, 0.0, scale, cdt).reshape(w.shape)
            self.ws[k] = G.binary('plus', w, noise, cdt)
        return [G.cast(w, 'float32', self.dt) if self.mp else w for w in self.ws]


def _opt(mp):
    from compat import mxnet_optimizer_sgld as mxopt
    return mxopt.SGLD(multi_precision=mp, **OPT)


def _eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


CASES = [('resnet50', 'float32', False), ('bert', 'float32', False), ('small', 'float16', True)]


@pytest.mark.parametrize("name,dt,mp", CASES)
def test_local_updater(mx, name, dt, mp):
    from compat import mxnet_optimizer_sgld as mxopt
    w0 = weights0(name, dt)
    model = Restated(w0, dt, mp)
    mx.random.seed(SEED)
    upd = mxopt.get_updater(_opt(mp))
    ws = [mx.nd.array(w, mx.gpu(0), dt) for w in w0]
    for step in range(STEPS):
        gs = gradients(name, dt, step)
        for k, g in enumerate(gs):
            upd(k, mx.nd.array(g, mx.gpu(0), dt), ws[k])
        want = model.step(gs)
        for k in range(len(ws)):
            assert _eq(ws[k].asnumpy(), want[k]), (name, step, k)


@pytest.mark.parametrize("name,dt,mp", CASES)
def test_store_callback(mx, name, dt, mp):
    w0 = weights0(name, dt)
    model = Restated(w0, dt, mp)
    keys = list(range(len(w0)))
    kv = mx.kv.create('device')
    for k in keys:
        kv.init(k, mx.nd.array(w0[k], mx.gpu(0), dt))
    mx.random.seed(SEED)
    kv.set_optimizer(_opt(mp))
    outs = [mx.nd.empty(w.shape, mx.gpu(0), dt) for w in w0]
    for step in range(STEPS):
        gs = gradients(name, dt, step)
        vals = [[mx.nd.array((g / g.dtype.type(2)).astype(g.dtype), mx.gpu(0), dt) for _ in range(2)] for g in gs]
        kv.pushpull(keys, vals, out=outs)
        want = model.step(gs)
        for k in keys:
            assert _eq(outs[k].asnumpy(), want[k]), (name, step, k)
