"""Pull anchors (csrc/kvstore.h, DevState): after a pushpull the key's value lives in the caller's
pull target and the store's own copy is neither written nor read. Every case runs with anchors on and
with B200KV_PULL_ANCHOR=0 and is compared bit for bit with both that run and the CPU oracle
(LocalKVStoreModel): anchors change where the value lives, never what it is."""
import gc

import numpy as np
import pytest

import bench
import kvoracle as K
from compat import mxnet_optimizer as mxopt   # the reference's optimizer front-end, mirrored (test infrastructure)

pytestmark = pytest.mark.gpu
SHAPES = [(64, 3, 7, 7), (64,), (3,), (128, 64, 3, 3), (1000, 512), (1000,)]
SGD = dict(learning_rate=0.1, momentum=0.9, wd=1e-4, rescale_grad=1.0 / 256)


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def eq(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


class Run(object):
    """A store on GPU 0 and its oracle model with the same keys, weights and SGD-momentum optimizer."""

    def __init__(self, mx, shapes=SHAPES, seed=7):
        self.mx, self.shapes = mx, shapes
        self.rng = np.random.default_rng(seed)
        self.keys = list(range(len(shapes)))
        self.kv = mx.kv.create('device')
        self.model = K.LocalKVStoreModel('device')
        w0 = [self.rnd(s) for s in shapes]
        self.kv.init(self.keys, [mx.nd.array(w, mx.gpu(0)) for w in w0])
        for k in self.keys:
            self.model.init(k, w0[k])
        self.set_sgd(SGD)

    def rnd(self, s):
        return self.rng.uniform(-1, 1, s).astype(np.float32)

    def set_sgd(self, kw):
        self.kv.set_optimizer(self.mx.optimizer.SGD(**kw))
        m = dict(kw)
        m['lr'] = m.pop('learning_rate')
        self.model.set_optimizer('sgd', **m)

    def grads(self):
        g = [self.rnd(s) for s in self.shapes]
        return g, [self.mx.nd.array(a, self.mx.gpu(0)) for a in g]

    def outs(self):
        return [self.mx.nd.empty(s, self.mx.gpu(0)) for s in self.shapes]

    def step(self, outs, keys=None):
        """one pushpull of fresh gradients into `outs`, mirrored in the model"""
        keys = self.keys if keys is None else keys
        g, gd = self.grads()
        self.kv.pushpull(keys, [gd[k] for k in keys], out=[outs[k] for k in keys])
        for k in keys:
            self.model.push(k, g[k])

    def check_store(self):
        """the stored values, pulled into fresh arrays, against the model"""
        fresh = self.outs()
        self.kv.pull(self.keys, out=fresh)
        got = [o.asnumpy() for o in fresh]
        for k in self.keys:
            assert eq(got[k], self.model.pull(k)), k
        return got


def both(monkeypatch, fn):
    """fn() with anchors on and off: identical results"""
    monkeypatch.setenv('B200KV_PULL_ANCHOR', '1')
    on = fn()
    monkeypatch.setenv('B200KV_PULL_ANCHOR', '0')
    off = fn()
    assert len(on) == len(off)
    for i, (a, b) in enumerate(zip(on, off)):
        assert eq(a, b), i
    return on


@pytest.mark.parametrize("workload,steps", [("resnet50_sgd", 5), ("bert_adam", 3)])
def test_flagship_sets_bit_exact(mx, monkeypatch, workload, steps):
    """bench.py's workloads through its own setup: the weights after `steps` grouped pushpulls"""
    shapes = bench.WORKLOADS[workload]["shapes"]()
    sizes = [int(np.prod(s)) for s in shapes]
    keys = list(range(len(shapes)))
    w0, g0 = bench.flat_set(bench.weight_seed(), sizes), bench.flat_set(bench.grad_seed(0), sizes)

    def run():
        kv = mx.kv.create('device')
        kv.init(keys, [mx.nd.array(w0[k].reshape(shapes[k]), mx.gpu(0)) for k in keys])
        kv.set_optimizer(bench.make_optimizer(mx, workload, 1))
        grads = [mx.nd.array(g0[k].reshape(shapes[k]), mx.gpu(0)) for k in keys]
        outs = [mx.nd.empty(s, mx.gpu(0)) for s in shapes]
        for _ in range(steps):
            kv.pushpull(keys, grads, out=outs)
        return [o.asnumpy() for o in outs]
    got = both(monkeypatch, run)
    want = bench.oracle_expected(workload, 1, steps)
    assert bench.compare_sets(got, want, exact=True)["ok"]


def test_push_only_after_anchored_pushpull(mx, monkeypatch):
    """a push that pulls nothing: the caller's array keeps what it last pulled, the next pull is new"""
    def run():
        r = Run(mx)
        outs = r.outs()
        for _ in range(2):
            r.step(outs)
        before = [o.asnumpy() for o in outs]
        g, gd = r.grads()
        r.kv.push(r.keys, gd)
        for k in r.keys:
            r.model.push(k, g[k])
        after = [o.asnumpy() for o in outs]
        for k in r.keys:
            assert eq(after[k], before[k]), k
        r.kv.pull(r.keys, out=outs)
        got = [o.asnumpy() for o in outs]
        for k in r.keys:
            assert eq(got[k], r.model.pull(k)), k
        r.step(outs)
        return [o.asnumpy() for o in outs] + r.check_store()
    both(monkeypatch, run)


def test_library_writes_to_the_anchor(mx, monkeypatch):
    """out[:] = 0, copyto and an operator's out= on anchored arrays leave the stored values alone"""
    def run():
        r = Run(mx)
        outs = r.outs()
        for _ in range(2):
            r.step(outs)
        outs[0][:] = 0
        mx.nd.array(r.rnd(SHAPES[4]), mx.gpu(0)).copyto(outs[4])
        outs[3] += 1.0                                   # _plus_scalar, out= the anchor
        res = [outs[0].asnumpy(), outs[3].asnumpy(), outs[4].asnumpy()]
        assert not res[0].any()
        res += r.check_store()
        r.kv.pull(r.keys, out=outs)
        for k in r.keys:
            assert eq(outs[k].asnumpy(), r.model.pull(k)), k
        outs[1][:] = 5
        r.step(outs)
        return res + [o.asnumpy() for o in outs] + r.check_store()
    both(monkeypatch, run)


def test_raw_exports_written_from_torch(mx, monkeypatch):
    """memory handed out through DLPack or MXNDArrayGetData and written by torch"""
    import ctypes
    import torch

    def run():
        r = Run(mx)
        outs = r.outs()
        for _ in range(2):
            r.step(outs)
        t = mx.nd.to_torch(outs[4])
        t.fill_(3.0)
        p = ctypes.c_void_p()
        mx.base.check_call(mx.base._LIB.MXNDArrayGetData(outs[3].handle, ctypes.byref(p)))
        torch.cuda.synchronize()
        store = r.check_store()
        r.step(outs)
        torch.cuda.synchronize()
        return store + [o.asnumpy() for o in outs] + r.check_store()
    both(monkeypatch, run)


def test_aliasing_targets(mx, monkeypatch):
    """out=grad in place, one array as the target of two keys, targets that are slices of one buffer
    (disjoint, then overlapping): none of them may take another key's value"""
    shapes = [(1000, 512), (1000, 512), (64,), (64,)]

    def run():
        r = Run(mx, shapes)
        res = []
        # in place: the gradient arrays receive the new weights
        for _ in range(2):
            g, gd = r.grads()
            r.kv.pushpull(r.keys, gd, out=gd)
            for k in r.keys:
                r.model.push(k, g[k])
            res += [a.asnumpy() for a in gd]
        res += r.check_store()
        # keys 2 and 3 share one target: only the stored values are compared
        shared = mx.nd.empty((64,), mx.gpu(0))
        outs = r.outs()
        for _ in range(2):
            r.step(outs[:2] + [shared, shared])
        res += r.check_store()
        # keys 0 and 1 into two halves of one buffer
        buf = mx.nd.empty((2000, 512), mx.gpu(0))
        for _ in range(2):
            r.step([buf[0:1000], buf[1000:2000]] + outs[2:])
        whole = buf.asnumpy()
        assert eq(whole[:1000], r.model.pull(0)) and eq(whole[1000:], r.model.pull(1))
        res += [whole] + r.check_store()
        # overlapping halves: the stored values only
        for _ in range(2):
            r.step([buf[0:1000], buf[500:1500]] + outs[2:])
        return res + r.check_store()
    both(monkeypatch, run)


def test_store_side_changes(mx, monkeypatch):
    """a pull into a second array, the anchored targets freed by the caller, optimizer-state
    checkpoints, set_optimizer between steps, a row_sparse push to an anchored dense key and the
    per-key calls of gluon's Trainer"""
    import os
    import tempfile

    def run():
        r = Run(mx)
        outs = r.outs()
        for _ in range(2):
            r.step(outs)
        second = r.outs()
        r.kv.pull(r.keys, out=second)
        res = [o.asnumpy() for o in second]
        for k in r.keys:
            assert eq(res[k], r.model.pull(k)), k
        # the caller drops the anchored arrays: the store keeps the values
        del outs
        gc.collect()
        res += r.check_store()
        outs = r.outs()
        r.step(outs)
        # checkpoint: save, step, load, step again from the saved state
        fname = os.path.join(tempfile.mkdtemp(), 'opt.states')
        r.kv.save_optimizer_states(fname)
        r.kv.load_optimizer_states(fname)
        r.step(outs)
        res += [o.asnumpy() for o in outs]
        # new hyper-parameters between steps
        kw = dict(SGD)
        kw['learning_rate'] = 0.05
        r.set_sgd(kw)
        r.step(outs)
        res += r.check_store()
        # Trainer: one pushpull per key with priority -i, queued and run as one bucket
        for _ in range(2):
            g, gd = r.grads()
            for k in r.keys:
                r.kv.pushpull(k, gd[k], out=outs[k], priority=-k)
                r.model.push(k, g[k])
            mx.nd.waitall()
            for k in r.keys:
                assert eq(outs[k].asnumpy(), r.model.pull(k)), k
        res += [o.asnumpy() for o in outs] + r.check_store()
        # a row_sparse gradient for the anchored dense key 4 updates the stored rows, not the
        # caller's array; then a pushpull of every key (compared between the two runs only)
        before = outs[4].asnumpy()
        rows = np.array([1, 7, 500], dtype=np.int64)
        r.kv.push(4, mx.nd.sparse.row_sparse_array((r.rnd((3, 512)), rows), shape=SHAPES[4], ctx=mx.gpu(0)))
        assert eq(outs[4].asnumpy(), before)
        fresh = r.outs()
        r.kv.pull(r.keys, out=fresh)
        res += [o.asnumpy() for o in fresh]
        g, gd = r.grads()
        r.kv.pushpull(r.keys, gd, out=outs)
        return res + [o.asnumpy() for o in outs]
    both(monkeypatch, run)


def test_updater_callback_after_anchors(mx, monkeypatch):
    """an optimizer run through the updater callback writes the stored value in place"""
    def run():
        r = Run(mx)
        outs = r.outs()
        for _ in range(2):
            r.step(outs)
        monkeypatch.setenv('B200KV_FUSED_OPTIMIZER', '0')
        try:
            r.kv.set_optimizer(mxopt.SGD(**SGD))
            g, gd = r.grads()
            r.kv.pushpull(r.keys, gd, out=outs)
        finally:
            monkeypatch.delenv('B200KV_FUSED_OPTIMIZER')
        fresh = r.outs()
        r.kv.pull(r.keys, out=fresh)
        return [o.asnumpy() for o in outs + fresh]
    both(monkeypatch, run)


def test_steady_state_is_one_launch_per_step(mx, monkeypatch):
    monkeypatch.setenv('B200KV_PULL_ANCHOR', '1')
    r = Run(mx)
    outs = r.outs()
    g, gd = r.grads()
    for _ in range(3):
        r.kv.pushpull(r.keys, gd, out=outs)
    mx.nd.waitall()
    mx.base.reset_kernel_launch_count()
    for _ in range(5):
        r.kv.pushpull(r.keys, gd, out=outs)
    mx.nd.waitall()
    assert mx.base.kernel_launch_count() == 5
    # gradient, weight and momentum read, weight and momentum written: 20 B per element
    assert mx.base.last_kernel_info()[1] == 20 * sum(int(np.prod(s)) for s in SHAPES)


def test_refused_call_leaves_the_stored_values(mx, monkeypatch):
    """a call refused while it is planned (here: a target of the wrong shape for the last key)
    changes no stored value -- neither on the call that would form the anchors nor on one that would
    end an anchor -- and the corrected retry continues from the stored values (oracle model)"""
    def run():
        r = Run(mx)
        outs = r.outs()
        wrong = mx.nd.empty((7,), mx.gpu(0))
        g, gd = r.grads()
        with pytest.raises(Exception):
            r.kv.pushpull(r.keys, gd, out=outs[:-1] + [wrong])
        res = r.check_store()
        r.step(outs)
        other = mx.nd.empty(SHAPES[0], mx.gpu(0))
        with pytest.raises(Exception):
            r.kv.pushpull(r.keys, gd, out=[other] + outs[1:-1] + [wrong])
        res += r.check_store()
        for _ in range(2):
            r.step(outs)
        return res + [o.asnumpy() for o in outs] + r.check_store()
    both(monkeypatch, run)


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_16bit_key_refused_without_master_weights(mx, monkeypatch, dtype):
    """SGD on 16-bit keys without multi_precision is refused; after the fix the store continues from
    the initial weights, exactly as a store that never saw the refused call"""
    shapes = [(1000, 512), (64,)]
    keys = [0, 1]
    rng = np.random.default_rng(3)
    w0 = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]
    g0 = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]
    kw = dict(learning_rate=0.1, momentum=0.9, wd=1e-4)

    def run(refuse_first):
        kv = mx.kv.create('device')
        kv.init(keys, [mx.nd.array(w, mx.gpu(0), dtype) for w in w0])
        grads = [mx.nd.array(g, mx.gpu(0), dtype) for g in g0]
        outs = [mx.nd.zeros(s, mx.gpu(0), dtype) for s in shapes]
        if refuse_first:
            kv.set_optimizer(mx.optimizer.SGD(**kw))
            with pytest.raises(Exception):
                kv.pushpull(keys, grads, out=outs)
            fresh = [mx.nd.empty(s, mx.gpu(0), dtype) for s in shapes]
            kv.pull(keys, out=fresh)
            for k in keys:
                assert eq(fresh[k].asnumpy(), mx.nd.array(w0[k], mx.gpu(0), dtype).asnumpy()), k
        kv.set_optimizer(mx.optimizer.SGD(multi_precision=True, **kw))
        for _ in range(3):
            kv.pushpull(keys, grads, out=outs)
        fresh = [mx.nd.empty(s, mx.gpu(0), dtype) for s in shapes]
        kv.pull(keys, out=fresh)
        return [o.asnumpy() for o in outs + fresh]
    want = run(False)
    got = both(monkeypatch, lambda: run(True))
    for i, (a, b) in enumerate(zip(got, want)):
        assert eq(a, b), i


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_16bit_keys_anchor_without_optimizer(mx, monkeypatch, dtype):
    """16-bit keys without an optimizer (the stored value is the merged gradient) anchor: pushpull,
    push only, pull, pushpull; each stored value equals the gradient pushed last"""
    shapes = [(1000, 512), (64,), (3,)]
    keys = list(range(len(shapes)))

    def run():
        rng = np.random.default_rng(5)
        kv = mx.kv.create('device')
        kv.init(keys, [mx.nd.array(rng.uniform(-1, 1, s), mx.gpu(0), dtype) for s in shapes])
        outs = [mx.nd.empty(s, mx.gpu(0), dtype) for s in shapes]
        res = []

        def grads():
            return [mx.nd.array(rng.uniform(-1, 1, s), mx.gpu(0), dtype) for s in shapes]
        for _ in range(2):
            gd = grads()
            kv.pushpull(keys, gd, out=outs)
            for k in keys:
                assert eq(outs[k].asnumpy(), gd[k].asnumpy()), k
        before = [o.asnumpy() for o in outs]
        gd = grads()
        kv.push(keys, gd)
        for k in keys:
            assert eq(outs[k].asnumpy(), before[k]), k
        kv.pull(keys, out=outs)
        for k in keys:
            assert eq(outs[k].asnumpy(), gd[k].asnumpy()), k
        res += [o.asnumpy() for o in outs]
        gd = grads()
        kv.pushpull(keys, gd, out=outs)
        fresh = [mx.nd.empty(s, mx.gpu(0), dtype) for s in shapes]
        kv.pull(keys, out=fresh)
        for k in keys:
            assert eq(fresh[k].asnumpy(), gd[k].asnumpy()), k
        return res + [o.asnumpy() for o in outs + fresh]
    both(monkeypatch, run)


def test_switch_off_ends_live_anchors(mx, monkeypatch):
    """B200KV_PULL_ANCHOR=0 on a store that has anchored: its anchors end at the next call it plans
    (the launch then moves 24 B per SGD-momentum element again instead of 20), and the values go on
    unchanged (oracle model)"""
    monkeypatch.setenv('B200KV_PULL_ANCHOR', '1')
    r = Run(mx)
    n = sum(int(np.prod(s)) for s in SHAPES)
    outs = r.outs()
    for _ in range(2):
        r.step(outs)
    assert mx.base.last_kernel_info()[1] == 20 * n
    monkeypatch.setenv('B200KV_PULL_ANCHOR', '0')
    r.step(r.outs())                   # a new call signature: planned, so the anchors end
    r.step(outs)
    assert mx.base.last_kernel_info()[1] == 24 * n
    for k in r.keys:
        assert eq(outs[k].asnumpy(), r.model.pull(k)), k
    r.check_store()
