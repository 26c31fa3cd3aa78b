"""Row_sparse values pushed to dense keys, without a GPU: the checker model's
(oracle/kvoracle_sparse_grad.py) storage-type transitions, its lazy and standard (dense, row_sparse) updates against the reference's compiled
kernels and this oracle's restatement, and the broadcast kernel compiles for sm_90a without spills."""
import os
import re
import subprocess

import numpy as np
import pytest

import kvoracle as K
import kvoracle_sparse_grad as SG

live = pytest.mark.skipif(K.ref() is None or not K.ref().has_sparse(),
                          reason="needs oracle/_ref/libmxref.so")


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def rsp(rng, shape, nnr):
    idx = np.sort(rng.choice(shape[0], nnr, replace=False))
    return SG.Rsp(idx, rng.uniform(-1, 1, (nnr,) + shape[1:]).astype(np.float32), shape)


def test_model_storage_type_transitions():
    rng = np.random.default_rng(0)
    shape = (20, 3)
    m = SG.DenseKeySparseGradModel('device')
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    m.init(0, w0)
    assert m.stype[0] == 'default' and eq(m.pull(0), w0)
    a, b = SG.Rsp([1, 4], np.ones((2, 3)), shape), SG.Rsp([4, 7], np.full((2, 3), 2.0), shape)
    m.push(0, [a, b])                               # no updater: local = merged
    assert m.stype[0] == 'row_sparse'
    idx, val = m.pull_rsp(0)
    assert np.array_equal(idx, [1, 4, 7]) and eq(val, np.array([[1] * 3, [3] * 3, [2] * 3], np.float32))
    d = m.pull(0)
    assert eq(d[[1, 4, 7]], val) and not np.delete(d, [1, 4, 7], axis=0).any()
    g = rng.uniform(-1, 1, shape).astype(np.float32)
    m.push(0, [g])                                  # a dense push makes the value dense again
    assert m.stype[0] == 'default' and eq(m.pull(0), g)
    m.set_optimizer('sgd', lr=0.1, momentum=0.9)
    m.push(0, [rsp(rng, shape, 5)])                 # with an optimizer the value stays dense
    assert m.stype[0] == 'default' and m.count[0] == 1 and m.state[0].shape == shape


def test_model_empty_push_without_updater():
    m = SG.DenseKeySparseGradModel('device')
    m.init(0, np.ones((6, 2), np.float32))
    m.push(0, [SG.Rsp([], np.zeros((0, 2)), (6, 2)), SG.Rsp([], np.zeros((0, 2)), (6, 2))])
    assert m.stype[0] == 'row_sparse' and m.pull_rsp(0)[0].size == 0 and not m.pull(0).any()


def _cases():
    out = []
    for kind in ('sgd', 'sgd_mom', 'adam'):
        for lazy in (True, False):
            for clip in (None, 0.3):
                out.append((kind, lazy, clip))
    return out


@live
@pytest.mark.parametrize("kind,lazy,clip", _cases())
def test_model_updates_match_reference_and_restatement(kind, lazy, clip):
    """three row_sparse pushes on random layouts; the model's weights equal a hand-driven run of
    the reference's kernels (SGDDnsRspKernel, SGDMomDnsRspDnsKernel, AdamDnsRspDnsKernel and the
    standard forms) and of this oracle's own restatement of them"""
    rng = np.random.default_rng(_cases().index((kind, lazy, clip)))
    shape = (97, 7)
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    m = SG.DenseKeySparseGradModel('device')
    m.init(0, w0)
    mom = 0.9 if kind == 'sgd_mom' else 0.0
    lr = 1e-2 if kind == 'adam' else 0.1
    m.set_optimizer('adam' if kind == 'adam' else 'sgd', lr=lr, momentum=mom, wd=1e-3, rescale_grad=0.5,
                    clip_gradient=clip, lazy_update=lazy)
    sp = K.scalar_param
    c = sp(clip) if clip else None
    for lib in (K.ref(), K.get_oracle()):
        w = w0.copy()
        s1, s2 = np.zeros_like(w), np.zeros_like(w)
        drive_model = lib is K.ref()   # the model runs once, beside the first library
        for t in range(1, 4):
            srcs = [rsp(np.random.default_rng(100 * t + i), shape, int(10 + 20 * i)) for i in range(3)]
            gi, gv = lib.rsp_reduce([s.idx for s in srcs], [s.val for s in srcs])
            if kind == 'sgd':
                (lib.sgd_rsp_update if lazy else lib.sgd_std_rsp_update)(w, gi, gv, sp(lr), sp(1e-3), sp(0.5), c)
            elif kind == 'sgd_mom':
                (lib.sgd_mom_rsp_update if lazy else lib.sgd_mom_std_rsp_update)(
                    w, s1, gi, gv, sp(lr), sp(mom), sp(1e-3), sp(0.5), c)
            else:
                (lib.adam_rsp_update if lazy else lib.adam_std_rsp_update)(
                    w, s1, s2, gi, gv, sp(K.adam_lr(lr, 0.9, 0.999, t)), sp(0.9), sp(0.999), sp(1e-8),
                    sp(1e-3), sp(0.5), c)
            if not drive_model:
                continue
            m.push(0, srcs)
            if lazy:
                cold = np.setdiff1d(np.arange(shape[0]), gi)
                assert eq(m.pull(0)[cold], (w0 if t == 1 else prev)[cold])
            prev = m.pull(0)
            assert eq(prev, w), (lib, t)
        assert eq(m.pull(0), w), lib


def test_broadcast_kernel_compiles_without_spills(tmp_path):
    """the three unit widths of rsp_broadcast_kernel (16, 4 and 1 bytes)"""
    from anand_mxnet_b200 import build as B
    src = os.path.join(B.CSRC, "rowsparse_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "r.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    blocks = re.split(r"Compiling entry function ", r.stderr)[1:]
    found = [re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", b).groups()
             for b in blocks if re.match(r"'\w*rsp_broadcast_kernel", b)]
    assert len(found) == 3, r.stderr[-4000:]
    assert all(f == ('0', '0', '0') for f in found), found
