"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/*.npz from the REFERENCE's own code.

Run in the build container (where /root/reference exists):

    make -C oracle ref && python oracle/gen_golden.py

Every array under tests/golden/ is an input or an output of oracle/_ref/libmxref.so, i.e. of the
reference's headers compiled in place (oracle/ref_harness.cc lists the functions). The fixtures are
small (a few hundred KB) and travel with the repository, so the GPU box -- which has no
/root/reference -- can still check both the oracle and the CUDA path against reference outputs.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import kvoracle as K  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")


def u(rng, *shape):
    return rng.uniform(-1, 1, shape).astype(np.float32)


def rsp_cases():
    """row_sparse reduce / retain / unique inputs (own RNG stream, shared with tests/test_oracle.py):
    duplicates across sources, an empty source, a source holding every row, one source only,
    unsorted + repeated pull ids, ids the source does not hold."""
    rng = np.random.default_rng(0xB200 + 5)
    rows, rl = 211, 19
    red = {}
    layouts = {"dup4": [60, 60, 60, 60], "empty_mid": [40, 0, 25], "full_plus": [rows, 30], "single": [50],
               "nine": [12] * 9, "all_empty": [0, 0]}
    for tag, counts in layouts.items():
        idxs = [np.sort(rng.choice(rows, c, replace=False)).astype(np.int64) for c in counts]
        vals = [u(rng, c, rl) for c in counts]
        red[tag] = (idxs, vals)
    src_i = np.sort(rng.choice(rows, 80, replace=False)).astype(np.int64)
    src_v = u(rng, 80, rl)
    dense_v = u(rng, rows, rl)
    ret = {
        "sorted_unique": (src_i, src_v, np.unique(rng.integers(0, rows, 70)).astype(np.int64), False),
        "unsorted_dup": (src_i, src_v, rng.integers(0, rows, 90).astype(np.int64), False),
        "none_present": (src_i, src_v, np.setdiff1d(np.arange(rows), src_i)[:33].astype(np.int64), False),
        "empty_src": (np.zeros(0, np.int64), np.zeros((0, rl), np.float32),
                      np.arange(0, rows, 7, dtype=np.int64), False),
        "dense_src": (np.arange(rows, dtype=np.int64), dense_v, rng.integers(0, rows, 64).astype(np.int64), True),
    }
    uniq = {"random": rng.integers(0, rows, 500).astype(np.int64), "one": np.array([7], np.int64),
            "same": np.full(33, 5, np.int64), "descending": np.arange(100, 0, -1, dtype=np.int64)}
    return red, ret, uniq


def gen_rsp(r):
    """the reference's own ElementwiseSumRsp / sparse_retain kernels / UniqueImpl (oracle/ref_sparse.cc)"""
    red, ret, uniq = rsp_cases()
    d = {}
    for tag, (idxs, vals) in red.items():
        for nt in (1, 4):
            oi, ov = r.rsp_reduce(idxs, vals, nthreads=nt)
            if nt == 1:
                d["reduce_%s_idx" % tag], d["reduce_%s_val" % tag] = oi, ov
            else:       # the reference's threading splits the union rows: same bits for any thread count
                assert np.array_equal(oi, d["reduce_%s_idx" % tag])
                assert np.array_equal(ov.view(np.uint32), d["reduce_%s_val" % tag].view(np.uint32))
    for tag, (si, sv, ids, dense) in ret.items():
        oi, ov = r.sparse_retain(si, sv, ids, src_dense_rows=dense)
        d["retain_%s_idx" % tag], d["retain_%s_val" % tag] = oi, ov
        if tag == "sorted_unique":      # the reference's row-block kernel agrees with its per-id kernel
            bi, bv = r.sparse_retain(si, sv, ids, row_block=True)
            assert np.array_equal(bi, oi) and np.array_equal(bv.view(np.uint32), ov.view(np.uint32))
    for tag, ids in uniq.items():
        d["unique_%s" % tag] = r.unique(ids)
    np.savez_compressed(os.path.join(GOLD, "rowsparse_reduce_retain.npz"), **d)


def updater_cases():
    """optimizer trajectories on the store's dense path: (index, gradient, weight) per key per step
    through the reference's own Updater (oracle/ref_python.py). 'model' = the same hyper-parameters in
    kvoracle.LocalKVStoreModel's vocabulary; 'lr_at' = the learning rate the scheduler yields at each
    step (restated; the live test proves the restatement)."""
    rng = np.random.default_rng(0xB200 + 6)
    shapes = [(4, 4), (100, 100), (1027,), (3,), (7001,)]

    def plan(steps):
        return dict(shapes=shapes, w0=[u(rng, *s) for s in shapes],
                    grads=[[u(rng, *s) for s in shapes] for _ in range(steps)])
    cases = {}
    cases['sgd_mom'] = dict(plan(4), opt=('SGD', dict(learning_rate=0.1, momentum=0.9, wd=1e-4, rescale_grad=1 / 256)),
                            model=dict(kind='sgd', lr=0.1, momentum=0.9, wd=1e-4, rescale_grad=1 / 256),
                            lr_mult={1: 0.5, 3: 2.0}, wd_mult={0: 0.0})
    cases['sgd_plain_clip'] = dict(plan(3), opt=('SGD', dict(learning_rate=0.05, wd=1e-3, clip_gradient=0.02,
                                                              rescale_grad=0.125)),
                                   model=dict(kind='sgd', lr=0.05, momentum=0.0, wd=1e-3, clip_gradient=0.02,
                                              rescale_grad=0.125))
    cases['sgd_factor_sched'] = dict(plan(5), opt=('SGD', dict(momentum=0.9, wd=1e-4)),
                                     sched=('FactorScheduler', dict(step=2, factor=0.5, base_lr=0.2)),
                                     lr_at=[0.2, 0.2, 0.1, 0.1, 0.05],
                                     model=dict(kind='sgd', lr=0.2, momentum=0.9, wd=1e-4))
    cases['adam'] = dict(plan(6), opt=('Adam', dict(learning_rate=1e-3, wd=0.01)),
                         model=dict(kind='adam', lr=1e-3, wd=0.01), lr_mult={2: 0.1})
    cases['adam_clip_betas'] = dict(plan(4), opt=('Adam', dict(learning_rate=3e-4, beta1=0.8, beta2=0.98,
                                                                epsilon=1e-6, clip_gradient=0.5, rescale_grad=0.5)),
                                    model=dict(kind='adam', lr=3e-4, beta1=0.8, beta2=0.98, epsilon=1e-6,
                                               clip_gradient=0.5, rescale_grad=0.5))
    cases['test'] = dict(plan(3), opt=('Test', dict(rescale_grad=2.0)), model=dict(kind='test', rescale_grad=2.0))
    # fp16 weights and gradients with fp32 master weights (multi_mp_sgd_mom_update); no numpy model
    p16 = plan(4)
    p16['w0'] = [w.astype(np.float16) for w in p16['w0']]
    p16['grads'] = [[g.astype(np.float16) for g in gs] for gs in p16['grads']]
    cases['sgd_mp_fp16'] = dict(p16, opt=('SGD', dict(learning_rate=0.1, momentum=0.9, wd=1e-4, rescale_grad=1 / 64,
                                                      multi_precision=True)), model=None)
    # update_on_kvstore=False: Trainer hands the Updater every parameter of a device at once; LARS and
    # LAMB aggregate them into multi-tensor operator calls (4 tensors per call)
    names = ['conv0_weight', 'conv0_bias', 'bn0_gamma', 'bn0_beta', 'fc_weight', 'fc_bias', 'emb_weight']
    lshapes = [(8, 3, 3, 3), (8,), (8,), (8,), (10, 72), (10,), (37, 5)]

    def lplan(steps):
        return dict(shapes=lshapes, names=names, mode='list', model=None, w0=[u(rng, *s) for s in lshapes],
                    grads=[[u(rng, *s) for s in lshapes] for _ in range(steps)])
    cases['lars_list'] = dict(lplan(3), opt=('LARS', dict(momentum=0.9, wd=1e-4, eta=0.02, eps=1e-6, rescale_grad=1 / 32)),
                              sched=('FactorScheduler', dict(step=2, factor=0.5, base_lr=0.4)), lr_at=[0.4, 0.4, 0.2])
    cases['lamb_list'] = dict(lplan(3), opt=('LAMB', dict(learning_rate=2e-3, wd=0.01, rescale_grad=0.25)))
    # a rescale_grad whose dmlc::stof and std::stod-then-float parses differ: Test's `grad * rescale_grad`
    # is _mul_scalar, which takes std::stod (appended last so that no earlier case's draws move)
    cases['test_rescale_stod'] = dict(plan(3), opt=('Test', dict(rescale_grad=1.2345e-05)),
                                      model=dict(kind='test', rescale_grad=1.2345e-05))
    return cases


def run_updater_case(opt_mod, sched_mod, case):
    """one case through an optimizer front-end module (the reference's, or a mirror of it)"""
    import ref_python as RP
    name, kw = case['opt']
    kw = dict(kw)
    if 'sched' in case:
        sname, skw = case['sched']
        kw['lr_scheduler'] = getattr(sched_mod, sname)(**skw)
    if 'names' in case:
        kw['param_idx2name'] = dict(enumerate(case['names']))
    opt = getattr(opt_mod, name)(**kw)
    if case.get('lr_mult'):
        opt.set_lr_mult(case['lr_mult'])
    if case.get('wd_mult'):
        opt.set_wd_mult(case['wd_mult'])
    upd = opt_mod.get_updater(opt)          # what KVStore.set_optimizer installs (kvstore.py:450-453)
    ws = [RP.NDArray(w.copy()) for w in case['w0']]
    for gs in case['grads']:
        if case.get('mode') == 'list':              # Trainer._update: updater(indices, grads, weights)
            upd(list(range(len(ws))), [RP.NDArray(g.copy()) for g in gs], ws)
            continue
        for k, g in enumerate(gs):
            upd(k, RP.NDArray(g.copy()), ws[k])   # the store's callback: updater(key, merged, stored)
    return [w.a for w in ws]


def gen_updater():
    import ref_python as RP
    d = {}
    with RP.reference_python() as (opt, sched):
        for name, case in updater_cases().items():
            for k, w in enumerate(run_updater_case(opt, sched, case)):
                d["%s_w%d" % (name, k)] = w
    np.savez_compressed(os.path.join(GOLD, "updater_trajectories.npz"), **d)


def main():
    r = K.ref()
    assert r is not None, "build oracle/_ref first: make -C oracle ref"
    os.makedirs(GOLD, exist_ok=True)
    if "--rsp-only" in sys.argv:       # add this fixture without rewriting the others' zip timestamps
        gen_rsp(r)
        return
    if "--updater-only" in sys.argv:
        gen_updater()
        return
    gen_rsp(r)
    gen_updater()
    rng = np.random.default_rng(0xB200)

    # ---- dense reduce, CommCPU association, 1..9 sources + a >BIGARRAY_BOUND threaded case ----
    d = {}
    for n in (1, 2, 3, 4, 5, 6, 7, 8, 9):
        srcs = [u(rng, 1031) for _ in range(n)]
        d["n%d_src" % n] = np.stack(srcs)
        d["n%d_out" % n] = r.reduce(srcs)
    np.savez_compressed(os.path.join(GOLD, "reduce_local.npz"), **d)

    # ---- optimizers ----
    d = {}
    n = 2053
    hp = dict(lr=0.1, wd=1e-4, rescale=1.0 / 256, momentum=0.9)
    for tag, clip in (("noclip", None), ("clip", 0.002)):
        w, g, m = u(rng, n), u(rng, n), u(rng, n)
        d["sgd_%s_in" % tag] = np.stack([w, g])
        d["sgd_%s_out" % tag] = r.sgd_update(w.copy(), g, hp["lr"], hp["wd"], hp["rescale"], clip)
        w2, m2 = w.copy(), m.copy()
        r.sgd_mom_update(w2, g, m2, hp["lr"], hp["momentum"], hp["wd"], hp["rescale"], clip)
        d["sgdmom_%s_in" % tag] = np.stack([w, g, m])
        d["sgdmom_%s_out" % tag] = np.stack([w2, m2])
        w2, m2 = w.copy(), m.copy()
        r.multi_sgd_update([w2], [g], [m2], [hp["lr"]], [hp["wd"]], hp["momentum"], hp["rescale"],
                           clip)
        d["multisgdmom_%s_out" % tag] = np.stack([w2, m2])
        w2 = w.copy()
        r.multi_sgd_update([w2], [g], None, [hp["lr"]], [hp["wd"]], 0.0, hp["rescale"], clip)
        d["multisgd_%s_out" % tag] = w2
        v = np.abs(u(rng, n))
        w2, m2, v2 = w.copy(), m.copy(), v.copy()
        # five Adam steps with the python-side bias-corrected lr (optimizer.py:1617-1620)
        outs = []
        aclip = None if clip is None else 0.5
        sp = lambda x: r.dmlc_stof(repr(float(x)))  # noqa: E731  the reference's own scalar parse
        for t in range(1, 6):
            lr_t = sp(K.adam_lr(1e-3, 0.9, 0.999, t))
            r.adam_update(w2, g, m2, v2, lr_t, sp(0.9), sp(0.999), sp(1e-8), sp(0.01), 1.0, aclip)
            outs.append(np.stack([w2.copy(), m2.copy(), v2.copy()]))
        d["adam_%s_in" % tag] = np.stack([w, g, m, v])
        d["adam_%s_out" % tag] = np.stack(outs)
        # fp16 mixed precision
        w32 = u(rng, n)
        w16 = w32.astype(np.float16).view(np.uint16)
        g16 = u(rng, n).astype(np.float16).view(np.uint16)
        a16, a32, am = w16.copy(), w32.copy(), m.copy()
        r.multi_mp_sgd_update_f16([a16], [a32], [g16], [am], [hp["lr"]], [hp["wd"]],
                                  hp["momentum"], hp["rescale"], clip)
        d["mp_%s_in16" % tag] = np.stack([w16, g16])
        d["mp_%s_in32" % tag] = np.stack([w32, m])
        d["mpmom_%s_out16" % tag] = a16
        d["mpmom_%s_out32" % tag] = np.stack([a32, am])
        a16, a32 = w16.copy(), w32.copy()
        r.mp_sgd_update_f16(a16, a32, g16, hp["lr"], hp["wd"], hp["rescale"], clip)
        d["mpsgd_%s_out16" % tag] = a16
        d["mpsgd_%s_out32" % tag] = a32
    d["hp"] = np.array([hp["lr"], hp["wd"], hp["rescale"], hp["momentum"]], dtype=np.float64)
    np.savez_compressed(os.path.join(GOLD, "optimizers.npz"), **d)

    # ---- lazy row_sparse updates ----
    d = {}
    R, L, nnr = 200, 24, 40
    for tag, clip in (("noclip", None), ("clip", 0.3)):
        w, m = u(rng, R, L), u(rng, R, L)
        v = np.abs(u(rng, R, L))
        gi = np.sort(rng.choice(R, nnr, replace=False)).astype(np.int64)
        gv = u(rng, nnr, L)
        d["rsp_%s_in" % tag] = np.stack([w, m, v])
        d["rsp_%s_gidx" % tag] = gi
        d["rsp_%s_gval" % tag] = gv
        d["rsp_sgd_%s_out" % tag] = r.sgd_rsp_update(w.copy(), gi, gv, 0.1, 1e-3, 0.5, clip)
        w2, m2 = w.copy(), m.copy()
        r.sgd_mom_rsp_update(w2, m2, gi, gv, 0.1, 0.9, 1e-3, 0.5, clip)
        d["rsp_sgdmom_%s_out" % tag] = np.stack([w2, m2])
        w2, m2, v2 = w.copy(), m.copy(), v.copy()
        r.adam_rsp_update(w2, m2, v2, gi, gv, 1e-3, wd=0.01, clip=clip)
        d["rsp_adam_%s_out" % tag] = np.stack([w2, m2, v2])
    np.savez_compressed(os.path.join(GOLD, "rowsparse_updates.npz"), **d)

    # ---- standard (non-lazy) updates with a row_sparse gradient (8f-f3) ----
    d = {}
    rows, rl = 37, 24
    rng3 = np.random.default_rng(0xB200 + 3)       # own stream: the fixtures above / below stay as is
    for tag, clip in (("noclip", None), ("clip", 0.3)):
        w, m, v = u(rng3, rows, rl), u(rng3, rows, rl), np.abs(u(rng3, rows, rl))
        gi = np.sort(rng3.choice(rows, 11, replace=False)).astype(np.int64)
        gi[0], gi[-1] = 0, rows - 1               # first and last row present
        gi = np.unique(gi)
        gv = u(rng3, gi.size, rl)
        d["std_%s_in" % tag] = np.stack([w, m, v])
        d["std_%s_gidx" % tag], d["std_%s_gval" % tag] = gi, gv
        d["std_sgd_%s_out" % tag] = r.sgd_std_rsp_update(w.copy(), gi, gv, 0.1, 1e-3, 0.5, clip)
        w2, m2 = w.copy(), m.copy()
        r.sgd_mom_std_rsp_update(w2, m2, gi, gv, 0.1, 0.9, 1e-3, 0.5, clip)
        d["std_sgdmom_%s_out" % tag] = np.stack([w2, m2])
        w2, m2, v2 = w.copy(), m.copy(), v.copy()
        r.adam_std_rsp_update(w2, m2, v2, gi, gv, 1e-3, wd=0.01, clip=clip)
        d["std_adam_%s_out" % tag] = np.stack([w2, m2, v2])
        # an all-zero gradient (no rows) still decays / moves every row
        e_i, e_v = np.zeros(0, np.int64), np.zeros((0, rl), np.float32)
        w2, m2 = w.copy(), m.copy()
        r.sgd_mom_std_rsp_update(w2, m2, e_i, e_v, 0.1, 0.9, 1e-3, 0.5, clip)
        d["std_sgdmom_%s_empty_out" % tag] = np.stack([w2, m2])
    np.savez_compressed(os.path.join(GOLD, "rowsparse_std_updates.npz"), **d)

    # ---- NDArray::Save bytes (8f-f4: what pickled optimizer states / mx.nd.save files hold) ----
    rng4 = np.random.default_rng(0xB200 + 4)
    d = {}
    a = u(rng4, 3, 5)
    d["dense_f32_gpu0_in"] = a
    d["dense_f32_gpu0_bytes"] = np.frombuffer(r.ndarray_save_bytes(a.shape, a, ctx=(2, 0)), np.uint8)
    h = u(rng4, 7).astype(np.float16)
    d["dense_f16_cpu_in"] = h
    d["dense_f16_cpu_bytes"] = np.frombuffer(r.ndarray_save_bytes(h.shape, h, ctx=(1, 0)), np.uint8)
    i64 = rng4.integers(-5, 5, (2, 2, 2)).astype(np.int64)
    d["dense_i64_cpu_in"] = i64
    d["dense_i64_cpu_bytes"] = np.frombuffer(r.ndarray_save_bytes(i64.shape, i64, ctx=(1, 0)), np.uint8)
    rows, idx = u(rng4, 2, 4), np.array([1, 4], np.int64)
    d["rsp_f32_gpu0_rows"], d["rsp_f32_gpu0_idx"] = rows, idx
    d["rsp_f32_gpu0_bytes"] = np.frombuffer(r.ndarray_save_bytes((6, 4), rows, ctx=(2, 0), idx=idx), np.uint8)
    np.savez_compressed(os.path.join(GOLD, "ndarray_raw_bytes.npz"), **d)

    # ---- 2-bit compression ----
    g = u(rng, 1003)
    res = np.zeros_like(g)
    comp1 = r.quantize_2bit(g, res, 0.5)
    res1 = res.copy()
    comp2 = r.quantize_2bit(g, res, 0.5)
    np.savez_compressed(os.path.join(GOLD, "twobit.npz"), grad=g, comp1=comp1, res1=res1,
                        comp2=comp2, res2=res.copy(), deq1=r.dequantize_2bit(comp1, g.size, 0.5))

    # ---- scalar plumbing: python repr -> dmlc::stof, on values a training run produces ----
    import random
    random.seed(0xB200)
    vals = [0.1, 0.01, 1e-4, 1e-5, 2.5e-5, 1.2345e-5, 0.9, 0.999, 1e-8, 1 / 256, 1 / 2048, 5.0, 2.5]
    for _ in range(3000):
        k = random.random()
        if k < 0.3:
            vals.append(random.uniform(0, 1))
        elif k < 0.6:
            vals.append(10 ** random.uniform(-9, 3))
        elif k < 0.8:
            vals.append(0.1 * 0.97 ** random.randint(0, 300))
        else:
            vals.append(K.adam_lr(1e-3, 0.9, 0.999, random.randint(1, 5000)))
    vals = np.array(vals, dtype=np.float64)
    parsed = np.array([r.dmlc_stof(repr(float(v))) for v in vals], dtype=np.float32)
    np.savez_compressed(os.path.join(GOLD, "scalar_parse.npz"), values=vals, parsed=parsed)
    print("wrote", sorted(os.listdir(GOLD)))


if __name__ == "__main__":
    main()
