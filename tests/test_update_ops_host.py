"""The NAG / Signum / RMSProp / FTML / Ftrl operators without a GPU: their names resolve, the numpy
restatement (oracle/golden_update_ops.py) equals tests/golden/update_ops.npz everywhere and the
reference's own operators live (fixture cases plus random layouts), the tests/compat mirror of the
five optimizer classes issues the reference classes' operator calls and reaches their weights, and
the kernels compile for sm_90a without spills."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import golden_update_ops as GU
import ref_python as RP
import ref_python_update as RPU

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
live = pytest.mark.skipif(GU.ref() is None, reason="needs oracle/_ref/libmxref_update.so")
live_py = pytest.mark.skipif(not RPU.available(), reason="needs /root/reference and oracle/_ref/ libraries")


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_update_operators_are_registered():
    import anand_mxnet_b200 as mx
    for name in GU.OPS:
        h = ctypes.c_void_p()
        assert mx.base._LIB.NNGetOpHandle(name.encode(), ctypes.byref(h)) == 0 and h.value, name
        assert callable(getattr(mx.nd, name)), name


def test_fixture_covers_every_case():
    g = np.load(os.path.join(ROOT, "tests", "golden", "update_ops.npz"))
    assert {k.split('|')[0] for k in g.files} == set(GU.CASES)
    assert {c['op'] for c in GU.CASES.values()} == set(GU.OPS)


def _check(g, name, case, out, states):
    for tag, a in [('out', out)] + [('s%d' % i, s) for i, s in enumerate(states)]:
        a = np.ascontiguousarray(a)
        if case['n'] <= GU.FULL_MAX:
            assert eq(a, g['%s|%s' % (name, tag)]), (name, tag)
        else:
            assert eq(a[:GU.HEAD], g['%s|%s|head' % (name, tag)]), (name, tag)
            assert eq(GU.digest(a), g['%s|%s|sha256' % (name, tag)]), (name, tag)


@pytest.mark.parametrize("name", sorted(GU.CASES))
def test_restatement_matches_golden(golden, name):
    case = GU.CASES[name]
    out, st = GU.run_restated(case)
    _check(golden("update_ops"), name, case, out, st)


@live
@pytest.mark.parametrize("name", sorted(n for n, c in GU.CASES.items() if c['dtype'] != 'bfloat16'))
def test_restatement_matches_live_reference(name):
    case = GU.CASES[name]
    ins = GU.inputs(case)
    o1, s1 = GU.run_ref(case, ins)
    o2, s2 = GU.run_restated(case, ins)
    assert eq(o1, o2) and all(eq(a, b) for a, b in zip(s1, s2)), name


@live
@pytest.mark.parametrize("seed", range(50))
def test_restatement_matches_live_reference_random(seed):
    """random operator, size, parameters (clip on / off, wd, rescale, the optional fields)"""
    rng = np.random.default_rng(seed)
    op = GU.OPS[seed % len(GU.OPS)]
    n = int(rng.choice([1, 2, 3, 5, 8, 17, 255, 1031]))
    params = dict(lr=float(rng.choice([0.1, 0.01, 1e-3, 0.37])), rescale_grad=float(rng.choice([1.0, 0.5, 1 / 96])))
    if rng.random() < 0.5:
        params['wd'] = float(rng.choice([1e-4, 0.01, 0.3]))
    if rng.random() < 0.5:
        params['clip_grad' if op == 'ftml_update' else 'clip_gradient'] = float(rng.choice([0.0, 0.05, 0.7]))
    extra = {'nag_mom_update': dict(momentum=0.9), 'mp_nag_mom_update': dict(momentum=0.5),
             'signum_update': dict(momentum=0.8, wd_lh=0.02), 'rmsprop_update': dict(gamma1=0.7, clip_weights=0.6),
             'rmspropalex_update': dict(gamma1=0.9, gamma2=0.7, epsilon=1e-6),
             'ftml_update': dict(t=int(rng.integers(1, 20)), beta1=0.5, epsilon=3.3e-07),
             'ftrl_update': dict(lamda1=0.05, beta=0.5)}.get(op, {})
    params.update({k: v for k, v in extra.items() if rng.random() < 0.7})
    if op == 'ftml_update':                     # t is required
        params['t'] = extra['t']
    case = dict(op=op, dtype='float16' if op == 'mp_nag_mom_update' else 'float32', n=n, params=params,
                distinct_out=bool(rng.random() < 0.3))
    ins = GU.inputs(case)
    o1, s1 = GU.run_ref(case, ins)
    o2, s2 = GU.run_restated(case, ins)
    assert eq(o1, o2) and all(eq(a, b) for a, b in zip(s1, s2)), (op, n, params)


def test_ftml_epsilon_goes_through_stod():
    """FTML's epsilon is a double field (dmlc::stod), then cast to float"""
    for s in ['1e-08', '1e-07', '3.3e-07', '0.001', '1e-10', '2.5']:
        assert GU.stod(s) == float(np.float64(GU.stod(s)))
        assert abs(GU.stod(s) - float(s)) <= 2e-16 * abs(float(s))


# ------------------------------------------------------------------ the tests/compat mirror
def _mirror():
    """tests/compat/mxnet_optimizer_update.py (and the base class module it builds on) with their
    operator imports replaced by the harness's, so both front-ends run the reference's operators"""
    from compat import mxnet_optimizer as B
    from compat import mxnet_optimizer_update as M
    saved = [(m, dict(m.__dict__)) for m in (B, M)]
    for m in (B, M):
        m.__dict__.update(RP.op_table())
        m.__dict__.update(RPU.op_table())
    return M, saved


@live_py
@pytest.mark.parametrize("name", sorted(RPU.trajectory_cases()))
def test_compat_mirror_vs_reference(golden, name):
    case = RPU.trajectory_cases()[name]
    with RPU.reference_python_update() as (opt, _):
        RP.LOG[:] = []
        want = RPU.run_trajectory(opt, case)
        want_log = list(RP.LOG)
        M, saved = _mirror()
        try:
            RP.LOG[:] = []
            got = RPU.run_trajectory(M, case)
            got_log = list(RP.LOG)
        finally:
            for m, d in saved:
                m.__dict__.clear()
                m.__dict__.update(d)
    assert got_log == want_log and len(want_log) > 0
    gold = golden("updater_trajectories_ext")
    for step, (ws_g, ws_w) in enumerate(zip(got, want)):
        for k, (a, b) in enumerate(zip(ws_g, ws_w)):
            assert eq(a, b), (name, step, k)
            assert eq(b, gold["%s_step%d_w%d" % (name, step, k)]), (name, step, k)


def test_ptxas_no_spills(tmp_path):
    from anand_mxnet_b200 import build as B
    src = os.path.join(B.CSRC, "update_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o",
                                                     str(tmp_path / "u.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) == 9, r.stderr[-4000:]          # 7 fp32 operators + mp_nag for fp16 and bf16
    assert all(s == ('0', '0') for s in spills), spills
