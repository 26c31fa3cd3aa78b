"""The fixtures of the dense-weight, row_sparse-gradient forms of the NAG / Signum / RMSProp / FTML /
Ftrl operators, without a GPU: tests/golden/rsp_grad_update_ops.npz against the reference's own
compiled operators on the densified gradient (when oracle/_ref is built) and against the numpy
restatement (always), and tests/golden/updater_trajectories_rsp_grad.npz's operator log and, when
the reference is present, its trajectories."""
import os
import re
import subprocess

import numpy as np
import pytest

import golden_rsp_grad_update_ops as GR
import golden_update_ops as GU
import ref_python_rsp_grad_update as RRG


def _check(gold, name, out, states):
    assert GR.matches(gold, '%s|out' % name, out), (name, 'out')
    for i, s in enumerate(states):
        assert GR.matches(gold, '%s|s%d' % (name, i), s), (name, i)


def test_fixture_covers_every_case(golden):
    gold = golden("rsp_grad_update_ops")
    keys = {f.split('|')[0] for f in gold.files}
    assert keys == set(GR.CASES)
    ops = {c['op'] for c in GR.CASES.values()}
    assert ops == set(GR.OPS) and 'mp_nag_mom_update' not in ops
    for op in GR.OPS:
        cs = [c for c in GR.CASES.values() if c['op'] == op]
        assert {c['rows'] for c in cs} == set(GR.ROWSETS)
        assert {c['shape'] for c in cs} == set(GR.SHAPES.values())
        assert any(c['distinct_out'] for c in cs)


@pytest.mark.parametrize("name", sorted(GR.CASES))
def test_fixture_vs_restatement(golden, name):
    _check(golden("rsp_grad_update_ops"), name, *GR.run_restated(GR.CASES[name]))


@pytest.mark.skipif(GU.ref() is None, reason="needs oracle/_ref/libmxref_update.so (the reference's sources)")
@pytest.mark.parametrize("name", sorted(GR.CASES))
def test_fixture_vs_reference_live(golden, name):
    _check(golden("rsp_grad_update_ops"), name, *GR.run_ref(GR.CASES[name]))


def test_densify_is_a_zero_fill_and_row_copy():
    vals = np.array([[1.5, -2.0], [3.0, 4.0]], np.float32)
    d = GR.densify((4, 2), [1, 3], vals)
    assert np.array_equal(d, [[0, 0], [1.5, -2], [0, 0], [3, 4]])
    assert not np.signbit(d[[0, 2]]).any(), "absent rows are +0.0f"
    assert np.array_equal(GR.densify((3,), np.zeros(0, np.int64), np.zeros(0, np.float32)), np.zeros(3))


def test_trajectory_operator_log(golden):
    """each case's optimizer called the operator expected, with a dense weight and dense states and
    the row_sparse gradient, once per key and step"""
    gold = golden("updater_trajectories_rsp_grad")
    cases = RRG.trajectory_cases()
    assert set(cases) == set(RRG.EXPECTED_CALL)
    for name, case in cases.items():
        log = gold['%s|log' % name].tolist()
        assert log == [RRG.EXPECTED_CALL[name]] * (len(case['grads']) * len(case['shapes'])), name


@pytest.mark.skipif(not RRG.available(), reason="needs the reference's sources and oracle/_ref")
def test_trajectories_vs_reference_live(golden):
    gold = golden("updater_trajectories_rsp_grad")
    import ref_python as RP
    with RRG.reference_python_rsp_grad_update() as (opt, _):
        for name, case in RRG.trajectory_cases().items():
            del RRG.OPLOG[:]
            for step, (ws, sts) in enumerate(RRG.run_trajectory(opt, case, RP.NDArray)):
                for k, (w, st) in enumerate(zip(ws, sts)):
                    assert GR.matches(gold, "%s_step%d_w%d" % (name, step, k), w), (name, step, k)
                    for i, s in enumerate(st):
                        assert GR.matches(gold, "%s_step%d_w%d_s%d" % (name, step, k, i), s), (name, step, k, i)
            assert RRG.OPLOG == gold['%s|log' % name].tolist()


def test_ptxas_no_spills_rsp_grad_and_std_sgd_adam(tmp_path):
    """the ten row_sparse-gradient kernels (seven operators and the standard sgd_update, sgd_mom_update
    and adam_update forms) compile for sm_90a with no spills and no stack frame"""
    from anand_mxnet_b200 import build as B
    src = os.path.join(B.CSRC, "update_rsp_grad_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "u.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(frames) == 10, r.stderr[-4000:]
    assert all(f == ('0', '0', '0') for f in frames), frames
