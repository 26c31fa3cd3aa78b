"""add_n / ElementWiseSum without a GPU: the four names resolve, the numpy restatement
(oracle/golden_add_n.py) equals tests/golden/add_n.npz and the reference's own code live, the
operator table declares the family in sum_ops.cc, and add_n_kernel compiles for sm_90a with no
spills and no stack frame in every dtype."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import golden_add_n as GAN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "anand_mxnet_b200", "csrc")
live = pytest.mark.skipif(GAN.ref_dense() is None or GAN.ref_rsp() is None,
                          reason="needs oracle/_ref/libmxref_add_n.so and libmxref.so")
NAMES = ["add_n", "ElementWiseSum", "_sparse_add_n", "_sparse_ElementWiseSum"]


def test_operators_are_registered():
    import anand_mxnet_b200 as mx
    h = ctypes.c_void_p()
    handles = set()
    for name in NAMES:
        assert mx.base._LIB.NNGetOpHandle(name.encode(), ctypes.byref(h)) == 0 and h.value, name
        handles.add(h.value)
    assert len(handles) == 4
    assert callable(mx.nd.add_n) and callable(mx.nd.ElementWiseSum) and callable(mx.nd.sparse.add_n)


def test_table_rows_and_handler():
    """one row per name in sum_ops.cc, all on one handler that never looks at the name"""
    with open(os.path.join(CSRC, "sum_ops.cc")) as f:
        src = f.read()
    rows = re.findall(r'\{"([^"]+)",\s*(\w+),', src)
    assert sorted(n for n, _ in rows) == sorted(NAMES)
    assert {h for _, h in rows} == {"AddN"}
    code = re.sub(r'"(?:\\.|[^"\\\n])*"|//[^\n]*', '""', src)
    for pat in (r'\bname\s*[!=]=', r'\bn\s*[!=]=\s*"', r'strn?cmp\(', r'\.find\('):
        assert not re.search(pat, code), pat
    assert src.count('"Cannot find argument') == 0   # the wording comes from RejectUnknownKeys


def test_fixture_covers_every_case():
    g = np.load(os.path.join(ROOT, "tests", "golden", "add_n.npz"))
    assert set(g.files) == {k for n in GAN.CASES for k in GAN.key_of(n)}
    dense = [c for c in GAN.CASES.values() if set(c['stypes']) == {'default'}]
    for dt in GAN.DTYPES:
        assert sorted(len(c['stypes']) for c in dense if c['dtype'] == dt and not c.get('zeros')) == GAN.COUNTS


def same(name, got, g):
    case = GAN.CASES[name]
    if isinstance(got, tuple):
        return np.array_equal(got[0], g[name + '_idx']) and GAN.same_bits(got[1], g[name + '_val'])
    return GAN.same_bits(got, g[name], case['dtype'])


@pytest.mark.parametrize("name", sorted(GAN.CASES))
def test_restatement_matches_golden(golden, name):
    case = GAN.CASES[name]
    assert same(name, GAN.restate(case, GAN.inputs(case, name)), golden("add_n")), name


LIVE = sorted(n for n, c in GAN.CASES.items() if c['dtype'] in GAN.MSHADOW_FLAG)


@live
@pytest.mark.parametrize("name", LIVE)
def test_live_reference_matches_golden(golden, name):
    case = GAN.CASES[name]
    assert same(name, GAN.ref(case, GAN.inputs(case, name)), golden("add_n")), name


@live
def test_live_reference_neg_zero_rows():
    """the > 4 form leaves a -0.0 of an absent row as it is; the <= 4 fallback adds +0.0 to it"""
    for name, want in (('mix_gt4_dense_first', 0x80000000), ('mix_gt4_rsp_first', 0),
                       ('mix_le4_dr', 0), ('mix_le4_drd', 0)):
        case = GAN.CASES[name]
        out = GAN.ref(case, GAN.inputs(case, name)).view(np.uint32)
        assert out[6, 3] == want, name


def test_ptxas_no_spills(tmp_path):
    """add_n_kernel for float16, bfloat16, float32, float64, uint8, int8, int32 and int64"""
    from anand_mxnet_b200 import build as B
    src = os.path.join(B.CSRC, "sum_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "s.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    blocks = re.split(r"Compiling entry function ", r.stderr)[1:]
    found = [(b.split("'")[1],) + re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, "
                                            r"(\d+) bytes spill loads", b).groups()
             for b in blocks if re.match(r"'\w*add_n_kernel", b)]
    assert len(found) == 8, r.stderr[-4000:]
    assert all(f == s == l == '0' for _, f, s, l in found), found
