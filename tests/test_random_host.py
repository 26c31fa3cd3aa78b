"""The GPU sampler without a GPU: the oracle recipe builds, the bookkeeping restatement
(oracle/golden_random.py: LaunchRNG's nthread / step, the runs each state draws, the copies' seeds and
the round robin) matches hand-worked cases, `_random_normal` is registered in random_ops.cc, its
kernels compile for sm_90a with no spills and no stack frame, and the seeding C entry points carry
the reference header's signatures."""
import ctypes
import os
import re
import subprocess

import pytest

import golden_random as GR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "anand_mxnet_b200", "csrc")
N = 64 * 32768


@pytest.mark.skipif(not os.path.isfile("/root/reference/src/common/random_generator.cu"),
                    reason="needs the reference's sources")
def test_recipe_builds():
    GR.build()
    assert os.path.exists(GR.LIB)


@pytest.mark.parametrize("n,nthread,step,last", [
    (1, 1, 1, (0, 0, 1)),
    (63, 1, 63, (0, 0, 63)),
    (64, 1, 64, (0, 0, 64)),
    (65, 2, 33, (1, 33, 65)),
    (N - 1, 32768, 64, (32767, 32767 * 64, N - 1)),
    (N, 32768, 64, (32767, 32767 * 64, N)),
    # 65 per state: states 32264.. (the last 504) draw nothing
    (N + 1, 32768, 65, (32263, 32263 * 65, N + 1)),
])
def test_launch_bookkeeping(n, nthread, step, last):
    assert GR.launch_shape(n) == (nthread, step)
    r = GR.runs(n)
    assert r[0][1] == 0 and r[-1] == last
    assert sum(e - b for _, b, e in r) == n
    assert all(r[i][2] == r[i + 1][1] for i in range(len(r) - 1))


def test_empty_launch():
    assert GR.launch_shape(0) == (0, 0) and GR.runs(0) == []


def test_seeds_and_round_robin():
    # SeedWithDeviceID: dev + i*16 + seed*127; Seed: i*16 + seed*127, mod 2^32
    assert [GR.copy_seed(i, 0, 0) for i in range(4)] == [0, 16, 32, 48]
    assert [GR.copy_seed(i, 3, 1) for i in range(4)] == [382, 398, 414, 430]
    assert [GR.copy_seed(i, 3) for i in range(4)] == [381, 397, 413, 429]
    assert GR.copy_seed(0, -1, 0) == (2 ** 32 - 127)
    ptr, taken = 0, []
    for _ in range(9):
        c, ptr = GR.next_copy(ptr)
        taken.append(c)
    assert taken == [1, 2, 3, 0, 1, 2, 3, 0, 1]


def test_operator_registered():
    import anand_mxnet_b200 as mx
    h = ctypes.c_void_p()
    assert mx.base._LIB.NNGetOpHandle(b"_random_normal", ctypes.byref(h)) == 0 and h.value
    assert mx.nd.random.normal is mx.random.normal
    with open(os.path.join(CSRC, "random_ops.cc")) as f:
        rows = re.findall(r'\{"([^"]+)",\s*(\w+),', f.read())
    assert rows == [("_random_normal", "RandomNormal")]


def test_refused_without_gpu_work():
    """a CPU context is refused before any generator exists; a seed must be an int"""
    import anand_mxnet_b200 as mx
    with pytest.raises(mx.MXNetError, match="GPU only"):
        mx.random.normal(0, 1, shape=(4,), ctx=mx.cpu(0))
    with pytest.raises(ValueError, match="seed_state must be int"):
        mx.random.seed(1.5)


def test_ptxas_no_spills(tmp_path):
    """normal_kernel for four dtypes x two store orders, and the seed kernel"""
    from anand_mxnet_b200 import build as B
    src = os.path.join(B.CSRC, "random_kernels.cu")
    assert "-fmad=true" in B.flags_for("random_kernels.cu")
    r = subprocess.run([B._nvcc()] + B.flags_for("random_kernels.cu") +
                       ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "r.o")],
                       capture_output=True, text=True, env=B._env())
    assert r.returncode == 0, r.stderr[-4000:]
    blocks = re.split(r"Compiling entry function ", r.stderr)[1:]
    found = [(b.split("'")[1],) + re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, "
                                            r"(\d+) bytes spill loads", b).groups()
             for b in blocks if re.match(r"'\w*(normal_kernel|rand_seed_kernel)", b)]
    assert len(found) == 9, r.stderr[-4000:]
    assert all(f == s == l == '0' for _, f, s, l in found), found


REF_C_API = "/root/reference/include/mxnet/c_api.h"
# include/mxnet/c_api.h:254 and :261, as (return type, parameter types)
SEED_SIGNATURES = {"MXRandomSeed": ("int", ["int"]), "MXRandomSeedContext": ("int", ["int", "int", "int"])}


def _signatures(path, macro):
    """{name: (return type, [parameter types])} of the MXRandomSeed* declarations of a C header"""
    with open(path) as f:
        txt = re.sub(r"/\*.*?\*/", " ", f.read(), flags=re.S)
    out = {}
    for ret, name, args in re.findall(macro + r"\s+(\w+)\s+(MXRandomSeed\w*)\s*\(([^)]*)\)\s*;", txt):
        out[name] = (ret, [a.split()[0] for a in args.split(",")])
    return out


def test_c_signatures_match_reference():
    """include/b200kv_random_api.h (included by b200kv_c_api.h) declares the reference's seeding
    functions type for type, and the library exports them"""
    mine = _signatures(os.path.join(ROOT, "include", "b200kv_random_api.h"), "B200KV_DLL")
    assert mine == SEED_SIGNATURES
    if os.path.isfile(REF_C_API):
        assert _signatures(REF_C_API, "MXNET_DLL") == SEED_SIGNATURES
    with open(os.path.join(ROOT, "include", "b200kv_c_api.h")) as f:
        assert '#include "b200kv_random_api.h"' in f.read()
    from anand_mxnet_b200 import build as B
    lib = ctypes.CDLL(B.LIB)
    for name in list(SEED_SIGNATURES) + ["B200KVRandomStates", "B200KVRandomNormalInto"]:
        assert hasattr(lib, name), name
