"""The imperative-operator table, without a GPU. Every operator is one row of its family's table
(csrc/ops.cc, multi_ops.cc, update_ops.cc) naming its handler; NNGetOpHandle resolves exactly those
names. Handlers never look at their operator's name to choose what to do, and the parameter and
output helpers they share are defined once."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "anand_mxnet_b200", "csrc")
FAMILIES = ("ops.cc", "multi_ops.cc", "update_ops.cc")
HELPERS = FAMILIES + ("ops.h", "op_params.h")

OPERATORS = [
    # ops.cc
    "sgd_update", "sgd_mom_update", "adam_update", "mp_sgd_update", "mp_sgd_mom_update",
    "multi_sgd_update", "multi_sgd_mom_update", "multi_mp_sgd_update", "multi_mp_sgd_mom_update",
    "preloaded_multi_sgd_update", "preloaded_multi_sgd_mom_update", "preloaded_multi_mp_sgd_update",
    "preloaded_multi_mp_sgd_mom_update", "_copyto", "_plus", "elemwise_add", "_minus", "elemwise_sub",
    "_mul", "elemwise_mul", "_plus_scalar", "_mul_scalar", "sqrt", "_set_value", "_full", "zeros_like",
    "_sparse_zeros_like", "cast", "Cast",
    # multi_ops.cc
    "multi_sum_sq", "all_finite", "multi_all_finite", "_b200kv_clip_global_norm", "_b200kv_multi_scale",
    "reset_arrays", "multi_lars", "_adamw_update", "_mp_adamw_update", "_multi_adamw_update",
    "_multi_mp_adamw_update", "lamb_update_phase1", "mp_lamb_update_phase1", "lamb_update_phase2",
    "mp_lamb_update_phase2", "_multi_lamb_update", "_multi_mp_lamb_update",
    # update_ops.cc
    "nag_mom_update", "mp_nag_mom_update", "signsgd_update", "signum_update", "rmsprop_update",
    "rmspropalex_update", "ftml_update", "ftrl_update", "_sparse_ftrl_update", "_sparse_adagrad_update",
    "_contrib_group_adagrad_update",
]
NEAR_MISSES = ["multi_", "multi_sgd", "preloaded_multi_sgd", "_sparse_sgd_update", "cast ", "Sgd_update",
               "", "preloaded_", "_multi_", "Convolution"]


def source(name):
    """the file with its comments blanked (string literals kept: they are what is checked)"""
    with open(os.path.join(CSRC, name)) as f:
        src = f.read()
    pat = re.compile(r'"(?:\\.|[^"\\\n])*"|//[^\n]*|/\*.*?\*/', re.S)
    return pat.sub(lambda m: m.group(0) if m.group(0).startswith('"') else " ", src)


def test_every_operator_resolves_and_nothing_else():
    import anand_mxnet_b200 as mx
    lib = mx.base._LIB
    assert len(OPERATORS) == len(set(OPERATORS)) == 57
    h = ctypes.c_void_p()
    handles = set()
    for name in OPERATORS:
        assert lib.NNGetOpHandle(name.encode(), ctypes.byref(h)) == 0, name
        handles.add(h.value)
    assert len(handles) == len(OPERATORS)
    for name in NEAR_MISSES:
        assert lib.NNGetOpHandle(name.encode(), ctypes.byref(h)) == -1, repr(name)
        assert b"not registered" in lib.MXGetLastError(), repr(name)


def definitions(name):
    """function definitions (not declarations) of `name` at namespace scope in the helper files"""
    pat = re.compile(r"^[A-Za-z][\w:<>,*& ]*?\b%s\([^;{}]*\)\s*(?:const\s*)?\{" % name, re.M)
    return [f for f in HELPERS for _ in pat.finditer(source(f))]


def test_handlers_do_not_parse_names_and_helpers_are_defined_once():
    for f in FAMILIES:
        src = source(f)
        for pat in (r'\bn\s*[!=]=\s*"', r'\bname\s*[!=]=\s*"', r'\.find\("_', r'\.rfind\("', r'\bn\[0\]',
                    r'strn?cmp\('):
            found = [src.count("\n", 0, m.start()) + 1 for m in re.finditer(pat, src)]
            assert not found, "%s:%s matches %s" % (f, found, pat)
    for helper in ("Required", "OutOr", "InPlace", "RejectUnknownKeys"):
        assert len(definitions(helper)) == 1, (helper, definitions(helper))
    assert sum(source(f).count('"Cannot find argument') for f in HELPERS) == 1
    # one table row per operator, whichever file declares it
    rows = [n for f in FAMILIES for n in re.findall(r'\{"([^"]+)",\s*\w+,', source(f))]
    assert sorted(rows) == sorted(OPERATORS)
