"""Builds libb200kv.so in-tree with nvcc for sm_90a (no torch dependency, static cudart).

    python -m anand_mxnet_b200.build [--force] [--verbose]

The .so lands next to this file (anand_mxnet_b200/libb200kv.so, git-ignored). nvcc cross-compiles
without a GPU.
"""
import concurrent.futures
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libb200kv.so")

NVCC_FLAGS = [
    "-std=c++17", "-O3", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    # bit-parity with the reference's CPU build: no fused multiply-add contraction, IEEE div/sqrt
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true",
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-Wall,-Wno-unused-function",
    "-I", os.path.join(ROOT, "include"), "-I", CSRC,
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libb200kv.so cannot be built")


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cc")))


def _newest_header():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".h")]
    hs += [os.path.join(ROOT, "include", h) for h in ("b200kv_c_api.h", "b200kv_random_api.h")]
    return max(os.path.getmtime(h) for h in hs)


def flags_for(src):
    """The reference's GPU sampler is built with nvcc's default contraction, and curand's Box-Muller
    arithmetic in its headers contracts with it: random_kernels.cu keeps -fmad=true to draw the same
    numbers. Every other file keeps the CPU reference's -fmad=false."""
    if src == "random_kernels.cu":
        return ["-fmad=true" if f == "-fmad=false" else f for f in NVCC_FLAGS]
    return NVCC_FLAGS


def _compile(nvcc, src, verbose):
    obj = os.path.join(OBJ, src + ".o")
    cmd = [nvcc] + flags_for(src) + (["-Xptxas", "-v"] if verbose else []) + \
        ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True, env=_env())
    if r.returncode != 0:
        raise RuntimeError("nvcc failed on %s:\n%s\n%s" % (src, r.stdout[-4000:], r.stderr[-8000:]))
    if verbose:
        sys.stderr.write(r.stderr)
    return obj


def _env():
    env = dict(os.environ)
    # the image exports CC/CXX=/opt/gcc/...; nvcc must use the system gcc it was validated with
    env.pop("CC", None)
    env.pop("CXX", None)
    return env


def build(force=False, verbose=False):
    nvcc = _nvcc()
    os.makedirs(OBJ, exist_ok=True)
    hdr_time = _newest_header()
    # objects built with other flags (another architecture, say) are stale whatever their mtimes
    stamp = os.path.join(OBJ, "nvcc_flags.txt")
    flags = "\n".join(NVCC_FLAGS) + "\n"
    if not os.path.exists(stamp) or open(stamp).read() != flags:
        force = True
    todo, objs = [], []
    for src in sources():
        obj = os.path.join(OBJ, src + ".o")
        objs.append(obj)
        stale = force or not os.path.exists(obj) or \
            os.path.getmtime(obj) < max(os.path.getmtime(os.path.join(CSRC, src)), hdr_time)
        if stale:
            todo.append(src)
    if todo:
        with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            list(ex.map(lambda s: _compile(nvcc, s, verbose), todo))
        with open(stamp, "w") as f:
            f.write(flags)
    if todo or not os.path.exists(LIB):
        cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-Xcompiler", "-fPIC", "-lpthread", "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True, env=_env())
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
