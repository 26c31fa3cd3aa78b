"""TEST INFRASTRUCTURE ONLY -- the reference's GPU normal sampler as the tests see it:

- `build()`: oracle/_ref/libmxref_random_gpu.so (oracle/random_gpu.mk), where the reference's
  sources exist;
- `launch_shape(n)`: LaunchRNG's bookkeeping (random/sampler.h), nthread and step, and `runs(n)`,
  the element range each state draws;
- `copy_seed(...)`: the seed of each generator copy (resource.cc ResourceParallelRandom);
- `RefGenerators`: one GPU's 4 copies of 32768 states held in host memory and advanced by the
  reference's own kernels, with the round robin of GetNext (++curr_ptr % 4), the seeds of
  SeedWithDeviceID / Seed, and lazy creation with the global seed. Needs a GPU.

float16 draws come from the reference; bfloat16 has no reference kernel and is the float32 draw
rounded once to nearest even (the extension's definition)."""
import ctypes
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_ref", "libmxref_random_gpu.so")
NUM_STATES = 32768
MIN_PER_THREAD = 64
STATE_BYTES = 64
COPIES = 4
MAX_GPUS = 16
MAGIC = 127
TYPE_FLAG = {'float32': 0, 'float64': 1, 'float16': 2}
NP = {'float32': np.float32, 'float64': np.float64, 'float16': np.float16, 'bfloat16': np.uint16}


def build():
    """oracle/_ref/libmxref_random_gpu.so, where the reference's sources exist"""
    if os.path.isfile("/root/reference/src/common/random_generator.cu"):
        import subprocess
        subprocess.run(["make", "-s", "-f", os.path.join(HERE, "random_gpu.mk")], check=True)


# ------------------------------------------------------------------------------- bookkeeping
def launch_shape(n):
    """(nthread, step) of LaunchRNG for n elements; (0, 0) when nothing launches"""
    if n <= 0:
        return 0, 0
    nloop = (n + MIN_PER_THREAD - 1) // MIN_PER_THREAD
    nthread = min(nloop, NUM_STATES)
    return nthread, (n + nthread - 1) // nthread


def runs(n):
    """[(state, first, end)] for every state that draws at least one element"""
    nthread, step = launch_shape(n)
    return [(t, t * step, min((t + 1) * step, n)) for t in range(nthread) if t * step < n]


def copy_seed(i, global_seed, dev_id=None):
    """SeedWithDeviceID (dev_id given) or Seed (dev_id None) of copy i, as uint32"""
    s = i * MAX_GPUS + (global_seed % 2 ** 32) * MAGIC
    if dev_id is not None:
        s += dev_id
    return s % 2 ** 32


def next_copy(curr_ptr):
    """GetNext: (the copy a call takes, the new curr_ptr)"""
    curr_ptr += 1
    return curr_ptr % COPIES, curr_ptr


def round_bf16(x):
    """float32 -> bfloat16 bits, to nearest even"""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


# ------------------------------------------------------------------------------- the reference
_lib = None


def ref():
    """the loaded libmxref_random_gpu.so, or None"""
    global _lib
    if _lib is None and os.path.exists(LIB):
        _lib = ctypes.CDLL(LIB)
        _lib.mxref_rand_seed.argtypes = [ctypes.c_uint32, ctypes.c_void_p]
        _lib.mxref_rand_normal.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_float,
                                           ctypes.c_int, ctypes.c_void_p]
    return _lib


def seeded_states(seed):
    st = np.zeros(NUM_STATES * STATE_BYTES, np.uint8)
    assert ref().mxref_rand_seed(ctypes.c_uint32(seed % 2 ** 32), st.ctypes.data) == 0
    return st


def draw(states, n, loc, scale, dtype):
    """the reference's normal_op draw of n elements from `states` (advanced in place); loc and
    scale as the float32 the operator parses"""
    flag_dt = 'float32' if dtype == 'bfloat16' else dtype
    out = np.zeros(max(n, 1), NP[flag_dt])
    assert ref().mxref_rand_normal(states.ctypes.data, int(n), ctypes.c_float(loc), ctypes.c_float(scale),
                                   TYPE_FLAG[flag_dt], out.ctypes.data) == 0
    out = out[:n]
    return round_bf16(out) if dtype == 'bfloat16' else out


class RefGenerators(object):
    """One GPU's parallel generators in the reference (ResourceParallelRandom<gpu>)"""

    def __init__(self, dev_id=0, global_seed=0):
        self.dev_id = dev_id
        self.copies = None
        self.global_seed = global_seed
        self.curr_ptr = 0

    def _ensure(self):
        if self.copies is None:
            self.copies = [seeded_states(copy_seed(i, self.global_seed, self.dev_id)) for i in range(COPIES)]

    def seed_all(self, seed):
        """MXRandomSeed"""
        self.global_seed = seed
        if self.copies is not None:
            self.copies = [seeded_states(copy_seed(i, seed, self.dev_id)) for i in range(COPIES)]
            self.curr_ptr = 0

    def seed_ctx(self, seed):
        """MXRandomSeedContext on this GPU"""
        self._ensure()
        self.copies = [seeded_states(copy_seed(i, seed)) for i in range(COPIES)]
        self.curr_ptr = 0

    def normal(self, n, loc, scale, dtype):
        self._ensure()
        i, self.curr_ptr = next_copy(self.curr_ptr)
        return draw(self.copies[i], n, loc, scale, dtype)
