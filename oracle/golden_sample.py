"""TEST INFRASTRUCTURE ONLY -- the reference's GPU uniform, exponential, gamma and randint samplers
as the tests see them, beside its normal sampler (oracle/golden_random.py):

- `build()`: oracle/_ref/libmxref_sample_gpu.so (oracle/sample_gpu.mk), where the reference's
  sources exist;
- `sample(states, dist, n, params, dtype)`: the reference's uniform_op / exponential_op / gamma_op /
  rand_int_op draw from one generator copy held in host memory (advanced in place);
- `SampleGenerators`: golden_random.RefGenerators (one GPU's 4 copies, their seeds and the round
  robin) with these four samplers beside normal, all drawing from the same copies in turn;
- `time_ref(...)`: the reference's own launch of a sampler timed alone, for bench_sample.py.

bfloat16 has no reference kernel and is the float32 draw rounded once to nearest even (the
extension's definition). Needs a GPU."""
import ctypes
import os

import numpy as np

import golden_random as GR

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_ref", "libmxref_sample_gpu.so")
TYPE_FLAG = {'float32': 0, 'float64': 1, 'float16': 2, 'int32': 4, 'int64': 6}
NP = {'float32': np.float32, 'float64': np.float64, 'float16': np.float16, 'int32': np.int32, 'int64': np.int64}
DIST = {'uniform': 0, 'exponential': 1, 'gamma': 2, 'randint': 3}


def build():
    """oracle/_ref/libmxref_sample_gpu.so, where the reference's sources exist"""
    if os.path.isfile("/root/reference/src/common/random_generator.cu"):
        import subprocess
        subprocess.run(["make", "-s", "-f", os.path.join(HERE, "sample_gpu.mk")], check=True)


_lib = None


def ref():
    """the loaded libmxref_sample_gpu.so, or None"""
    global _lib
    if _lib is None and os.path.exists(LIB):
        _lib = ctypes.CDLL(LIB)
        for name in ("uniform", "gamma"):
            getattr(_lib, "mxref_sample_" + name).argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_float,
                                                              ctypes.c_float, ctypes.c_int, ctypes.c_void_p]
        _lib.mxref_sample_exponential.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int,
                                                  ctypes.c_void_p]
        _lib.mxref_sample_randint.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                              ctypes.c_int, ctypes.c_void_p]
        _lib.mxref_sample_time.argtypes = [ctypes.c_int, ctypes.c_int64, ctypes.c_double, ctypes.c_double,
                                           ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
    return _lib


def available():
    """both reference libraries are present: the seeding and normal sampler, and these samplers"""
    return GR.ref() is not None and ref() is not None


def sample(states, dist, n, params, dtype):
    """the reference's draw of n elements of sampler `dist` from `states` (advanced in place).
    params: (low, high), (lam,) or (alpha, beta) as the float32 the operator parses, or randint's
    int64 (low, high)"""
    flag_dt = 'float32' if dtype == 'bfloat16' else dtype
    out = np.zeros(max(n, 1), NP[flag_dt])
    fn = getattr(ref(), "mxref_sample_" + dist)
    if dist == 'randint':
        args = [ctypes.c_int64(int(p)) for p in params]
    else:
        args = [ctypes.c_float(p) for p in params]
    assert fn(states.ctypes.data, int(n), *args, TYPE_FLAG[flag_dt], out.ctypes.data) == 0
    out = out[:n]
    return GR.round_bf16(out) if dtype == 'bfloat16' else out


def time_ref(dist, n, p0, p1, dtype, warmup=20, reps=200):
    """ms per call of the reference's own launch of sampler `dist` over n elements (its states on
    the device, CUDA events around the launches only)"""
    ms = ctypes.c_float()
    assert ref().mxref_sample_time(DIST[dist], int(n), float(p0), float(p1), TYPE_FLAG[dtype], warmup, reps,
                                   ctypes.byref(ms)) == 0
    return ms.value


class SampleGenerators(GR.RefGenerators):
    """One GPU's parallel generators in the reference, drawn from by every sampler in turn"""

    def _sample(self, dist, n, params, dtype):
        self._ensure()
        i, self.curr_ptr = GR.next_copy(self.curr_ptr)
        return sample(self.copies[i], dist, n, params, dtype)

    def uniform(self, n, low, high, dtype):
        return self._sample('uniform', n, (low, high), dtype)

    def exponential(self, n, lam, dtype):
        return self._sample('exponential', n, (lam,), dtype)

    def gamma(self, n, alpha, beta, dtype):
        return self._sample('gamma', n, (alpha, beta), dtype)

    def randint(self, n, low, high, dtype):
        return self._sample('randint', n, (low, high), dtype)
