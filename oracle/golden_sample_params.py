"""TEST INFRASTRUCTURE ONLY -- the reference's GPU multi-sample samplers (_sample_uniform,
_sample_normal, _sample_gamma, _sample_exponential) as the tests see them:

- `build()`: oracle/_ref/libmxref_sample_params_gpu.so (oracle/sample_params_gpu.mk), where the
  reference's sources exist;
- `multisample(states, dist, a, b, n, dtype)`: the reference's draw of n outputs from the parameter
  arrays a and b (numpy float16 / float32 / float64; b None for exponential) from one generator copy
  held in host memory (advanced in place);
- `ParamGenerators`: golden_sample.SampleGenerators (one GPU's 4 copies, their seeds and the round
  robin, drawn from by every scalar sampler) with these samplers beside them;
- `time_ref(...)`: the reference's own launch timed alone, for bench_sample_params.py;
- `rdiv_scalar(a, scalar)`: the reference's _rdiv_scalar (the 1.0 / scale of exponential), on the
  CPU through oracle/_ref/libmxref_rdiv.so (oracle/rdiv_scalar.mk, over the arithmetic oracle).

Never pass a gamma alpha whose draw cannot end (NaN, +-inf, <= -2/3): the reference's loop would not
return. Needs a GPU."""
import ctypes
import os

import numpy as np

import golden_random as GR
import golden_sample as GS

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_ref", "libmxref_sample_params_gpu.so")
RDIV_LIB = os.path.join(HERE, "_ref", "libmxref_rdiv.so")
TYPE_FLAG = {'float32': 0, 'float64': 1, 'float16': 2}
DIST = {'uniform': 0, 'normal': 1, 'gamma': 2, 'exponential': 3}


def build():
    """oracle/_ref/libmxref_sample_params_gpu.so and libmxref_rdiv.so, where the reference's sources
    exist"""
    import subprocess
    if os.path.isfile("/root/reference/src/common/random_generator.cu"):
        subprocess.run(["make", "-s", "-f", os.path.join(HERE, "sample_params_gpu.mk")], check=True)
    if os.path.isfile("/root/reference/src/operator/tensor/matrix_op-inl.h"):
        subprocess.run(["make", "-s", "-f", os.path.join(HERE, "rdiv_scalar.mk")], check=True)


_lib = None


def ref():
    """the loaded libmxref_sample_params_gpu.so, or None"""
    global _lib
    if _lib is None and os.path.exists(LIB):
        _lib = ctypes.CDLL(LIB)
        _lib.mxref_multisample.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                                           ctypes.c_void_p]
        _lib.mxref_multisample_time.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int64,
                                                ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
                                                ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
    return _lib


def available():
    """the seeding, scalar-sampler and multi-sample reference libraries are all present"""
    return GS.available() and ref() is not None


def _gamma_terminates(alpha):
    d = np.where(alpha < 1, alpha.astype(np.float64) + 2.0 / 3.0, alpha.astype(np.float64) - 1.0 / 3.0)
    return bool(np.all(np.isfinite(d) & (d > 0)))


def multisample(states, dist, a, b, n, dtype):
    """the reference's draw of n elements of sampler `dist` from parameters a (and b) of one numpy
    dtype, into `dtype`, from `states` (advanced in place)"""
    a = np.ascontiguousarray(a).ravel()
    b = a if b is None else np.ascontiguousarray(b).ravel()
    assert a.dtype == b.dtype and a.size == b.size and a.size > 0 and n % a.size == 0
    if dist == 'gamma':
        assert _gamma_terminates(a), "the reference's gamma draw would not end for these alphas"
    out = np.zeros(max(n, 1), np.dtype(dtype))
    assert ref().mxref_multisample(DIST[dist], states.ctypes.data, TYPE_FLAG[a.dtype.name], TYPE_FLAG[dtype],
                                   a.size, a.ctypes.data, b.ctypes.data, int(n), out.ctypes.data) == 0
    return out[:n]


def time_ref(dist, nparm, n, p0, p1, ptype, dtype, warmup=10, reps=50):
    """ms per call of the reference's own launch over n outputs from nparm parameter pairs, every
    pair (p0, p1) (its states on the device, CUDA events around the launches only)"""
    a = np.array([p0], ptype)
    b = np.array([p1], ptype)
    ms = ctypes.c_float()
    assert ref().mxref_multisample_time(DIST[dist], TYPE_FLAG[np.dtype(ptype).name], TYPE_FLAG[dtype], int(nparm),
                                        a.ctypes.data, b.ctypes.data, int(n), warmup, reps, ctypes.byref(ms)) == 0
    return ms.value


def rdiv_scalar(a, scalar):
    """(the parsed double, scalar / a) of the reference's _rdiv_scalar(scalar=str(scalar)) over numpy
    array a (float16, float32 or float64)"""
    lib = ctypes.CDLL(RDIV_LIB)
    a = np.ascontiguousarray(a)
    out = np.zeros_like(a)
    parsed = ctypes.c_double()
    err = ctypes.create_string_buffer(512)
    assert lib.mxref_ar_rdiv_scalar(ctypes.c_int(TYPE_FLAG[a.dtype.name]), ctypes.c_void_p(a.ctypes.data),
                                    str(scalar).encode(), ctypes.byref(parsed), ctypes.c_void_p(out.ctypes.data),
                                    ctypes.c_int64(a.size), err, ctypes.c_int(512)) == 0, err.value
    return parsed.value, out


class ParamGenerators(GS.SampleGenerators):
    """One GPU's parallel generators in the reference, drawn from by the scalar and the multi-sample
    samplers in turn"""

    def multisample(self, dist, a, b, n, dtype):
        self._ensure()
        i, self.curr_ptr = GR.next_copy(self.curr_ptr)
        return multisample(self.copies[i], dist, a, b, n, dtype)
