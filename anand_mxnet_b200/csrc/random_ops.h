// random_ops.h -- the GPU parallel random generators of random_ops.cc, for the C API and the
// sampling operators (random_ops.cc, sample_ops.cc).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <functional>
#include <string>
#include <vector>

#include "ndarray.h"
#include "op_params.h"

namespace b200kv {

// MXRandomSeed: the global seed, and every GPU's generator copies reseeded with it
void RandomSeed(uint32_t seed);
// MXRandomSeedContext: one GPU's copies reseeded without the device term (a CPU context: nothing)
void RandomSeedContext(uint32_t seed, Context ctx);
// One sampling call into a dense GPU array: the device's next generator copy (++curr_ptr % 4) and
// out are declared as writes of one operation on the GPU's compute lane, and launch(states, stream)
// issues the draw from that copy. launch_name and out's bytes go to Engine::CountLaunch. reads: the
// arrays the draw reads (the multi-sample operators' parameters; out may be one of them).
void SampleInto(const NDArray& out, const char* launch_name,
                const std::function<void(void* states, cudaStream_t stream)>& launch,
                const std::vector<NDArray>& reads = {});
// normal(loc, scale) into a dense GPU array from the device's next generator copy; staged = false
// selects the reference's per-thread store order (measurement only)
void RandNormalInto(const NDArray& out, float loc, float scale, bool staged);
// a copy of generator copy `copy` of GPU dev (bytes must be the copy's size), after its last writer
void RandomStates(int dev, int copy, void* host, size_t bytes);

// ---- the sampling operators' parameters (random/sample_op.h) ----
// "gpu(1)", "cpu(0)", "cpu_pinned(0)" (Context::FromString); an empty string is the CPU
Context ParseCtx(const std::string& s, const char* op);
// TShape "(2, 3)", "[2, 3]", "(5,)", "5" or "()"
std::vector<int64_t> ParseShape(const std::string& s, const char* op);
// The dtype enum of SampleNormalParam and its float siblings, with bfloat16 as an extension, or of
// SampleRandIntParam (integer: int32, int64); -1 is None
int ParseDType(const std::string& s, const char* op, bool integer = false);
// refused unless dtype is one a sampler writes: float16 / bfloat16 / float32 / float64, or int32 /
// int64 when integer
void CheckSampleDType(const char* op, int dtype, bool integer);

// Where a call with shape / ctx / dtype keys draws: out's context, shape and dtype when out is given
// (a given shape or dtype must agree with them, and out must be dense), else shape (required) on ctx.
// dtype None is float32 (int32 when integer). Refused unless the dtype is one the sampler writes and
// the context is a GPU.
struct SampleTarget {
  std::vector<int64_t> shape;
  Context ctx;
  int dtype;
};
SampleTarget ParseSampleTarget(const char* op, const Params& p, const std::vector<NDArray>& outputs,
                               bool integer);

}  // namespace b200kv
