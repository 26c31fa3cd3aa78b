// random_ops.h -- the GPU parallel random generators of random_ops.cc, for the C API.
#pragma once
#include <cstdint>

#include "ndarray.h"

namespace b200kv {

// MXRandomSeed: the global seed, and every GPU's generator copies reseeded with it
void RandomSeed(uint32_t seed);
// MXRandomSeedContext: one GPU's copies reseeded without the device term (a CPU context: nothing)
void RandomSeedContext(uint32_t seed, Context ctx);
// normal(loc, scale) into a dense GPU array from the device's next generator copy; staged = false
// selects the reference's per-thread store order (measurement only)
void RandNormalInto(const NDArray& out, float loc, float scale, bool staged);
// a copy of generator copy `copy` of GPU dev (bytes must be the copy's size), after its last writer
void RandomStates(int dev, int copy, void* host, size_t bytes);

}  // namespace b200kv
