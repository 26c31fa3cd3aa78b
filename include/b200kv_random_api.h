/*
 * b200kv_random_api.h -- the C ABI of libb200kv.so's GPU random number generators, included by
 * b200kv_c_api.h (whose types and conventions it uses).
 *
 * Each GPU holds the reference's parallel generators (src/resource.cc, ResourceParallelRandom<gpu>):
 * 4 copies of 32768 curand Philox4_32_10 states, allocated and seeded on the GPU's first sampling
 * call. The operator _random_normal (MXImperativeInvokeEx) draws from the next copy in turn.
 *
 * Part A: the reference's seeding functions, with the signatures of include/mxnet/c_api.h.
 * Part B: extensions (prefix B200KV) for tests and measurement.
 */
#ifndef B200KV_RANDOM_API_H_
#define B200KV_RANDOM_API_H_

#include "b200kv_c_api.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- Part A ---- */
/* c_api.h:254 -- the global seed; every GPU's generators reseeded (copy i: dev + i*16 + seed*127),
 * and GPUs first used later are seeded with it */
B200KV_DLL int MXRandomSeed(int seed);
/* c_api.h:261 -- one device's generators reseeded (copy i: i*16 + seed*127, no device term); a CPU
 * context changes nothing here (there is no CPU sampling) */
B200KV_DLL int MXRandomSeedContext(int seed, int dev_type, int dev_id);

/* ---- Part B ---- */
/* the bytes of generator copy `copy` (0..3) of GPU dev_id (bytes = 32768 * 64), allocating and
 * seeding the device's copies first if needed; waits for the copy's last writer */
B200KV_DLL int B200KVRandomStates(int dev_id, int copy, void* out, size_t bytes);
/* _random_normal into out (a dense GPU array) from the device's next copy, with the staged store
 * order (staged = 1) or each thread storing as it draws (staged = 0): the same numbers, for
 * measurement */
B200KV_DLL int B200KVRandomNormalInto(NDArrayHandle out, float loc, float scale, int staged);

#ifdef __cplusplus
}
#endif
#endif /* B200KV_RANDOM_API_H_ */
