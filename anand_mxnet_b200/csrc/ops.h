// ops.h -- the imperative-operator surface (MXImperativeInvokeEx subset): the reference's optimizer
// operators (src/operator/optimizer_op.cc:195-710) plus the few elementwise helpers that updaters
// written in the host language rely on. All run on the arrays' GPU through the dense fused kernel.
#pragma once
#include <cstdint>
#include <map>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "ndarray.h"
#include "op_params.h"

namespace b200kv {

struct OpInfo;
// outputs: caller-provided (in place) or empty -> allocated and appended
typedef void (*OpFn)(const OpInfo& op, const std::vector<NDArray>& inputs, std::vector<NDArray>* outputs,
                     const Params& params);

// One operator: its name, its handler, and what the handler varies on (a kernel op code, kOp* flag
// bits, or an index into the family's own table). Handlers use `name` in error messages only.
struct OpInfo {
  const char* name;
  OpFn run;
  int variant;
};

// variant bits of the operators that come in plain, mom, mp, multi and preloaded forms
enum OpFlags { kOpMom = 1, kOpMp = 2, kOpMulti = 4, kOpPreloaded = 8 };

// each family's operators: ops.cc, multi_ops.cc, update_ops.cc, arith_ops.cc, reduce_ops.cc, sum_ops.cc,
// random_ops.cc, sample_ops.cc, sample_param_ops.cc
extern const std::vector<OpInfo> kCoreOps, kMultiTensorOps, kUpdateOps, kArithOps, kReduceOps, kSumOps,
    kRandomOps, kSampleOps, kSampleParamOps;

// nullptr when the operator is not registered
const OpInfo* FindOp(const std::string& name);

// runs op->run; a malformed rescale_grad or clip_gradient is refused first, whichever the operator
void InvokeOp(const OpInfo* op, const std::vector<NDArray>& inputs, std::vector<NDArray>* outputs,
              const Params& params);

// outputs[i], or a new array appended to outputs when the caller passed fewer
NDArray OutOr(std::vector<NDArray>* outputs, size_t i, const std::vector<int64_t>& shape, Context ctx,
              int dtype);
// the front-end passes out=weight; a distinct out receives the weight first (then updated in place)
NDArray InPlace(const std::vector<NDArray>& in, size_t widx, std::vector<NDArray>* outputs, size_t oidx);

// "row_sparse" or "default", for error messages
const char* StypeName(int stype);

// FillDnsZerosRspImpl (init_op.h:474-487) for optimizer states: every row_sparse array of `states`
// that holds no rows gets all `rows` rows, zero values and ids 0..rows-1, in one operation on its
// GPU's lane, so that a kernel can address its rows by table row id. Dense arrays and row_sparse
// arrays that hold rows are left alone. launch_name is kept by Engine::CountLaunch.
void ZeroFillEmptyRspStates(const std::vector<NDArray>& states, int64_t rows, const char* launch_name);

// The operands of a row_sparse optimizer operator `op` whose rows are addressed by table row id:
// in[0] the weight, in[2...] the states. A row_sparse weight holds every row (CheckAllRowsPresent,
// operator_common.h:500-511, under the reference's function name `func`), a row_sparse state holds
// every row or none, and the one out is the weight itself (kWriteInplace).
void CheckRspTable(const char* op, const char* func, const std::vector<NDArray>& in,
                   const std::vector<NDArray>& outputs);

// out = op(a[, b], scalar[, scalar2]) through LaunchElementwise (an EwOp code) on out's GPU, after
// checking that every operand is a dense array on that GPU with out's size and dtype. A failed
// check throws before anything is enqueued.
void Elementwise(int op, const NDArray& a, const NDArray* b, double scalar, const NDArray& out,
                 double scalar2 = 0.0);
// out = op(a, b) for a binary EwOp code, where b holds one value per row of a's trailing axis
// (b[i / a.shape().back()]), with Elementwise's checks; b's size must be out's over that row length
void ElementwiseRows(int op, const NDArray& a, const NDArray& b, const NDArray& out);

// Device copies of the descriptor tables an operator call builds from its operands, kept per
// operand list so that a repeated call uploads nothing. The key holds everything the tables were
// built from (addresses, sizes, flags) and a hit compares it in full. Past 512 entries the whole
// cache is dropped. Each caller builds its own tables and keeps its own cache.
class TableCache {
 public:
  struct Tables {
    explicit Tables(int dev) : dev(dev) {}
    int dev;
    int n_chunks = 0;
    void* d[3] = {};
    size_t bytes[3] = {};
    // buffer i: `size` bytes on dev, the first `host_bytes` of them copied from `host`
    void Upload(int i, size_t size, const void* host, size_t host_bytes, cudaStream_t st);
    ~Tables();
  };
  // the tables of `key`, or nullptr
  const Tables* Find(const std::vector<uint64_t>& key) const;
  // stores tables the caller has filled in full: an entry is never seen half built, and tables
  // whose filling threw are freed by their owner instead
  const Tables* Insert(std::vector<uint64_t> key, std::unique_ptr<Tables> tables);

 private:
  std::map<std::vector<uint64_t>, std::unique_ptr<Tables>> map_;
};

}  // namespace b200kv
