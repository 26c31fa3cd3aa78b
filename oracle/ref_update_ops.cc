// TEST INFRASTRUCTURE ONLY -- never linked into or loaded by the product library.
//
// oracle/_ref/libmxref_update.so: the reference's own parameter parsers and FCompute<cpu> functions
// of the single-tensor optimizer operators of its NAG / Signum / RMSProp / FTML / Ftrl optimizers,
// compiled from src/operator/optimizer_op-inl.h where it lies (nothing is copied), behind the same
// generic entry point as oracle/ref_ops.cc (op name + flat arrays + the string attribute dict):
//   nag_mom_update       NAGMomUpdate<cpu>       optimizer_op-inl.h:1061-1106
//   mp_nag_mom_update    MP_NAGMomUpdate<cpu>    optimizer_op-inl.h:1108-1160
//   signsgd_update       SignSGDUpdate<cpu>      optimizer_op-inl.h:2344-2376
//   signum_update        SignumUpdate<cpu>       optimizer_op-inl.h:2412-2452
//   rmsprop_update       RMSPropUpdate<cpu>      optimizer_op-inl.h:2052-2099
//   rmspropalex_update   RMSPropAlexUpdate<cpu>  optimizer_op-inl.h:1953-2012
//   ftml_update          FTMLUpdate<cpu>         optimizer_op-inl.h:1205-1249
//   ftrl_update          FtrlUpdate<cpu>         optimizer_op-inl.h:2133-2183
// A library of its own (built by oracle/update_ops.mk), so libmxref.so stays as it is.
#include <cstdint>
#include <cstring>
#include <map>
#include <string>
#include <vector>
#include <dmlc/logging.h>
#include <mshadow/tensor.h>
#include <nnvm/op.h>
#include "operator/optimizer_op-inl.h"

using namespace mxnet;

namespace mxnet {
namespace op {
// the parameter managers optimizer_op.cc:36-44 registers
DMLC_REGISTER_PARAMETER(NAGMomParam);
DMLC_REGISTER_PARAMETER(SignSGDParam);
DMLC_REGISTER_PARAMETER(SignumParam);
DMLC_REGISTER_PARAMETER(RMSPropParam);
DMLC_REGISTER_PARAMETER(RMSPropAlexParam);
DMLC_REGISTER_PARAMETER(FTMLParam);
DMLC_REGISTER_PARAMETER(FtrlParam);
}  // namespace op
// the OMP thread-count policy consulted by Kernel<OP,cpu>::Launch (src/engine/openmp.cc): one thread
namespace engine {
OpenMP::OpenMP() : omp_num_threads_set_in_environment_(false) {}
OpenMP* OpenMP::Get() {
  static OpenMP inst;
  return &inst;
}
int OpenMP::GetRecommendedOMPThreadCount(bool) const { return 1; }
}  // namespace engine
}  // namespace mxnet

namespace {

typedef void (*Parser)(nnvm::NodeAttrs*);
typedef void (*Compute)(const nnvm::NodeAttrs&, const OpContext&, const std::vector<TBlob>&,
                        const std::vector<OpReqType>&, const std::vector<TBlob>&);
struct Entry { Parser parse; Compute fn; };

const std::map<std::string, Entry>& Table() {
  using namespace mxnet::op;
  // as optimizer_op.cc:49-890 registers them (attr_parser, FCompute<cpu>)
  static std::map<std::string, Entry> t = {
      {"nag_mom_update", {ParamParser<NAGMomParam>, NAGMomUpdate<cpu>}},
      {"mp_nag_mom_update", {ParamParser<NAGMomParam>, MP_NAGMomUpdate<cpu>}},
      {"signsgd_update", {ParamParser<SignSGDParam>, SignSGDUpdate<cpu>}},
      {"signum_update", {ParamParser<SignumParam>, SignumUpdate<cpu>}},
      {"rmsprop_update", {ParamParser<RMSPropParam>, RMSPropUpdate<cpu>}},
      {"rmspropalex_update", {ParamParser<RMSPropAlexParam>, RMSPropAlexUpdate<cpu>}},
      {"ftml_update", {ParamParser<FTMLParam>, FTMLUpdate<cpu>}},
      {"ftrl_update", {ParamParser<FtrlParam>, FtrlUpdate<cpu>}},
  };
  return t;
}

}  // namespace

extern "C" {

// Same contract as ref_ops.cc's mxref_op_invoke: flat arrays, mshadow dtype flags, sizes in
// elements; an output that is the same buffer as an input aliases it, as out=weight does.
// Returns 0, or -1 with the dmlc::Error text in `err`.
int mxref_op_invoke(const char* op, int nin, void** in_ptr, const int* in_dtype, const int64_t* in_size,
                    int nout, void** out_ptr, const int* out_dtype, const int64_t* out_size,
                    int nparam, const char** keys, const char** vals, char* err, int errlen) {
  try {
    auto it = Table().find(op);
    if (it == Table().end()) throw dmlc::Error(std::string("unknown operator ") + op);
    nnvm::NodeAttrs attrs;
    attrs.name = op;
    for (int i = 0; i < nparam; ++i) attrs.dict[keys[i]] = vals[i];
    it->second.parse(&attrs);
    OpContext ctx;
    ctx.is_train = false;
    ctx.need_grad = false;
    ctx.run_ctx.stream = nullptr;
    std::vector<TBlob> in, out;
    for (int i = 0; i < nin; ++i) {
      in.emplace_back(in_ptr[i], mxnet::TShape({static_cast<dim_t>(in_size[i])}), 1, in_dtype[i]);
    }
    for (int i = 0; i < nout; ++i) {
      out.emplace_back(out_ptr[i], mxnet::TShape({static_cast<dim_t>(out_size[i])}), 1, out_dtype[i]);
    }
    std::vector<OpReqType> req(nout, kWriteTo);
    it->second.fn(attrs, ctx, in, req, out);
    return 0;
  } catch (const std::exception& e) {
    if (err && errlen > 0) {
      std::strncpy(err, e.what(), errlen - 1);
      err[errlen - 1] = '\0';
    }
    return -1;
  }
}

int mxref_op_known(const char* op) { return Table().count(op) ? 1 : 0; }

}  // extern "C"
