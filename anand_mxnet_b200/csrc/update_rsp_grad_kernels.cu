// update_rsp_grad_kernels.cu -- nag_mom_update, signsgd_update, signum_update, rmsprop_update,
// rmspropalex_update, ftml_update and ftrl_update with a dense float32 weight and states and a
// row_sparse gradient, and the standard (lazy_update=False) forms of sgd_update, sgd_mom_update and
// adam_update: update_kernel<OP, float, true> (update_kernel.cuh) over the whole table, reading the
// gradient's stored rows through the row map of LaunchRowMap.
#include "update_kernel.cuh"

namespace b200kv {

void LaunchRspGradUpdateOp(const UpdateLaunch& L, cudaStream_t stream) {
  if (L.n == 0) return;
  KV_CHECK_EQ(L.dtype, kFloat32) << "a row_sparse gradient runs on float32 arrays";
  KV_CHECK(L.row_map && L.row_len > 0) << "a row_sparse gradient needs its row map and a row length";
  switch (L.op) {
    case kUpdNAG: Launch<kUpdNAG, float, true>(L, stream); break;
    case kUpdSignSGD: Launch<kUpdSignSGD, float, true>(L, stream); break;
    case kUpdSignum: Launch<kUpdSignum, float, true>(L, stream); break;
    case kUpdRMSProp: Launch<kUpdRMSProp, float, true>(L, stream); break;
    case kUpdRMSPropAlex: Launch<kUpdRMSPropAlex, float, true>(L, stream); break;
    case kUpdFTML: Launch<kUpdFTML, float, true>(L, stream); break;
    case kUpdFtrl: Launch<kUpdFtrl, float, true>(L, stream); break;
    case kUpdSGDStd: Launch<kUpdSGDStd, float, true>(L, stream); break;
    case kUpdSGDMom: Launch<kUpdSGDMom, float, true>(L, stream); break;
    case kUpdAdamStd: Launch<kUpdAdamStd, float, true>(L, stream); break;
    default: KV_FATAL << "operator " << L.op << " has no row_sparse-gradient form";
  }
}

}  // namespace b200kv
