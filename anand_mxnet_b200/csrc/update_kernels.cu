// update_kernels.cu -- the single-tensor optimizer operators that the per-key updater callback
// reaches through MXImperativeInvokeEx, with dense gradients: nag_mom_update / mp_nag_mom_update,
// signsgd_update / signum_update, rmsprop_update / rmspropalex_update, ftml_update, ftrl_update.
// The kernel, update_kernel<OP, T, false>, is in update_kernel.cuh.
#include "update_kernel.cuh"

namespace b200kv {
namespace {

template <int OP>
void LaunchFp32(const UpdateLaunch& L, cudaStream_t stream) {
  KV_CHECK_EQ(L.dtype, kFloat32) << "this optimizer operator runs on float32 arrays";
  Launch<OP, float>(L, stream);
}

}  // namespace

void LaunchUpdateOp(const UpdateLaunch& L, cudaStream_t stream) {
  if (L.n == 0) return;
  switch (L.op) {
    case kUpdNAG: LaunchFp32<kUpdNAG>(L, stream); break;
    case kUpdMPNAG:
      if (L.dtype == kFloat16) Launch<kUpdMPNAG, __half>(L, stream);
      else if (L.dtype == kBfloat16) Launch<kUpdMPNAG, __nv_bfloat16>(L, stream);
      else KV_FATAL << "mp_nag_mom_update runs on float16 / bfloat16 weights, not " << DTypeName(L.dtype);
      break;
    case kUpdSignSGD: LaunchFp32<kUpdSignSGD>(L, stream); break;
    case kUpdSignum: LaunchFp32<kUpdSignum>(L, stream); break;
    case kUpdRMSProp: LaunchFp32<kUpdRMSProp>(L, stream); break;
    case kUpdRMSPropAlex: LaunchFp32<kUpdRMSPropAlex>(L, stream); break;
    case kUpdFTML: LaunchFp32<kUpdFTML>(L, stream); break;
    case kUpdFtrl: LaunchFp32<kUpdFtrl>(L, stream); break;
    default: KV_FATAL << "unknown update operator " << L.op;
  }
}

}  // namespace b200kv
