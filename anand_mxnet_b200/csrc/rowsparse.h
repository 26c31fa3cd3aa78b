// rowsparse.h -- row_sparse helpers shared by the store (rowsparse.cc), the imperative operators
// (ops.cc) and CopyFromTo (ndarray.cc).
#pragma once
#include "kernels.h"
#include "ndarray.h"

namespace b200kv {

// Standard (non-lazy) optimizer step with a row_sparse gradient: every row of the dense weight
// `w` (and of the dense states) moves; rows absent from `g` see grad = 0
// (optimizer_op-inl.h:505-528, optimizer_op.cc:108-139, 195-229). `L` carries opt + scalars.
void RunRspStdUpdate(const NDArray& w, const NDArray& g, const NDArray& s1, const NDArray& s2,
                     RspUpdateLaunch L);

// CopyFromTo across storage types (src/ndarray/ndarray.cc:1147-1196 + cast_storage-inl.h:74-140):
// dense -> row_sparse keeps the rows with a non-zero element, row_sparse -> dense scatters the
// rows over zeros. float32 only; the cast runs on a GPU (the source's, else the target's).
void CastStorageCopy(const NDArray& from, const NDArray& to);

// CopyFromTo(src, out) for every out at once (a whole-value pull of a row_sparse value, comm.h:
// 598-616): ONE launch on src's GPU writes every target, row_sparse outs get the ids and rows,
// dense outs every table row (stored row or zeros). Outs on other GPUs are written by peer stores,
// host outs through a staging array. Every out is checked before anything is enqueued.
void BroadcastRspValue(const NDArray& src, const std::vector<NDArray>& outs);

}  // namespace b200kv
