// rowsparse.h -- row_sparse helpers shared by the store (rowsparse.cc), the imperative operators
// (ops.cc) and CopyFromTo (ndarray.cc).
#pragma once
#include <vector>

#include "kernels.h"
#include "ndarray.h"

namespace b200kv {

// An optimizer step with the row_sparse gradient `g` on a float32 table `w` whose rows are addressed
// by table row id: w is dense, or row_sparse with every row, and so is each of `states` (in the
// operator's input order; entries past the op's own states are not read and may be none). `L`
// carries the op (kUpd*) and its scalars.
// CountLaunch keeps `launch_name`; bytes_per_elem is the op's algorithmic traffic per element.
// Lazy: only the rows listed in g move, w in place (LaunchRspRowUpdateOp). An empty g changes nothing.
void RunRspRowUpdate(UpdateLaunch L, const NDArray& w, const NDArray& g, const std::vector<NDArray>& states,
                     const char* launch_name, int bytes_per_elem);
// Standard: every element of the table moves into `out` (w itself, or a dense array of w's shape),
// rows absent from g with g = +0.0f (LaunchRspGradUpdateOp over the row map of BuildRowMap).
void RunRspGradUpdate(UpdateLaunch L, const NDArray& w, const NDArray& g, const std::vector<NDArray>& states,
                      const NDArray& out, const char* launch_name, int bytes_per_elem);

// sgd_update (kind kOptSGDSingle), sgd_mom_update (kOptSGD) or adam_update (kOptAdam) with a
// row_sparse gradient, in place on w: the lazy form (only g's rows move, optimizer_op-inl.h:426-475,
// 749-801, 1383-1408) or the standard form (every row, optimizer_op-inl.h:505-528, optimizer_op.cc:
// 108-139, 195-229). `L` carries the scalars; states starts with mom (sgd_mom_update) or mean and
// var (adam_update).
void SgdAdamRspUpdate(int kind, bool lazy, UpdateLaunch L, const NDArray& w, const NDArray& g,
                      const std::vector<NDArray>& states);

// The row map of a row_sparse gradient `g` over a table of `rows` rows: an int32 per table row, the
// row's position among g's stored rows or -1 (LaunchRowMap). Declared written by `op` and built on
// its stream, so it is called after every other operand of `op` is declared.
NDArray BuildRowMap(LaneOp& op, const NDArray& g, int64_t rows);

// add_n of row_sparse float32 arrays on out's GPU (ElementwiseSumRsp, ndarray_function.cc:60-176):
// out holds the sorted union of the inputs' row ids, each row +0.0f plus the inputs that hold it in
// input order. The store's merge (LaunchRspMerge without an update) over up to kMaxSrc inputs at a
// time; past that the partial sum is the first source of the next merge, which is bit-identical
// (+0.0f + a partial row is that row: a partial sum is never -0.0f). out may be one of the inputs.
// The caller has checked shapes, dtypes and devices. Waits on the host for the row count.
void SumRowSparse(const std::vector<NDArray>& in, const NDArray& out);

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
