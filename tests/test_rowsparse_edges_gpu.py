"""The row_sparse union, retain and broadcast kernels on both sides of every size threshold in their
code. The thresholds are read from rowsparse_kernels.cu / kernels.h (oracle/rsp_edges.py), so a
retuned constant moves the cases with it. An off-by-one in a block base, a popcount mask or a tile
bound only shows past one of these edges; below it the results stay bit-exact.

Checkers: ids, unique counts and retained rows against numpy (np.unique, fancy indexing, zeros for
absent rows); merged sums and the fused lazy updates bit for bit against the CPU oracle, which adds
the sources in source order as the reference does. Every sum over 3 or more sources mixes
magnitudes around 2**24 with values of order 1, so a kernel that adds in any other order fails."""
import numpy as np
import pytest

import kvoracle as K
import rsp_edges as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mx():
    import anand_mxnet_b200 as mx
    return mx


def eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.fixture(params=["bitmap", "sort"])
def union_path(request, monkeypatch):
    """both id-union front-ends: the bitmap rank, and the radix sort B200KV_RSP_SORT=1 forces
    (read on every call)"""
    if request.param == "sort":
        monkeypatch.setenv("B200KV_RSP_SORT", "1")
    else:
        monkeypatch.delenv("B200KV_RSP_SORT", raising=False)
    return request.param


def mixed_vals(rng, n, row_len):
    """rows whose sum over several sources depends on the order of the adds: about half the
    elements are of magnitude 2**24, the rest of order 1, with random signs"""
    big = rng.random((n, row_len)) < 0.5
    mag = np.where(big, 2.0 ** 24, 1.0) * rng.uniform(0.5, 1.5, (n, row_len))
    return (mag * rng.choice([-1.0, 1.0], (n, row_len))).astype(np.float32)


def fp32_sum(idxs, vals, union, order):
    """the fp32 sum of the sources in the given order, at the union's rows (0.0f first)"""
    acc = np.zeros((union.size, vals[0].shape[1]), np.float32)
    for s in order:
        p = np.searchsorted(union, idxs[s])
        acc[p] = acc[p] + vals[s]
    return acc


def check_order_sensitive(idxs, vals, want_idx, want_val):
    """the case is one where the order of the adds shows: the oracle's source-order fp32 sum differs
    from the reverse-order fp32 sum in at least one element, and stays within the recursive-summation
    error bound of the float64 sum"""
    n = len(idxs)
    assert n >= 3
    assert not eq(fp32_sum(idxs, vals, want_idx, reversed(range(n))), want_val), "order-insensitive case"
    s64 = np.zeros(want_val.shape, np.float64)
    a64 = np.zeros(want_val.shape, np.float64)
    for i, v in zip(idxs, vals):
        p = np.searchsorted(want_idx, i)
        s64[p] += v
        a64[p] += np.abs(v.astype(np.float64))
    assert np.all(np.abs(want_val - s64) <= n * 2.0 ** -24 * a64)


def rsp(mx, idx, val, shape, dtype=None):
    return mx.nd.sparse.row_sparse_array((val, np.asarray(idx, np.int64)), shape=shape, ctx=mx.gpu(0), dtype=dtype)


def ids_nd(mx, ids, dtype=np.int64):
    return mx.nd.array(np.asarray(ids).astype(dtype), mx.gpu(0), dtype)


def whole_value(mx, kv, key, shape, dtype=np.float32):
    """the stored value itself (pull with ignore_sparse=False into a row_sparse out)"""
    out = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0), dtype)
    kv.pull(key, out=out, ignore_sparse=False)
    return out.indices.asnumpy(), out.data.asnumpy()


def check_retain(out, ids, dense):
    """row_sparse_pull result: the ascending unique ids requested, the table's rows for them"""
    u = np.unique(np.asarray(ids).astype(np.int64))
    got = out.indices.asnumpy()
    assert got.dtype == np.int64 and np.array_equal(got, u)
    assert eq(out.data.asnumpy().reshape((u.size,) + dense.shape[1:]), dense[u])


# ------------------------------------------------------------------------------------------------
# 1. scan-block and word edges: one and two scan blocks, and a bitmap of 64 blocks
@pytest.mark.parametrize("nsrc", E.SCAN_NSRC)
@pytest.mark.parametrize("rows", E.scan_tables())
def test_scan_block_edges(mx, oracle, union_path, rows, nsrc):
    rng = np.random.default_rng(rows + 31 * nsrc)
    shape = (rows, 4)
    edge = np.array(E.scan_edge_ids(rows), np.int64)
    kv = mx.kv.create('device')
    kv.init(0, mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0)))
    shared = rng.integers(0, rows, 16)     # in every source: sums of nsrc terms
    idxs, vals = [], []
    for s in range(nsrc):
        # the first source holds every edge id, the others about half of them; all hold random ids
        pick = edge if s == 0 else edge[rng.random(edge.size) < 0.5]
        i = np.unique(np.concatenate([pick, shared, rng.integers(0, rows, 200)]))
        idxs.append(i)
        vals.append(mixed_vals(rng, i.size, shape[1]))
    kv.push(0, [rsp(mx, i, v, shape) for i, v in zip(idxs, vals)])
    want_idx, want_val = oracle.rsp_reduce(idxs, vals)
    assert np.array_equal(want_idx, np.unique(np.concatenate(idxs)))
    if nsrc >= 3:
        check_order_sensitive(idxs, vals, want_idx, want_val)
    got_idx, got_val = whole_value(mx, kv, 0, shape)
    assert np.array_equal(got_idx, want_idx)
    assert eq(got_val, want_val)
    dense = np.zeros(shape, np.float32)
    dense[want_idx] = want_val
    # a full row_sparse_pull, then the edge ids unsorted with duplicates
    out = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
    kv.row_sparse_pull(0, out=out, row_ids=ids_nd(mx, np.arange(rows)))
    check_retain(out, np.arange(rows), dense)
    req = rng.permutation(np.concatenate([edge, edge[::2], rng.integers(0, rows, 50)]))
    out = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
    kv.row_sparse_pull(0, out=out, row_ids=ids_nd(mx, req))
    check_retain(out, req, dense)


# ------------------------------------------------------------------------------------------------
# 2. every source count a push takes, and the refusal of one more
@pytest.mark.parametrize("row_len", E.NSRC_ROW_LENS)
@pytest.mark.parametrize("nsrc", E.NSRC_ALL)
def test_every_source_count(mx, oracle, union_path, nsrc, row_len):
    rng = np.random.default_rng(100 * nsrc + row_len)
    rows = 3000
    shape = (rows, row_len)
    common = np.array([0, 5, 1234, rows - 1])      # in every source
    first_only, last_only = np.array([7, 2000]), np.array([8, 2001])
    others = np.setdiff1d(np.arange(rows), np.concatenate([common, first_only, last_only]))
    idxs, vals = [], []
    for s in range(nsrc):
        parts = [common, rng.choice(others, 150, replace=False)]
        if s == 0:
            parts.append(first_only)
        if s == nsrc - 1:
            parts.append(last_only)
        i = np.unique(np.concatenate(parts))
        idxs.append(i)
        vals.append(mixed_vals(rng, i.size, row_len))
    kv = mx.kv.create('device')
    kv.init(0, mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0)))
    kv.push(0, [rsp(mx, i, v, shape) for i, v in zip(idxs, vals)])
    want_idx, want_val = oracle.rsp_reduce(idxs, vals)
    if nsrc >= 2:
        # the first and the last source both change the rows every source holds
        pc = np.searchsorted(want_idx, common)
        for drop in (0, nsrc - 1):
            part = fp32_sum(idxs, vals, want_idx, [s for s in range(nsrc) if s != drop])
            assert not eq(part[pc], want_val[pc]), drop
    if nsrc >= 3:
        check_order_sensitive(idxs, vals, want_idx, want_val)
    got_idx, got_val = whole_value(mx, kv, 0, shape)
    assert np.array_equal(got_idx, want_idx)
    assert eq(got_val, want_val)
    # rows held by one source only carry that source's row
    for only, s in ((first_only, 0), (last_only, nsrc - 1)):
        p = np.searchsorted(want_idx, only)
        assert eq(got_val[p], vals[s][np.searchsorted(idxs[s], only)])


def test_one_source_too_many_is_refused(mx, union_path):
    rng = np.random.default_rng(17)
    shape = (500, 5)
    idx0 = np.sort(rng.choice(shape[0], 40, replace=False))
    val0 = mixed_vals(rng, idx0.size, shape[1])
    kv = mx.kv.create('device')
    kv.init(0, rsp(mx, idx0, val0, shape))
    srcs = []
    for _ in range(E.NSRC_REFUSED):
        i = np.sort(rng.choice(shape[0], 30, replace=False))
        srcs.append(rsp(mx, i, mixed_vals(rng, i.size, shape[1]), shape))
    with pytest.raises(mx.base.MXNetError):
        kv.push(0, srcs)
    got_idx, got_val = whole_value(mx, kv, 0, shape)
    assert np.array_equal(got_idx, idx0) and eq(got_val, val0)
    kv.push(0, srcs[:E.NSRC_REFUSED - 1])     # the store still serves the key
    assert np.array_equal(whole_value(mx, kv, 0, shape)[0],
                          np.unique(np.concatenate([s.indices.asnumpy() for s in srcs[:-1]])))


# ------------------------------------------------------------------------------------------------
# 3. row lengths around the vector tile of the ordered row sum, with and without a fused step
@pytest.mark.parametrize("opt", ["none", "sgd_mom", "adam"])
@pytest.mark.parametrize("row_len", E.tile_row_lens())
def test_row_tiles(mx, oracle, union_path, row_len, opt):
    rng = np.random.default_rng(row_len * 3 + len(opt))
    rows = 48
    shape = (rows, row_len)
    sp = K.scalar_param
    kv = mx.kv.create('device')

    def grads():
        # rows 0..7 are in every source: enough 3-term sums for the order to show at row_len 1
        idxs = [np.union1d(np.arange(8), rng.choice(rows, n, replace=False)) for n in (20, 30, 25)]
        return idxs, [mixed_vals(rng, i.size, row_len) for i in idxs]

    def push(idxs, vals):
        kv.push(0, [rsp(mx, i, v, shape) for i, v in zip(idxs, vals)])
        gi, gv = oracle.rsp_reduce(idxs, vals)
        check_order_sensitive(idxs, vals, gi, gv)
        return gi, gv

    if opt == "none":
        kv.init(0, mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0)))
        gi, gv = push(*grads())
        got_idx, got_val = whole_value(mx, kv, 0, shape)
        assert np.array_equal(got_idx, gi) and eq(got_val, gv)
        return
    w = rng.uniform(0.5, 1.5, shape).astype(np.float32)       # no zero row: the table holds every row
    kv.init(0, rsp(mx, np.arange(rows), w, shape))
    if opt == "sgd_mom":
        kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9, wd=1e-3, rescale_grad=0.5))
    else:
        kv.set_optimizer(mx.optimizer.Adam(learning_rate=1e-3, wd=0.01, rescale_grad=0.5))
    m, v = np.zeros(shape, np.float32), np.zeros(shape, np.float32)
    for t in range(1, 4):
        gi, gv = push(*grads())
        if opt == "sgd_mom":
            oracle.sgd_mom_rsp_update(w, m, gi, gv, sp(0.1), sp(0.9), sp(1e-3), sp(0.5))
        else:
            oracle.adam_rsp_update(w, m, v, gi, gv, sp(K.adam_lr(1e-3, 0.9, 0.999, t)), sp(0.9), sp(0.999),
                                   sp(1e-8), sp(0.01), sp(0.5))
        out = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
        kv.row_sparse_pull(0, out=out, row_ids=ids_nd(mx, np.arange(rows)))
        check_retain(out, np.arange(rows), w)


# ------------------------------------------------------------------------------------------------
# 4. the automatic bitmap -> sort switch of a push and a pull (no environment variable)
@pytest.mark.parametrize("rows", E.switch_tables())
def test_bitmap_to_sort_switch(mx, oracle, monkeypatch, rows):
    monkeypatch.delenv("B200KV_RSP_SORT", raising=False)
    rng = np.random.default_rng(rows % 1000)
    shape = (rows, 1)
    mid = 1 << 22
    hot = np.concatenate([np.arange(0, 40), np.arange(mid - 30, mid + 30), np.arange(rows - 40, rows)])
    idxs = []
    for s in range(3):
        i = hot[rng.random(hot.size) < 0.6]
        idxs.append(np.unique(np.concatenate([i, [0, mid, rows - 1]])))
    vals = [mixed_vals(rng, i.size, 1) for i in idxs]
    gi, gv = oracle.rsp_reduce(idxs, vals)
    check_order_sensitive(idxs, vals, gi, gv)
    req = rng.permutation(np.concatenate([np.arange(rows - 64, rows), np.arange(rows - 64, rows, 3),
                                          np.arange(mid - 8, mid + 8), [0]]))
    # the merged value
    kv = mx.kv.create('device')
    kv.init(0, mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0)))
    kv.push(0, [rsp(mx, i, v, shape) for i, v in zip(idxs, vals)])
    got_idx, got_val = whole_value(mx, kv, 0, shape)
    assert np.array_equal(got_idx, gi) and eq(got_val, gv)
    out = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
    kv.row_sparse_pull(0, out=out, row_ids=ids_nd(mx, req))
    u = np.unique(req)
    ri, rv = oracle.sparse_retain(gi, gv, u)
    assert np.array_equal(out.indices.asnumpy(), ri) and eq(out.data.asnumpy(), rv)
    # a fused lazy SGD step on a table that holds every row
    w = rng.uniform(0.5, 1.5, shape).astype(np.float32)
    kv = mx.kv.create('device')
    kv.init(0, rsp(mx, np.arange(rows), w, shape))
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, wd=1e-3, rescale_grad=0.5))
    kv.push(0, [rsp(mx, i, v, shape) for i, v in zip(idxs, vals)])
    sp = K.scalar_param
    oracle.sgd_rsp_update(w, gi, gv, sp(0.1), sp(1e-3), sp(0.5))
    out = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
    kv.row_sparse_pull(0, out=out, row_ids=ids_nd(mx, req))
    check_retain(out, req, w)


# ------------------------------------------------------------------------------------------------
# 5. many (key, out, row_ids) triples in one row_sparse_pull, all on one GPU
@pytest.mark.parametrize("max_rows,nitems", E.many_items_counts())
def test_many_item_pull(mx, union_path, max_rows, nitems):
    rng = np.random.default_rng(nitems)
    # (rows, row_len, stored rows or None for every row): different heights, so that the id space
    # of the call is the tallest table's; values that hold every row next to a few rows
    tables = [(max_rows, 4, None), (max_rows, 3, 300), (max_rows // 16 + 3, 8, None), (17, 5, 4)]
    kv = mx.kv.create('device')
    dense = []
    for k, (rows, row_len, nnr) in enumerate(tables):
        idx = np.arange(rows) if nnr is None else np.sort(rng.choice(rows, nnr, replace=False))
        val = rng.uniform(0.5, 1.5, (idx.size, row_len)).astype(np.float32)
        kv.init(k, rsp(mx, idx, val, (rows, row_len)))
        d = np.zeros((rows, row_len), np.float32)
        d[idx] = val
        dense.append(d)
    empty_at = {3, nitems // 2, nitems + 2}    # triples with no ids: settled without a kernel
    keys, outs, ids = [], [], []
    for t in range(nitems + len(empty_at)):
        k = t % len(tables) if t % 7 else 0    # several triples on every key, most on key 0
        rows = tables[k][0]
        if t in empty_at:
            r = np.zeros(0, np.int64)
        else:
            r = rng.integers(0, rows, int(rng.integers(1, 12)))
            r = np.concatenate([r, r[:2], [rows - 1] if t % 5 == 0 else []]).astype(np.int64)
            r = rng.permutation(r)
        keys.append(k)
        ids.append(r)
        outs.append(mx.nd.sparse.zeros('row_sparse', tables[k][:2], mx.gpu(0)))
    assert sum(1 for r in ids if r.size) == nitems
    kv.row_sparse_pull(keys, out=outs, row_ids=[ids_nd(mx, r) for r in ids])
    for k, o, r in zip(keys, outs, ids):
        check_retain(o, r, dense[k])


# ------------------------------------------------------------------------------------------------
# 6. every id dtype row_sparse_pull reads, with ids each dtype represents exactly
ID_DTYPE_CASES = [
    (128, [np.int64, np.int32, np.float32, np.float64, np.float16, np.uint8, np.int8]),
    (2049, [np.int64, np.int32, np.float32, np.float64, np.float16]),
    (32 * E.SCAN_BLOCK_ROWS + 1, [np.int64, np.int32, np.float32, np.float64]),
]


@pytest.mark.parametrize("rows,dtypes", ID_DTYPE_CASES, ids=[str(c[0]) for c in ID_DTYPE_CASES])
def test_id_dtypes(mx, union_path, rows, dtypes):
    rng = np.random.default_rng(rows)
    shape = (rows, 3)
    idx = np.sort(rng.choice(rows, rows // 2, replace=False))
    val = rng.uniform(0.5, 1.5, (idx.size, 3)).astype(np.float32)
    kv = mx.kv.create('device')
    kv.init(0, rsp(mx, idx, val, shape))
    dense = np.zeros(shape, np.float32)
    dense[idx] = val
    req = rng.permutation(np.concatenate([rng.integers(0, rows, 60), [0, 0, 31, 32, 33, rows - 1, rows - 1]]))
    results = []
    for dt in dtypes:
        assert np.array_equal(req.astype(dt).astype(np.int64), req), dt   # exact in this dtype
        out = mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0))
        kv.row_sparse_pull(0, out=out, row_ids=ids_nd(mx, req, dt))
        check_retain(out, req, dense)
        results.append((out.indices.asnumpy(), out.data.asnumpy()))
    for (i, d), dt in zip(results[1:], dtypes[1:]):
        assert np.array_equal(i, results[0][0]) and eq(d, results[0][1]), dt


# ------------------------------------------------------------------------------------------------
# 7. whole-value pulls (rsp_broadcast_kernel): 16-, 4- and 1-byte units, kMaxDst targets of each kind
def _bcast_cases():
    out = []
    for rows in E.BCAST_TABLES:
        # (dtype, row_len): the unit is the widest of 16 / 4 / 1 bytes that divides the row's bytes
        layouts = [(np.float32, 4), (np.float32, 5), (np.float16, 3)]
        if rows < 8:
            layouts += [(np.float32, 516), (np.float32, 129), (np.float16, 65)]   # 97+ units per row
        for dt, row_len in layouts:
            for fill in ("none", "some", "all"):
                if fill == "some" and rows == 1:
                    continue
                out.append((rows, dt, row_len, fill))
    return out


@pytest.mark.parametrize("rows,dtype,row_len,fill", _bcast_cases(),
                         ids=["%d-%s-%d-%s" % (r, np.dtype(d).name, n, f) for r, d, n, f in _bcast_cases()])
def test_whole_value_pull(mx, rows, dtype, row_len, fill):
    rng = np.random.default_rng(rows + row_len)
    shape = (rows, row_len)
    nnr = {"none": 0, "some": max(1, min(rows // 2, 3000)), "all": rows}[fill]
    idx = np.sort(rng.choice(rows, nnr, replace=False)) if fill == "some" else np.arange(nnr)
    val = rng.uniform(-2, 2, (nnr, row_len)).astype(dtype)
    kv = mx.kv.create('device')
    kv.init(0, rsp(mx, idx, val, shape, dtype) if nnr else mx.nd.sparse.zeros('row_sparse', shape, mx.gpu(0), dtype))
    want = np.zeros(shape, dtype)
    want[idx] = val
    ndst = E.BCAST_DST
    junk = rng.uniform(5, 6, shape).astype(dtype)                  # stale rows in every target
    for interleave in (True, False):
        rsp_outs = [rsp(mx, np.arange(rows), junk, shape, dtype) for _ in range(ndst)]
        # dense targets are float32 only (storage casts); they start from a non-zero pattern
        dns_outs = [mx.nd.array(junk, mx.gpu(0)) for _ in range(ndst)] if dtype == np.float32 else []
        outs = rsp_outs + dns_outs
        if interleave and dns_outs:
            outs = [o for pair in zip(rsp_outs, dns_outs) for o in pair]
        kv.pull(0, out=outs, ignore_sparse=False)
        for o in rsp_outs:
            assert np.array_equal(o.indices.asnumpy(), idx)
            assert eq(o.data.asnumpy().reshape(nnr, row_len), val)
        for o in dns_outs:
            assert eq(o.asnumpy(), want)
