"""Without a GPU: the thresholds of the row_sparse kernels are found in their source, and the shapes
tests/test_rowsparse_edges_gpu.py runs put a case at or below every threshold and one above it.
Without this check the shapes could drift into the interior of a path and test nothing."""
import os

import pytest

import rsp_edges as E


def test_every_constant_is_found():
    c = E.read_constants()
    assert set(c) == {"kScanThreads", "kBitmapMaxWords", "kBitmapMaxTotalWords", "kBmMaxItems", "kMaxSrc",
                      "kMaxDst", "kWarpsPerBlock", "kNumSMs", "U"}
    assert all(isinstance(v, int) and v > 0 for v in c.values()), c


def test_missing_or_odd_constant_is_an_error(tmp_path):
    for name in ("rowsparse_kernels.cu", "kernels.h", "common.h"):
        with open(os.path.join(E.CSRC, name)) as f:
            (tmp_path / name).write_text(f.read())
    src = (tmp_path / "rowsparse_kernels.cu").read_text()
    (tmp_path / "rowsparse_kernels.cu").write_text(src.replace("constexpr int kBmMaxItems", "constexpr int kBmMaxItemz"))
    with pytest.raises(LookupError):
        E.read_constants(str(tmp_path))
    (tmp_path / "rowsparse_kernels.cu").write_text(src.replace("int64_t{1} << 22", "kSomething << 22"))
    with pytest.raises(ValueError):
        E.read_constants(str(tmp_path))


def test_id_bits_matches_bits_for():
    assert [E.id_bits(n) for n in (1, 2, 3, 32768, 32769, 1 << 23, (1 << 23) + 1)] == [1, 1, 2, 15, 16, 23, 24]


def straddles(values, edge):
    return min(values) <= edge < max(values)


def test_scan_block_edge():
    words = [E.bitmap_words(r) for r in E.scan_tables()]
    assert straddles(words, E.C["kScanThreads"])                  # one scan block, then two
    assert max(words) // E.C["kScanThreads"] >= 64                # the last-CTA fold over many blocks
    for rows in E.scan_tables():
        ids = E.scan_edge_ids(rows)
        assert ids[0] == 0 and ids[-1] == rows - 1 and all(0 <= i < rows for i in ids)
        blocks = {i // E.SCAN_BLOCK_ROWS for i in ids}
        assert len(blocks) == (rows - 1) // E.SCAN_BLOCK_ROWS + 1   # every block of the table holds an id
        for m in range(1, (rows - 1) // E.SCAN_BLOCK_ROWS + 1):
            assert {m * E.SCAN_BLOCK_ROWS - 1, m * E.SCAN_BLOCK_ROWS} <= set(ids)
    assert {31, 32} <= set(E.scan_edge_ids(E.scan_tables()[0]))   # a word boundary


def test_source_count_edge():
    assert E.NSRC_ALL == list(range(1, E.C["kMaxSrc"] + 1))
    assert E.NSRC_REFUSED == E.C["kMaxSrc"] + 1
    assert any(r % 4 == 0 for r in E.NSRC_ROW_LENS) and any(r % 4 for r in E.NSRC_ROW_LENS)


def test_row_tile_edges():
    lens = E.tile_row_lens()
    assert E.ROW_TILE == E.C["U"] * 32 * 4
    for edge in (4, E.ROW_TILE // 4, E.ROW_TILE, 2 * E.ROW_TILE):
        assert straddles(lens, edge), edge
    # a vector row of more than one tile, and one that ends inside the third tile
    assert any(r % 4 == 0 and r > E.ROW_TILE for r in lens)
    assert any(r % 4 == 0 and r > 2 * E.ROW_TILE for r in lens)
    assert any(r % 4 for r in lens) and any(r % 4 == 0 for r in lens)


def test_bitmap_switch_edge():
    below, above = E.switch_tables()
    assert E.bitmap_words(below) <= E.C["kBitmapMaxWords"] < E.bitmap_words(above)
    assert E.push_uses_bitmap(below) and not E.push_uses_bitmap(above)
    assert E.pull_uses_bitmap(below, 1) and not E.pull_uses_bitmap(above, 1)


def test_many_item_edges():
    cases = E.many_items_counts()
    (rows_a, n0), (rows_b, n1), (rows_c, n2), (rows_d, n3) = cases
    # the item count alone changes: both sides stay within the total-words budget
    assert rows_a == rows_b and n0 == E.C["kBmMaxItems"] and n1 == n0 + 1
    assert E.bitmap_words(rows_a) * n1 <= E.C["kBitmapMaxTotalWords"]
    assert E.pull_uses_bitmap(rows_a, n0) and not E.pull_uses_bitmap(rows_a, n1)
    # the total-words budget alone changes: both item counts stay within kBmMaxItems
    assert rows_c == rows_d and n3 == n2 + 1 and n3 <= E.C["kBmMaxItems"]
    assert E.bitmap_words(rows_c) * n2 <= E.C["kBitmapMaxTotalWords"] < E.bitmap_words(rows_c) * n3
    assert E.pull_uses_bitmap(rows_c, n2) and not E.pull_uses_bitmap(rows_c, n3)


def test_broadcast_edges():
    assert E.BCAST_DST == E.C["kMaxDst"]
    # tables with fewer rows than one block has warps, and one with more rows than the grid has
    # warps that they do not divide: its last warp walks a shorter range
    assert min(E.BCAST_TABLES) < E.C["kWarpsPerBlock"]
    big = max(E.BCAST_TABLES)
    assert big > E.BCAST_MAX_WARPS and big % E.BCAST_MAX_WARPS != 0
