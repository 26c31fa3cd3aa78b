"""TEST INFRASTRUCTURE ONLY -- the size thresholds at which the row_sparse union, retain and
broadcast kernels (anand_mxnet_b200/csrc/rowsparse_kernels.cu) change path, read from their source,
and the test shapes that put a case on both sides of each of them.

Importers: tests/test_rowsparse_edges_gpu.py (runs the shapes) and tests/test_rowsparse_edges_host.py
(checks, without a GPU, that the constants are found and that every threshold is straddled). When a
constant is retuned the shapes follow it instead of silently testing the interior.
"""
import os
import re

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(_ROOT, "anand_mxnet_b200", "csrc")

# name -> (file, C type of the declaration)
_DECLS = {
    "kScanThreads": ("rowsparse_kernels.cu", "int"),
    "kBitmapMaxWords": ("rowsparse_kernels.cu", "int64_t"),
    "kBitmapMaxTotalWords": ("rowsparse_kernels.cu", "int64_t"),
    "kBmMaxItems": ("rowsparse_kernels.cu", "int"),
    "kMaxSrc": ("kernels.h", "int"),
    "kMaxDst": ("kernels.h", "int"),
    "kWarpsPerBlock": ("rowsparse_kernels.cu", "int"),
    "kNumSMs": ("common.h", "int"),
}


def _eval_int(expr):
    """the integer value of a constexpr initialiser such as `1024` or `int64_t{1} << 18`"""
    e = re.sub(r"int64_t\{(\d+)\}", r"\1", expr)
    if not re.fullmatch(r"[\d\s()<*+-]+", e):
        raise ValueError("not a plain integer expression: %r" % expr)
    return int(eval(e, {"__builtins__": {}}))


def read_constants(csrc=CSRC):
    """{name: value} for every constant in _DECLS, plus the row tile of the ordered row sum (`U`
    float4 per lane and step in rsp_sum_row). Raises if a declaration is missing or appears twice."""
    out = {}
    texts = {}
    for name, (fname, ctype) in _DECLS.items():
        if fname not in texts:
            with open(os.path.join(csrc, fname)) as f:
                texts[fname] = f.read()
        pat = r"constexpr\s+%s\s+%s\s*=\s*([^;]+);" % (re.escape(ctype), name)
        found = re.findall(pat, texts[fname])
        if len(found) != 1:
            raise LookupError("%s: %d declarations of %s %s" % (fname, len(found), ctype, name))
        out[name] = _eval_int(found[0])
    body = texts["rowsparse_kernels.cu"].split("rsp_sum_row(", 1)[1].split("\n}\n", 1)[0]
    found = re.findall(r"constexpr\s+int\s+U\s*=\s*(\d+)\s*;", body)
    if len(found) != 1:
        raise LookupError("rsp_sum_row: %d declarations of its unroll U" % len(found))
    out["U"] = int(found[0])
    return out


C = read_constants()

# one scan block ranks kScanThreads bitmap words of 32 rows each
SCAN_BLOCK_ROWS = C["kScanThreads"] * 32
# the ordered row sum walks a row in tiles of U x 32 lanes x 4 floats; the vector path needs row_len % 4 == 0
ROW_TILE = C["U"] * 32 * 4


def id_bits(rows):
    """BitsFor in rowsparse.cc: the bits that hold every id in [0, rows)"""
    b = 1
    while b < 62 and (1 << b) < rows:
        b += 1
    return b


def bitmap_words(rows):
    """words of the bitmap of one push / pull item over a table of `rows` rows: it spans 2**id_bits"""
    return ((1 << id_bits(rows)) + 31) // 32


def push_uses_bitmap(rows):
    return bitmap_words(rows) <= C["kBitmapMaxWords"]


def pull_uses_bitmap(max_rows, nitems):
    """nitems: the (key, out, row_ids) triples of one owner GPU that request at least one id"""
    w = bitmap_words(max_rows)
    return nitems <= C["kBmMaxItems"] and w <= C["kBitmapMaxWords"] and w * nitems <= C["kBitmapMaxTotalWords"]


# ---- case 1: scan-block and word edges
def scan_tables():
    """one scan block, exactly one, one row over it (a second block), and a table whose bitmap spans
    64 blocks"""
    b = SCAN_BLOCK_ROWS
    return [b - 1, b, b + 1, 32 * b + 1]


def scan_edge_ids(rows):
    """ids where a word, a scan block or the table ends, and their neighbours, inside [0, rows)"""
    b = SCAN_BLOCK_ROWS
    ids = {0, 31, 32, 33, b - 1, b, rows - 1}
    for m in range(1, rows // b + 1):
        ids.update((m * b - 1, m * b, m * b + 1))
    return sorted(i for i in ids if 0 <= i < rows)


SCAN_NSRC = [1, 2, 5]

# ---- case 2: every source count
NSRC_ALL = list(range(1, C["kMaxSrc"] + 1))
NSRC_REFUSED = C["kMaxSrc"] + 1
NSRC_ROW_LENS = [4, 5]   # vector and scalar row paths

# ---- case 3: row lengths around the vector tile
def tile_row_lens():
    t, q = ROW_TILE, ROW_TILE // 4
    return [1, 3, 4, q - 1, q, q + 1, t - 1, t, t + 1, 2 * t + 4]


# ---- case 4: the automatic bitmap -> sort switch of a push and a pull
def switch_tables():
    top = C["kBitmapMaxWords"] * 32
    return [top, top + 1]


# ---- case 5: many-item pulls
def many_items_small_rows():
    """the largest table (a power of two) on which one more item than kBmMaxItems still keeps
    items x words within kBitmapMaxTotalWords: there the item count alone decides the path"""
    w = 1
    while (C["kBmMaxItems"] + 1) * (2 * w) <= C["kBitmapMaxTotalWords"]:
        w *= 2
    return 32 * w


def many_items_counts():
    """(largest table rows, non-empty triples) for the item-count edge and the total-words edge"""
    small = many_items_small_rows()
    big = 1 << 20
    n_total = C["kBitmapMaxTotalWords"] // bitmap_words(big)
    return [(small, C["kBmMaxItems"]), (small, C["kBmMaxItems"] + 1), (big, n_total), (big, n_total + 1)]


# ---- case 7: whole-value pulls
BCAST_DST = C["kMaxDst"]
# rsp_broadcast_kernel's grid holds at most kNumSMs * 8 blocks of kWarpsPerBlock warps; each warp
# walks ceil(domain / warps) rows
BCAST_MAX_WARPS = C["kNumSMs"] * 8 * C["kWarpsPerBlock"]
BCAST_TABLES = [1, 2, 32 * SCAN_BLOCK_ROWS + 1]
