"""The engine's dependency protocol in the host sources, without a GPU. An operation on one lane
declares its arrays once through LaneOp (csrc/ndarray.h), which takes each array's wait and mark from
the same list. Direct BeginRead / BeginWrite / MarkRead / MarkWrite / Engine::Issue calls remain only
where one operation spans several lanes. Zero-filled arrays come from ZerosOn, so a recycled pool
block always gets its first-writer wait."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "anand_mxnet_b200", "csrc")

# Engine::Issue(sid) takes the lane; LaneOp::Issue() takes nothing
ENGINE_CALL = re.compile(r"\b(?:BeginRead|BeginWrite|MarkRead|MarkWrite)\(|->Issue\((?!\s*\))")
ZERO_FILL = re.compile(r"cudaMemsetAsync\([^;]*ByteSize\(\)")

# (file, function) -> direct engine calls
DIRECT = {
    # the dense step: one kernel per owner GPU, dependencies on every participating lane
    ("dense_exec.cc", "KVStore::RunPrepared"): 12,
    # the pack table is uploaded on the compute lane and read on a copy lane
    ("dense_exec.cc", "BuildPackList"): 1,
    # row_sparse sources are read on their own GPUs' lanes
    ("rowsparse.cc", "KVStore::PushRowSparse"): 3,
}
ZERO_FILLS = {("ndarray.cc", "ZerosOn"): 1, ("rowsparse.cc", "CastStorageCopy"): 1}


def strip(src):
    """Comments and string / char literals blanked, offsets kept."""
    pat = re.compile(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', re.S)
    return pat.sub(lambda m: re.sub(r"[^\n]", " ", m.group(0)), src)


def blocks(src):
    """(name, start, end) of every brace block opened at namespace scope: the function it defines,
    or None for a struct / class body."""
    out, stack, head = [], [], 0  # stack: (is_namespace, start, name)
    for i, ch in enumerate(src):
        at_ns = all(s[0] for s in stack)
        if ch == "{":
            name = None
            if at_ns:
                text = src[head:i]
                if re.search(r"\bnamespace\b[^;{}]*$", text):
                    stack.append((True, i, None))
                    head = i + 1
                    continue
                while re.search(r"<[^<>]*>", text):  # std::function<void()> F(...)
                    text = re.sub(r"<[^<>]*>", "", text)
                m = re.search(r"([A-Za-z_][\w:]*)\s*\(", text)
                name = m.group(1) if m else None
            stack.append((False, i, name))
        elif ch == "}":
            ns, start, name = stack.pop()
            if all(s[0] for s in stack):
                if not ns:
                    out.append((name, start, i))
                head = i + 1
        elif ch == ";" and at_ns:
            head = i + 1
    return out


def count(pattern, skip):
    found = {}
    for f in sorted(os.listdir(CSRC)):
        if not f.endswith((".cc", ".h")) or f in skip:
            continue
        with open(os.path.join(CSRC, f)) as fh:
            src = strip(fh.read())
        spans = blocks(src)
        for m in pattern.finditer(src):
            where = [b for b in spans if b[1] <= m.start() <= b[2]]
            name = (where[0][0] or "<class body>") if where else "<namespace scope>"
            if f == "ndarray.cc" and name.startswith("LaneOp::"):
                continue  # the protocol's one implementation
            found[(f, name)] = found.get((f, name), 0) + 1
    return found


def test_scanner_names_functions():
    with open(os.path.join(CSRC, "rowsparse.cc")) as fh:
        names = {b[0] for b in blocks(strip(fh.read()))}
    assert {"KVStore::PushRowSparse", "KVStore::PullRowSparseGroup", "CastStorageCopy",
            "KVStore::PushRowSparseGroup", "RankSources", None} <= names


def test_single_lane_operations_go_through_laneop():
    assert count(ENGINE_CALL, skip={"engine.cc", "engine.h"}) == DIRECT


def test_zero_fills_go_through_zeroson():
    assert count(ZERO_FILL, skip=set()) == ZERO_FILLS
