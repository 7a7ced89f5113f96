"""Every per-slot library call reads the caller's memory, places its results and decides when to return through one frame
(CallFrame, vaex_b200/csrc/common.cuh); on the Python side one function (_lib.memspace) decides a call's memspace."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "vaex_b200", "csrc")
PKG = os.path.join(ROOT, "vaex_b200")

ENTRY_POINTS = {"b200_bin", "b200_eval", "b200_compact", "b200_minmax", "b200_stat_bin", "b200_grid_percentile", "b200_grid_mutual_information",
                "b200_set_update", "set_map_common", "b200_set_combine", "b200_set_from_keys", "b200_set_merge", "b200_strset_update",
                "b200_strset_map_ordinal"}


def sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh")):
            text = open(os.path.join(CSRC, name)).read()
            text = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), text, flags=re.S)
            yield name, [re.sub(r"//.*", "", line) for line in text.split("\n")]


def functions(lines):
    """(qualified name of the function whose definition starts at column 0, its lines) for every such definition"""
    out, name, body = [], None, []
    for line in lines:
        m = re.match(r"(?=[A-Za-z_])(?:[^(;]*?[\s*&])?((?:\w+::)*~?\w+)\s*\(", line)
        if m and not line.rstrip().endswith(";"):
            if name:
                out.append((name, body))
            name, body = m.group(1), []
        if name:
            body.append(line)
    if name:
        out.append((name, body))
    return out


def test_memspace_decided_only_by_the_frame():
    compare = re.compile(r"\bmemspace_?\s*(==|!=|<=|>=|<|>)\s*B200_MEM_|B200_MEM_\w+\s*(==|!=|<=|>=|<|>)\s*memspace_?\b")
    found, stray = 0, []
    for name, lines in sources():
        for fn, body in functions(lines):
            for line in body:
                if compare.search(line) or re.search(r"\bis_device_pointer\s*\(", line):
                    found += 1
                    if not (fn.startswith("CallFrame::") or fn == "is_device_pointer" or name == "strings.cuh"):
                        stray.append((name, fn, line.strip()))
    assert found, "the scan found no memspace decision at all"
    assert not stray, stray


def test_frame_built_only_in_the_entry_points_and_always_finished():
    built = {}
    for name, lines in sources():
        assert not any(re.search(r"\bStager\b", line) for line in lines), name
        for fn, body in functions(lines):
            text = "\n".join(body)
            if re.search(r"\bCallFrame\s+\w+\s*\(", text):
                built[fn] = text
    assert set(built) == ENTRY_POINTS, sorted(set(built) ^ ENTRY_POINTS)
    unfinished = [fn for fn, text in built.items() if not re.search(r"\.finish\(", text)]
    assert not unfinished, unfinished


def test_mixed_memspace_decided_only_in_lib():
    users = sorted(f for f in os.listdir(PKG) if f.endswith(".py") and re.search(r"\bMEM_MIXED\b", open(os.path.join(PKG, f)).read()))
    assert users == ["_lib.py"], users


def test_memspace_of_columns():
    from vaex_b200 import _lib

    class Col:
        def __init__(self, memspace):
            self.memspace = memspace
    H, D = Col(_lib.MEM_HOST), Col(_lib.MEM_DEVICE)
    assert _lib.memspace() == _lib.MEM_HOST
    assert _lib.memspace(None) == _lib.MEM_HOST
    assert _lib.memspace(H, None, H) == _lib.MEM_HOST
    assert _lib.memspace(D, D, None) == _lib.MEM_DEVICE
    assert _lib.memspace(H, D) == _lib.MEM_MIXED
    assert _lib.memspace(D, None, H) == _lib.MEM_MIXED
