"""Every device block of the library outside the per-slot arenas comes from the context's cache through one owning handle
(DevBuf, vaex_b200/csrc/common.cuh): the raw CUDA allocator is called only by the cache and the arenas, and only the handle
gives a block back."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vaex_b200", "csrc")

# the cache itself (ctx_alloc / ctx_release) and the per-slot arenas, which keep their own grow-with-sync policy
RAW_ALLOWED = {"ctx_alloc", "ctx_release", "slot_reserve", "slot_scratch", "b200_ctx_create", "b200_ctx_destroy"}


def sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh")):
            text = open(os.path.join(CSRC, name)).read()
            text = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), text, flags=re.S)
            yield name, [re.sub(r"//.*", "", line) for line in text.split("\n")]


def enclosing_function(lines, i):
    """name of the function whose definition starts at column 0 most recently before line i"""
    for line in reversed(lines[:i + 1]):
        m = re.match(r"[A-Za-z_][\w:<>,\s\*&]*?\b(\w+)\s*\(.*", line)
        if m and not line.rstrip().endswith(";"):
            return m.group(1)
    return None


def test_raw_allocator_only_in_cache_and_arenas():
    found = []
    for name, lines in sources():
        for i, line in enumerate(lines):
            if re.search(r"\bcuda(Malloc|Free)(Async)?\s*\(", line):
                found.append((name, i + 1, enclosing_function(lines, i)))
    assert found, "the scan found no allocator call at all"
    stray = [f for f in found if f[2] not in RAW_ALLOWED]
    assert not stray, stray


def test_ctx_release_only_in_the_handle():
    calls = []
    for name, lines in sources():
        for i, line in enumerate(lines):
            if re.search(r"\bctx_release\s*\(", line):
                calls.append((name, line.strip()))
    # the declaration and the handle's call in common.cuh, the definition in api.cu
    assert sorted(n for n, _ in calls) == ["api.cu", "common.cuh", "common.cuh"], calls
    assert any(n == "common.cuh" and "ctx_release(ctx_, ptr_, bytes_)" in l for n, l in calls), calls
