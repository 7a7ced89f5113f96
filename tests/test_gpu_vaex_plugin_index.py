"""vaex_plugin.install(index_hash=True) / uninstall() against a stub vaex that restates the pieces they touch: vaex.cpu's task-part
registry and vaex.hash.index_type_from_dtype.  The index handed out is then driven like vaex/join.py drives it (host lookups)."""
import sys
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture()
def stub_vaex(monkeypatch):
    vaex = types.ModuleType("vaex")
    cpu = types.ModuleType("vaex.cpu")
    registry = {}

    def register(cls):
        registry[cls.snake_name] = cls
        return cls

    class TaskPartAggregation:
        snake_name = "aggregations"

    class TaskPartHashmapUniqueCreate:
        snake_name = "hash_map_unique_create"
    cpu.register, cpu.registry = register, registry
    cpu.TaskPartAggregation, cpu.TaskPartHashmapUniqueCreate = register(TaskPartAggregation), register(TaskPartHashmapUniqueCreate)
    hash_mod = types.ModuleType("vaex.hash")

    class index_hash_string:
        pass

    def index_type_from_dtype(dtype, transient=True, prime_growth=False):
        if str(dtype) in ("string", "str", "<U0") or getattr(dtype, "kind", "") in "OU":
            return index_hash_string
        raise AssertionError("numeric dtypes go to the device classes")
    hash_mod.index_type_from_dtype = index_type_from_dtype
    hash_mod.index_hash_string = index_hash_string
    vaex.cpu, vaex.hash = cpu, hash_mod
    for name, mod in (("vaex", vaex), ("vaex.cpu", cpu), ("vaex.hash", hash_mod)):
        monkeypatch.setitem(sys.modules, name, mod)
    return vaex


def test_install_index_hash_and_uninstall(stub_vaex):
    from vaex_b200 import superutils, vaex_plugin
    original = stub_vaex.hash.index_type_from_dtype
    vaex_plugin.install(index_hash=True)
    try:
        lookup_type = stub_vaex.hash.index_type_from_dtype
        assert lookup_type(np.dtype("int32")) is superutils.index_hash_int32
        assert lookup_type(np.dtype("datetime64[ns]")) is superutils.index_hash_int64
        assert lookup_type(np.dtype("O")) is stub_vaex.hash.index_hash_string
        # join.py:168-209 with one thread: index the right, host lookup of the left, duplicates
        index = lookup_type(np.dtype("int64"))(1)
        index.update(np.array([4, 7, 4, 9]), 0)
        lookup = np.full(5, np.iinfo(np.int8).max, np.int8)
        unknown = index.map_index(np.array([9, 4, 1, 7, 4]), lookup)
        assert unknown and lookup.tolist() == [3, 0, -1, 1, 0]
        left, right = index.map_index_duplicates(np.array([9, 4, 1, 7, 4]), 0)
        assert left.tolist() == [1, 4] and right.tolist() == [2, 2]
    finally:
        vaex_plugin.uninstall()
    assert stub_vaex.hash.index_type_from_dtype is original
