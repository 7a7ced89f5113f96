"""The front end makes each of its per-column and per-argument decisions in one place: whether a block is device memory, how a
column is read, a column's dtype, how a selection mask is unmasked and how a selection argument is resolved (vaex_b200/_lib.py,
vaex_b200/frame.py).  The scans below keep the copies from coming back; the unit tests pin what the shared helpers answer."""
import ast
import os
import re
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "vaex_b200")


def sources():
    for name in sorted(os.listdir(PKG)):
        if name.endswith(".py"):
            yield name, open(os.path.join(PKG, name)).read()


def calls_of(tree, callee):
    """the names of the functions (innermost def) that call `callee(...)`, once per call"""
    out = []

    def visit(node, fn):
        for child in ast.iter_child_nodes(node):
            if isinstance(child, (ast.FunctionDef, ast.AsyncFunctionDef)):
                visit(child, child.name)
                continue
            if isinstance(child, ast.Call) and isinstance(child.func, ast.Name) and child.func.id == callee:
                out.append(fn)
            visit(child, fn)
    visit(tree, None)
    return out


def test_device_test_lives_only_in_lib():
    spelled = re.compile(r"hasattr\(\s*\w+\s*,\s*[\"']__cuda_array_interface__[\"']\s*\)\s*and\s+not\s+isinstance\(\s*\w+\s*,\s*np\.ndarray\s*\)")
    found = {name: (bool(re.search(r"\bdef _?is_device\b", text)), len(spelled.findall(text))) for name, text in sources()}
    assert found["_lib.py"] == (True, 1), found["_lib.py"]
    stray = {name: f for name, f in found.items() if name != "_lib.py" and f != (False, 0)}
    assert not stray, stray


def test_selection_masks_unmasked_in_one_function():
    pattern = re.compile(r"\.data\s*&\s*~\s*np\.ma\.getmaskarray")
    hits = [(name, line.strip()) for name, text in sources() for line in text.split("\n") if pattern.search(line)]
    assert len(hits) == 1 and hits[0][0] == "_lib.py", hits
    tree = ast.parse(dict(sources())["_lib.py"])
    holder = [fn.name for fn in ast.walk(tree) if isinstance(fn, ast.FunctionDef) and pattern.search(ast.get_source_segment(dict(sources())["_lib.py"], fn))]
    assert holder == ["unmask_selection"], holder


def test_selection_message_written_once():
    count = sum(text.count("a selection must be a boolean expression") for _, text in sources())
    assert count == 1, count


def test_frames_derived_in_one_method():
    texts = dict(sources())
    assert calls_of(ast.parse(texts["frame.py"]), "Frame") == ["_derive"]
    # extract and the join result build frames without categories or filter on purpose
    assert set(calls_of(ast.parse(texts["join.py"]), "Frame")) == {"extract", "join"}
    others = {name: calls_of(ast.parse(text), "Frame") for name, text in texts.items() if name not in ("frame.py", "join.py")}
    assert not any(others.values()), others


def test_one_task_part_for_the_count_grid_finishes():
    tree = ast.parse(dict(sources())["taskpart.py"])
    subclasses = [c.name for c in tree.body if isinstance(c, ast.ClassDef) and any(getattr(b, "id", None) == "TaskPartAggregation" for b in c.bases)]
    assert subclasses == ["TaskPartCountGrid"], subclasses


# ---- the helpers ----------------------------------------------------------------------------------------------------------------
class FakeDevice:
    """an array that only exposes __cuda_array_interface__, like a torch CUDA tensor does"""

    def __init__(self, dtype, n=4):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": np.dtype(dtype).str, "data": (0, False), "version": 3, "strides": None}
        self.n = n

    def __len__(self):
        return self.n


class FakeVirtual:
    device_virtual = True
    dtype = np.dtype("int64")

    def __init__(self, *inputs):
        self.columns = list(inputs)
        self.seen = []

    def chunk(self, thread_index, i1, i2):
        self.seen.append((thread_index, i1, i2))
        return np.arange(i1, i2)


def test_is_device():
    from vaex_b200 import _lib
    assert _lib.is_device(FakeDevice("f4"))
    assert not _lib.is_device(np.zeros(3))
    assert not _lib.is_device(np.ma.zeros(3))
    assert not _lib.is_device([1, 2])


def test_unmask_selection():
    from vaex_b200 import _lib
    sel = np.ma.array([True, True, False, True], mask=[False, True, True, False])
    out = _lib.unmask_selection(sel)
    assert not np.ma.isMaskedArray(out) and out.tolist() == [True, False, False, True]
    assert _lib.unmask_selection(np.array([True, False])).tolist() == [True, False]
    dev = FakeDevice("?")
    assert _lib.unmask_selection(dev) is dev


def test_rows_of_a_chunk():
    from vaex_b200.taskpart import _rows
    assert _rows(10, 25, None, [np.zeros(15)]) == 15
    assert _rows(10, 25, None, []) == 15
    mask = np.array([1, 0, 1, 1], np.uint8)
    assert _rows(0, 4, mask, [np.zeros(3)]) == 3   # compacted blocks carry the kept length
    assert _rows(0, 4, mask, []) == 3              # count(*) without blocks: the mask's own count
    kept = types.SimpleNamespace(kept=2)            # the executor's device filter mask records what it kept
    assert _rows(0, 4, kept, []) == 2


def test_split_mask():
    from vaex_b200 import _lib
    m = np.ma.array(np.arange(8.0)[::2], mask=[0, 1, 0, 0])
    data, mask = _lib.split_mask(m)
    assert type(data) is np.ndarray and data.flags.c_contiguous and data.tolist() == [0.0, 2.0, 4.0, 6.0]
    assert mask.tolist() == [False, True, False, False]
    plain = np.arange(3)
    assert _lib.split_mask(plain)[0] is plain and _lib.split_mask(plain)[1] is None
    dev = FakeDevice("i4")
    assert _lib.split_mask(dev) == (dev, None)


def test_device_rule_and_chunks_of_virtual_columns():
    from vaex_b200 import _lib
    assert _lib.on_device(FakeDevice("f4")) and not _lib.on_device(np.zeros(2))
    assert _lib.on_device(FakeVirtual(FakeDevice("f4"), FakeDevice("i8")))
    assert not _lib.on_device(FakeVirtual(FakeDevice("f4"), np.zeros(4)))
    assert _lib.on_device(FakeVirtual())  # no inputs (a constant expression): the executor feeds it as one device pass
    v = FakeVirtual(np.zeros(4))
    assert _lib.chunk_of(v, 3, 1, 4).tolist() == [1, 2, 3] and v.seen == [(3, 1, 4)]
    assert _lib.chunk_of(np.arange(5), 3, 1, 4).tolist() == [1, 2, 3]


def test_join_materializes_a_virtual_column_without_inputs_on_the_host():
    """the join's exception to the device rule: a virtual column without inputs comes back as host values"""
    from vaex_b200 import join
    col = FakeVirtual()
    frame = types.SimpleNamespace(columns={"c": col}, evaluate=lambda name: np.arange(3))
    values = join._materialize(frame, "c")
    assert isinstance(values, np.ndarray) and values.tolist() == [0, 1, 2]
    frame.columns["c"] = FakeVirtual(np.zeros(3))
    assert isinstance(join._materialize(frame, "c"), np.ndarray)


def test_dtype_of():
    import pyarrow as pa
    from vaex_b200 import _lib
    assert _lib.dtype_of(np.arange(3, dtype="i2")) == np.dtype("i2")
    assert _lib.dtype_of(np.ma.array(np.zeros(2, ">f8"), mask=[0, 1])) == np.dtype(">f8")
    assert _lib.dtype_of(FakeDevice("u1")) == np.dtype("u1")
    assert _lib.dtype_of(FakeVirtual(np.zeros(3))) == np.dtype("int64")
    assert _lib.dtype_of(np.array(["a", "b"])) == np.dtype("O")
    assert _lib.dtype_of(pa.array(["a", None])) == np.dtype("O")
    assert _lib.dtype_of(np.array(["2020-01-01"], dtype="M8[s]")) == np.dtype("M8[s]")


def test_device_expressions_do_not_read_arrow_columns():
    """an arrow column has no numpy dtype in a device expression, numeric or not"""
    import pyarrow as pa
    from vaex_b200.expression import DeviceExpression
    assert DeviceExpression("x + 1", {"x": np.arange(3)}).dtype == np.int64
    for col in (pa.array([1, 2, 3]), pa.array(["a", "b", "c"]), np.array(["a", "b", "c"])):
        with pytest.raises(NotImplementedError, match="not supported in device expressions"):
            DeviceExpression("x + 1", {"x": col})


def test_binned_args():
    from vaex_b200.frame import _binned_args
    assert _binned_args(None, 128, None) == ([], [], [])
    assert _binned_args("x", 64, None) == (["x"], [64], [None])
    assert _binned_args("x", 64, [0, 1]) == (["x"], [64], [[0, 1]])
    assert _binned_args(["x", "y"], 8, "minmax") == (["x", "y"], [8, 8], [None, None])
    assert _binned_args(["x", "y"], 8, "90%") == (["x", "y"], [8, 8], [None, None])  # a string means minmax on these paths
    assert _binned_args(("x", "y"), [4, 5], [[0, 1], None]) == (["x", "y"], [4, 5], [[0, 1], None])
    spec = {"binner-type": "hash"}
    assert _binned_args(spec, 8, None) == ([spec], [8], [None])


def test_selection_resolver():
    from vaex_b200.frame import Frame

    class Stub:
        _selection = Frame._selection

        def expression(self, text):
            return types.SimpleNamespace(text=text, dtype=np.dtype("?") if "<" in text else np.dtype("f8"))
    f = Stub()
    assert f._selection(None) is None
    assert f._selection(False) is None
    assert f._selection("x < 1").text == "x < 1"
    mask = np.array([True, False])
    assert f._selection(mask) is mask
    out = f._selection([None, False, "x < 1", mask])
    assert out[:2] == [None, None] and out[2].text == "x < 1" and out[3] is mask
    with pytest.raises(ValueError, match="a selection must be a boolean expression"):
        f._selection("x + 1")
    with pytest.raises(ValueError, match="a selection must be a boolean expression"):
        f._selection([None, "x + 1"])
