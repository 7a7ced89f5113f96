"""Named selections without a device (vaex_b200/selections.py, Frame.select*): histories, undo / redo and the clipping of the redo
tail, every mode with and without a previous selection (the compiled programs run by tests/expr_oracle.py), to_dict round trips, the
exact text of box, circle and ellipse held to numpy evaluating the reference's text, and the resolution of names and its errors."""
import numpy as np
import pytest

import expr_oracle
import lasso_oracle as L
from vaex_b200 import selections as S
from vaex_b200.frame import Frame


def host_mask(df, selection=True):
    """a resolved selection evaluated on the host: the host masks, the lassos by the restatement, the programs by expr_oracle"""
    sel = df._selection(selection)
    return run(df, sel)


def run(df, sel):
    if not isinstance(sel, S.SelectionMask):
        return expr_oracle.run(sel.program, df.columns).astype(bool)
    values = {}
    for name, sub in sel.named:
        values[name] = run(df, sub)
    for name, fn, col in sel.host_masks:
        values[name] = np.asarray(fn(col), bool)
    for name, lasso in sel.lassos:
        xy = [expr_oracle.run(expr.program, cols) for expr, cols in (lasso.x, lasso.y)]
        p = lasso.plan
        assert not p.banded  # the plain plan keeps the vertices in order
        values[name] = L.pnpoly(*p.edges[:, :2].T, *xy, p.meanx, p.meany, p.radius)
    out = None
    for name, expr, cols in sel.programs:
        assert S._fits(expr), expr.program.expression  # every program within b200_eval's 8 inputs, 64 ops and stack of 12
        out = values[name] = expr_oracle.run(expr.program, {**cols, **values}).astype(bool)
    return out


X = np.arange(10.0)


def df10():
    return Frame({"x": X, "y": X ** 2})


def test_history_undo_redo_and_clipping():
    df = df10()
    assert not df.has_selection() and not df.selection_can_undo() and not df.selection_can_redo()
    df.select_nothing()
    assert not df.has_selection() and not df.selection_can_undo() and not df.selection_can_redo()
    df.select("x > 5")
    assert df.has_selection() and df.selection_can_undo() and not df.selection_can_redo()
    df.select("x < 7", mode="and")
    df.selection_undo()
    assert df.get_selection().boolean_expression == "x > 5" and df.selection_can_redo()
    df.selection_undo()
    assert not df.has_selection() and not df.selection_can_undo() and df.selection_can_redo()
    df.selection_redo()
    df.select("x < 3", mode="or")  # clips the redo tail
    assert not df.selection_can_redo() and len(df.selection_histories["default"]) == 2
    df.select_nothing()
    assert not df.has_selection() and df.selection_can_undo()
    assert df.selection_histories["default"][-1] is None
    df.selection_undo()
    assert df.has_selection() and df.selection_can_redo()
    with pytest.raises(ValueError):
        Frame({"x": X}).selection_undo()


def test_current_entry_after_undoing_everything_is_the_last():
    """with the index at -1 the reference's `current` is history[-1]: a new and-selection combines with the last entry"""
    df = df10()
    df.select("x > 5")
    df.select("x > 7")
    df.selection_undo()
    df.selection_undo()
    df.select("x < 9", mode="and")
    assert df.get_selection().previous_selection.boolean_expression == "x > 7"
    assert host_mask(df).tolist() == ((X > 7) & (X < 9)).tolist()


@pytest.mark.parametrize("mode", ["replace", "and", "or", "xor", "subtract"])
def test_modes(mode):
    df = df10()
    df.select("x > 5", mode=mode)  # no previous selection: the current mask as it is, subtract included
    assert host_mask(df).tolist() == (X > 5).tolist()
    df.select("x < 8", mode=mode)
    want = S._select_functions[mode](X > 5, X < 8)
    assert host_mask(df).tolist() == np.asarray(want).tolist()


def test_invert_and_names():
    df = df10()
    with pytest.raises(ValueError):
        df.select_inverse()
    assert not df.selection_histories.get("default")
    df.select("x > 5")
    df.select_inverse()
    assert host_mask(df).tolist() == (X <= 5).tolist()
    df.select("x < 2", name="low")
    assert host_mask(df, "default | low").tolist() == ((X <= 5) | (X < 2)).tolist()
    sels = df._selection(["default", "low", "default"])
    assert sels[0] is sels[2]


def test_column_wins_and_cycles():
    df = Frame({"x": X, "default": X > 100})
    df.select("x > 5")
    assert host_mask(df, "default").tolist() == [False] * 10
    df = df10()
    df.select("x > 1", name="a")
    df.select("a & (x < 5)", name="b")
    with pytest.raises(ValueError, match="refers to itself"):
        df.select("b | (x > 8)", name="a")
    assert df.get_selection("a").boolean_expression == "x > 1"
    with pytest.raises(KeyError, match="default"):
        df._selection(True)
    with pytest.raises(ValueError, match="a selection must be a boolean expression"):
        df.select("x + 1")
    assert not df.selection_histories.get("default")


def test_to_dict_round_trip():
    e = S.SelectionExpression("x > 5", None, "and")
    lasso = S.SelectionLasso("x", "y", np.array([0, 10, 10, 0]), [-1, -1, 100, 100], e, "and")
    inv = S.SelectionInvert(lasso)
    drop = S.SelectionDropNa(True, False, ["x"], inv, "or")
    d = drop.to_dict()
    assert S.selection_from_dict(d).to_dict() == d
    assert d["previous_selection"]["previous_selection"]["xseq"] == [0, 10, 10, 0]
    assert S.SelectionExpression("x > 5", e, "replace").previous_selection is None
    with pytest.raises(ValueError):
        S.selection_from_dict({"type": "nope", "previous_selection": None})


def test_geometric_text():
    assert S.box_text(["x", "y"], [(1.2345678, -0.5), (-1, 2)]) == "((x) >= -0.500000) & ((x) <= 1.234568)&((y) >= -1.000000) & ((y) <= 2.000000)"
    t = S.circle_text("x", "y", 2, -3.5, 1.5)
    assert t.reference == "((((x - 2) ** 2) + ((y - -3.5) ** 2)) <= 2.25)"
    assert t.device == "((((x - 2) * (x - 2)) + ((y - -3.5) * (y - -3.5))) <= 2.25)"
    t = S.ellipse_text("x", "y", 2, -1, 5, 1, 30, inclusive=False)
    c, s = np.cos(np.deg2rad(30)), np.sin(np.deg2rad(30))
    assert t.reference == (f"(((((((x - 2) * {c}) + ((y - -1) * {s})) ** 2) / 1.0) + (((((x - 2) * {s}) - ((y - -1) * {c})) ** 2) / "
                           f"{(0.5 / 2.5) ** 2})) < 6.25)")
    rng = np.random.default_rng(0)
    for dtype in ("f8", "f4", "i8"):
        cols = {"x": (rng.standard_normal(500) * 3).astype(dtype), "y": (rng.standard_normal(500) * 3).astype(dtype)}
        for t in (S.circle_text("x", "y", 0.5, -1, 2), S.ellipse_text("x", "y", 2, -1, 5, 1, 30), S.ellipse_text("x", "y", 0, 0, 2, 6, 100, inclusive=False)):
            with np.errstate(all="ignore"):
                want = eval(t.reference, dict(cols))
            assert np.array_equal(expr_oracle.evaluate(t.device, cols).astype(bool), want)


def test_compiled_programs_and_split():
    df = Frame({f"c{k}": np.arange(10.0) - k for k in range(12)})
    for k in range(12):
        df.select(f"c{k} > -3", mode="and")
    sel = df._selection(True)
    assert len(sel.programs) >= 2
    assert all(len(e.program.inputs) <= 8 for _, e, _ in sel.programs)
    want = np.all([df.columns[f"c{k}"] > -3 for k in range(12)], axis=0)
    assert host_mask(df).tolist() == want.tolist()
    df = df10()
    df.select("x > 2")
    df.select("x < 6", mode="xor")
    df.select_inverse()
    (_, expr, _), = df._selection(True).programs
    assert expr.program.expression == "~((x > 2) != (x < 6))"


def test_masked_inputs_refused_in_expressions():
    df = Frame({"m": np.ma.array(X, mask=X > 7), "y": X})
    with pytest.raises(NotImplementedError, match="masked"):
        df.select("m > 2")
    df.select_lasso("m", "y", [0, 9, 9, 0], [-1, -1, 100, 100])
    sel = df._selection(True)
    assert len(sel.lassos) == 1 and len(sel.host_masks) == 1
    assert host_mask(df).tolist() == (L.lasso([0, 9, 9, 0], [-1, -1, 100, 100], df.columns["m"], X)).tolist()
    df.select_non_missing()
    assert len(df._selection(True).host_masks) == 1


def test_select_non_missing_over_many_columns():
    """every real column by default: more terms than one program reads, packed into several"""
    rng = np.random.default_rng(1)
    cols = {f"f{k}": np.where(rng.random(200) < 0.03, np.nan, rng.standard_normal(200)) for k in range(12)}
    cols["m"] = np.ma.array(rng.standard_normal(200), mask=rng.random(200) < 0.05)
    cols["o"] = np.array([None if v < 0.05 else "s" for v in rng.random(200)], dtype=object)
    df = Frame(cols)
    df.select_non_missing()
    sel = df._selection(True)
    assert len(sel.programs) >= 2
    want = np.ones(200, bool)
    for k in range(12):
        want &= ~np.isnan(cols[f"f{k}"])
    want &= ~np.ma.getmaskarray(cols["m"]) & np.array([v is not None for v in cols["o"]])
    assert host_mask(df).tolist() == want.tolist()


def test_full_step_after_a_previous_selection():
    """an 8-column expression combined with a previous selection: the combination reads 9 inputs and is split"""
    rng = np.random.default_rng(2)
    cols = {f"c{k}": rng.standard_normal(100) for k in range(9)}
    df = Frame(cols)
    df.select("c8 > 0")
    eight = " & ".join(f"(c{k} > -1)" for k in range(8))
    df.select(eight, mode="and")
    want = cols["c8"] > 0
    for k in range(8):
        want &= cols[f"c{k}"] > -1
    assert host_mask(df).tolist() == want.tolist()
    df.select_lasso("c0", "c1", [-1, 1, 1, -1], [-1, -1, 1, 1], mode="or")
    want = want | L.lasso([-1, 1, 1, -1], [-1, -1, 1, 1], cols["c0"], cols["c1"])
    assert host_mask(df).tolist() == want.tolist()


def test_expression_over_too_many_columns_is_refused_when_made():
    df = Frame({f"c{k}": np.arange(5.0) for k in range(9)})
    with pytest.raises(NotImplementedError, match="at most 8 inputs"):
        df.select(" & ".join(f"(c{k} > 1)" for k in range(9)))
    assert not df.has_selection()


def test_big_endian_columns_are_not_copied():
    """a column in the other byte order is typed through a zero-length placeholder; its chunks are swapped when read"""
    x = np.arange(20.0).astype(">f8")
    df = Frame({"x": x, "y": np.arange(20.0), "unused": np.arange(20.0).astype(">f8")})
    df.select_non_missing(column_names=["x"])
    df.select_lasso("x", "y", [2, 8, 8, 2], [0, 0, 30, 30], mode="and")
    sel = df._selection(True)
    kept = [c for _, _, cols in sel.programs for c in cols.values()] + [c for _, lasso in sel.lassos for _, cols in (lasso.x, lasso.y) for c in cols.values()]
    assert all(c.size == 0 or c is df.columns[k] for c, k in zip(kept, [k for _, _, cols in sel.programs for k in cols] +
                                                                    [k for _, lasso in sel.lassos for _, cols in (lasso.x, lasso.y) for k in cols]))
    assert host_mask(df).tolist() == L.lasso([2, 8, 8, 2], [0, 0, 30, 30], x.astype("f8"), np.arange(20.0)).tolist()
