"""Named selections: vaex's selection objects (vaex/selections.py) and their evaluation on the device.

A frame keeps one history per selection name (Frame.select, select_box, select_lasso, ...).  A history entry is one of the
objects below; each holds the entry before it (`previous_selection`) unless its mode is "replace", and combines its own mask with
the previous one by its mode, exactly as the reference's `evaluate` does.  Here an entry is never evaluated on the host: when a
statistic resolves `selection=` (Frame._selection), `resolve` turns the chain into one device object shaped like
expression.DeviceExpression (SelectionMask: `device_virtual`, `dtype`, `columns`, `__len__`, `chunk`), so the executor and every task
part treat it as any other boolean column.

The chain compiles into b200_eval programs with the existing opcodes: & for and, | for or, != for xor, & ~ for subtract, ~ for
invert, `x != x` for NaN; the mask of a masked column, an arrow column's nulls, an object column's None and a lasso's answer
(b200_lasso, csrc/lasso.cu) enter as bool inputs.  A chain that reads more than b200_eval's 8 inputs is cut into several programs,
each reading the previous program's mask.  Names of other selections inside an expression are looked up when the selection is
resolved, not when it is made, as vaex's _BlockScope does; a column of the same name wins.
"""
import ast
import threading

import numpy as np

from . import _lib

# ---- the reference's mode functions (vaex/selections.py:11-36), on host masks -----------------------------------------------------
def _select_replace(maskold, masknew):
    return masknew


def _select_and(maskold, masknew):
    return masknew if maskold is None else np.asarray(maskold) & np.asarray(masknew)


def _select_or(maskold, masknew):
    return masknew if maskold is None else np.asarray(maskold) | np.asarray(masknew)


def _select_xor(maskold, masknew):
    return masknew if maskold is None else np.asarray(maskold) ^ np.asarray(masknew)


def _select_subtract(maskold, masknew):
    return ~masknew if maskold is None else np.asarray(maskold) & ~np.asarray(masknew)


_select_functions = {"replace": _select_replace, "and": _select_and, "or": _select_or, "xor": _select_xor, "subtract": _select_subtract}

# the same combinations as expression text over bool operands, for the device programs
_COMBINE = {"and": "({0}) & ({1})", "or": "({0}) | ({1})", "xor": "({0}) != ({1})", "subtract": "({0}) & ~({1})"}


# ---- the selection objects (vaex/selections.py:38-231) -----------------------------------------------------------------------------
class Selection:
    def __init__(self, previous_selection, mode):
        # the previous selection is dropped only when the mode replaces it
        self.previous_selection = previous_selection if mode != "replace" else None
        self.mode = mode

    def _previous_dict(self):
        return self.previous_selection.to_dict() if self.previous_selection else None


class SelectionDropNa(Selection):
    def __init__(self, drop_nan, drop_masked, expressions, previous_selection, mode):
        super().__init__(previous_selection, mode)
        self.drop_nan = drop_nan
        self.drop_masked = drop_masked
        self.expressions = expressions

    def to_dict(self):
        return dict(type="dropna", drop_nan=self.drop_nan, drop_masked=self.drop_masked, expressions=self.expressions, mode=self.mode,
                    previous_selection=self._previous_dict())


class SelectionExpression(Selection):
    def __init__(self, boolean_expression, previous_selection, mode):
        super().__init__(previous_selection, mode)
        self.boolean_expression = str(boolean_expression)
        self.expressions = [self.boolean_expression]

    def to_dict(self):
        return dict(type="expression", boolean_expression=str(self.boolean_expression), mode=self.mode, previous_selection=self._previous_dict())


class SelectionInvert(Selection):
    def __init__(self, previous_selection):
        super().__init__(previous_selection, "")
        self.expressions = []

    def to_dict(self):
        return dict(type="invert", previous_selection=self._previous_dict())


class SelectionLasso(Selection):
    def __init__(self, boolean_expression_x, boolean_expression_y, xseq, yseq, previous_selection, mode):
        super().__init__(previous_selection, mode)
        self.boolean_expression_x = boolean_expression_x
        self.boolean_expression_y = boolean_expression_y
        self.xseq = xseq
        self.yseq = yseq
        self.expressions = [boolean_expression_x, boolean_expression_y]

    def to_dict(self):
        return dict(type="lasso", boolean_expression_x=str(self.boolean_expression_x), boolean_expression_y=str(self.boolean_expression_y),
                    xseq=_make_list(self.xseq), yseq=_make_list(self.yseq), mode=self.mode, previous_selection=self._previous_dict())


def _make_list(seq):
    """vaex.utils.make_list"""
    return seq.tolist() if hasattr(seq, "tolist") else list(seq)


def selection_from_dict(values):
    kwargs = dict(values)
    del kwargs["type"]
    kinds = {"lasso": SelectionLasso, "expression": SelectionExpression, "invert": SelectionInvert, "dropna": SelectionDropNa}
    if values["type"] not in kinds:
        raise ValueError("unknown type: %r, in dict: %r" % (values["type"], values))
    kwargs["previous_selection"] = selection_from_dict(values["previous_selection"]) if values["previous_selection"] else None
    return kinds[values["type"]](**kwargs)


# ---- the geometric selections' expression text ---------------------------------------------------------------------------------
class Text:
    """an expression built the way vaex's Expression operators build theirs ('({0} {1} {2})'.format(a, op, b), str() of a
    constant), kept twice: `reference` with the reference's `** 2`, `device` with the square written as a product, which is what
    numpy computes for `ndarray ** 2` (np.square) and what the device compiler accepts"""

    def __init__(self, reference, device=None):
        self.reference, self.device = reference, reference if device is None else device

    def _op(self, code, other, reverse=False):
        a, b = (self, other) if not reverse else (other, self)
        ref = lambda v: v.reference if isinstance(v, Text) else v  # noqa: E731
        dev = lambda v: v.device if isinstance(v, Text) else v  # noqa: E731
        return Text("({0} {1} {2})".format(ref(a), code, ref(b)), "({0} {1} {2})".format(dev(a), code, dev(b)))

    def __add__(self, other):
        return self._op("+", other)

    def __sub__(self, other):
        return self._op("-", other)

    def __mul__(self, other):
        return self._op("*", other)

    def __truediv__(self, other):
        return self._op("/", other)

    def __le__(self, other):
        return self._op("<=", other)

    def __lt__(self, other):
        return self._op("<", other)

    def __pow__(self, power):
        if power != 2:
            raise NotImplementedError("only squares")
        return Text("({0} ** 2)".format(self.reference), "({0} * {0})".format(self.device))


def box_text(spaces, limits):
    """select_box's expression (vaex/dataframe.py:5170-5173): %f rounds every limit to 6 decimals"""
    sorted_limits = [(min(lim), max(lim)) for lim in limits]
    return "&".join("((%s) >= %f) & ((%s) <= %f)" % (e, lmin, e, lmax) for e, (lmin, lmax) in zip(spaces, sorted_limits))


def circle_text(x, y, xc, yc, r, inclusive=True):
    """select_circle's expression (vaex/dataframe.py:5194-5197) as a Text"""
    X, Y = Text(str(x)), Text(str(y))
    lhs = (X - xc) ** 2 + (Y - yc) ** 2
    return lhs <= r ** 2 if inclusive else lhs < r ** 2


def ellipse_text(x, y, xc, yc, width, height, angle=0, radians=False, inclusive=True):
    """select_ellipse's expression (vaex/dataframe.py:5225-5240) as a Text; the constants are the reference's (np.deg2rad, np.cos,
    np.sin on the host, xr / r, r**2 in Python).  With radians=True the angle is taken as radians (the reference leaves alpha unset
    and fails)."""
    alpha = angle if radians else np.deg2rad(angle)
    xr = width / 2
    yr = height / 2
    r = max(xr, yr)
    a = xr / r
    b = yr / r
    X, Y = Text(str(x)), Text(str(y))
    lhs = ((X - xc) * np.cos(alpha) + (Y - yc) * np.sin(alpha)) ** 2 / a ** 2 + ((X - xc) * np.sin(alpha) - (Y - yc) * np.cos(alpha)) ** 2 / b ** 2
    return lhs <= r ** 2 if inclusive else lhs < r ** 2


# ---- the lasso's polygon, staged for b200_lasso ----------------------------------------------------------------------------------
# the vertex count from which the banded loop is used (DESIGN.md §4)
LASSO_BAND_MIN_VERTICES = 64
_MAX_ENTRIES_PER_EDGE = 32


def lasso_constants(xseq, yseq):
    """the polygon as float64 and meanx, meany, radius exactly as SelectionLasso.evaluate computes them (vaex/selections.py:178-181)"""
    x, y = np.array(xseq, dtype=np.float64), np.array(yseq, dtype=np.float64)
    with np.errstate(all="ignore"):
        meanx = x.mean()
        meany = y.mean()
        radius = np.sqrt((meanx - x) ** 2 + (meany - y) ** 2).max()
    return x, y, float(meanx), float(meany), float(radius)


def band_of(v, lo, scale, nbands):
    """the band b200_lasso reads for a row of y = v (lo <= v < hi): the same IEEE operations, so the host lists each edge in every
    band a row it can toggle maps to"""
    with np.errstate(all="ignore"):
        t = (np.asarray(v, dtype=np.float64) - lo) * scale
    t = np.where(np.isnan(t), 0.0, t)
    return np.clip(np.trunc(np.clip(t, -1.0, float(nbands))), 0, nbands - 1).astype(np.int64)


class LassoPlan:
    """the edges b200_lasso tests: (x_i, y_i, x_j, y_j) for j = i - 1 in the reference's order (plain loop), or sorted into y bands
    (banded loop, from LASSO_BAND_MIN_VERTICES vertices on)"""

    def __init__(self, xseq, yseq, banded=None):
        x, y, self.meanx, self.meany, self.radius = lasso_constants(xseq, yseq)
        n = len(x)
        j = np.roll(np.arange(n), 1)
        edges = np.stack([x, y, x[j], y[j]], axis=1) if n else np.zeros((0, 4))
        self.banded = n >= LASSO_BAND_MIN_VERTICES if banded is None else bool(banded)
        self.nbands, self.lo, self.hi, self.scale = 0, 0.0, 0.0, 0.0
        self.band_start = None
        if not self.banded or n == 0:
            self.banded = False
            self.edges = np.ascontiguousarray(edges)
            return
        ylo, yhi = np.minimum(y, y[j]), np.maximum(y, y[j])
        if not np.all(np.isfinite(y)):
            # a NaN or infinite vertex: one band over every y, every edge in it
            nbands, lo, hi, scale = 1, -np.inf, np.inf, 0.0
            b0 = b1 = np.zeros(n, np.int64)
        else:
            lo, hi = float(y.min()), float(y.max())
            nbands = n
            while True:
                with np.errstate(all="ignore"):
                    scale = float(np.float64(nbands) / np.float64(hi - lo)) if hi > lo else 0.0
                if not np.isfinite(scale):
                    nbands, scale = 1, 0.0
                b0, b1 = band_of(ylo, lo, scale, nbands), band_of(yhi, lo, scale, nbands)
                if nbands == 1 or int((b1 - b0 + 1).sum()) <= _MAX_ENTRIES_PER_EDGE * n:
                    break
                nbands = max(1, nbands // 2)
        reps = b1 - b0 + 1
        total = int(reps.sum())
        edge_ids = np.repeat(np.arange(n), reps)
        first = np.repeat(np.cumsum(reps) - reps, reps)
        band_ids = np.repeat(b0, reps) + (np.arange(total) - first)
        order = np.argsort(band_ids, kind="stable")
        self.edges = np.ascontiguousarray(edges[edge_ids[order]])
        self.band_start = np.searchsorted(band_ids[order], np.arange(nbands + 1)).astype(np.int32)
        self.nbands, self.lo, self.hi, self.scale = nbands, float(lo), float(hi), float(scale)

    def band_edges(self, b):
        """the edges band b lists (tests)"""
        return self.edges[self.band_start[b]:self.band_start[b + 1]]


class _Lasso:
    """one lasso of a resolved selection: x and y as float64 device blocks, the polygon staged once per resolution"""

    def __init__(self, plan, x, y):
        self.plan, self.x, self.y = plan, x, y
        self._staged = None
        self._lock = threading.Lock()
        self._buffers = {}

    def _stage(self, ctx):
        import torch
        with self._lock:
            if self._staged is None:
                device = f"cuda:{ctx.device}"
                edges = torch.from_numpy(self.plan.edges.reshape(-1)).to(device) if len(self.plan.edges) else None
                bands = torch.from_numpy(self.plan.band_start).to(device) if self.plan.banded else None
                torch.cuda.synchronize(device)  # every slot's stream reads the polygon
                self._staged = (edges, bands)
        return self._staged

    def chunk(self, thread_index, i1, i2):
        import torch
        from .expression import DeviceArray
        ctx = _lib.context()
        n = int(i2 - i1)
        buf = self._buffers.get(thread_index)
        if buf is None or buf.numel() < max(n, 1):
            buf = self._buffers[thread_index] = torch.empty(max(n, 1) + 16, dtype=torch.uint8, device=f"cuda:{ctx.device}")
        if n:
            edges, bands = self._stage(ctx)
            x, y = (_lib.column(_float64_block(src, thread_index, i1, i2)) for src in (self.x, self.y))
            p = self.plan
            _lib.check(_lib.lib().b200_lasso(ctx._h, ctx.slot(thread_index), x.ptr, y.ptr, n, None if edges is None else edges.data_ptr(), len(p.edges),
                                              None if bands is None else bands.data_ptr(), p.nbands, p.lo, p.hi, p.scale, p.meanx, p.meany, p.radius,
                                              buf.data_ptr()))
        return DeviceArray(buf.data_ptr(), n, np.bool_, keep=buf)


def _float64_block(src, thread_index, i1, i2):
    """a native float64 device column is passed as it is; anything else is (program, columns): its (expr).astype('float64') program
    over the columns' rows"""
    if isinstance(src, tuple):
        expr, cols = src
        return expr.run(thread_index, i1, i2, [cols[k][i1:i2] for k in expr.program.inputs])
    return src[i1:i2]


# ---- resolution: a selection chain -> one device object ------------------------------------------------------------------------
_MAX_INPUTS, _MAX_OPS, _MAX_STACK = 8, 64, 12  # b200_eval's limits (csrc/expr.cu)


def _stack_depth(ops):
    from . import expression as X
    depth = top = 0
    for op in ops:
        if op[0] in (X.EX_INPUT, X.EX_CONST_F64, X.EX_CONST_I64):
            depth += 1
        elif op[0] not in (X.EX_NEG, X.EX_ABS, X.EX_SQRT, X.EX_NOT, X.EX_CAST, X.EX_ORDINAL):
            depth -= 1
        top = max(top, depth)
    return top


def _fits(expr):
    p = expr.program
    return len(p.inputs) + len(p.strcalls) <= _MAX_INPUTS and len(p.ops) <= _MAX_OPS and _stack_depth(p.ops) <= _MAX_STACK


class SelectionMask:
    """a resolved selection, evaluated chunk by chunk on the worker's slot like a DeviceExpression: first the named selections it
    reads, the host masks and the lassos, then its programs in order; the last program's output is the mask"""

    device_virtual = True
    dtype = np.dtype(np.bool_)

    def __init__(self, length):
        self.length = length
        self.columns = []     # every array read, for the executor's host / device decision
        self.named = []       # (input name, SelectionMask)
        self.host_masks = []  # (input name, function of a block -> bool array, column)
        self.lassos = []      # (input name, _Lasso)
        self.programs = []    # (input name of its output, DeviceExpression, {column name: array})

    def __len__(self):
        return self.length

    def _read(self, col):
        if not any(col is c for c in self.columns):
            self.columns.append(col)

    def chunk(self, thread_index, i1, i2):
        values = {}
        for name, sub in self.named:
            values[name] = sub.chunk(thread_index, i1, i2)
        for name, fn, col in self.host_masks:
            values[name] = np.ascontiguousarray(fn(col[i1:i2]), dtype=np.bool_)
        for name, lasso in self.lassos:
            values[name] = lasso.chunk(thread_index, i1, i2)
        out = None
        for name, expr, cols in self.programs:
            parts = [values[k] if k in values else cols[k][i1:i2] for k in expr.program.inputs]
            out = values[name] = expr.run(thread_index, i1, i2, parts)
        return out

    def evaluate(self, i1=0, i2=None, thread_index=0):
        """host copy of the mask (tests)"""
        i2 = self.length if i2 is None else i2
        return self.chunk(thread_index, i1, i2).to_numpy()


def _names(text):
    return {n.id for n in ast.walk(ast.parse(text, mode="eval")) if isinstance(n, ast.Name)}


def _is_masked(col):
    return isinstance(col, np.ndarray) and np.ma.isMaskedArray(col)


def _is_arrow(col):
    return type(col).__module__.startswith("pyarrow")


def _missing_fn(col):
    """the host function that gives a block's missing rows (vaex.functions.ismissing), or None for a column without any"""
    if _is_masked(col):
        if col.dtype.kind == "O":
            return lambda b: np.asarray(np.equal(b.data, None)) | np.ma.getmaskarray(b)
        return np.ma.getmaskarray
    if _is_arrow(col):
        return lambda b: b.is_null().to_numpy(zero_copy_only=False)
    if isinstance(col, np.ndarray) and col.dtype.kind == "O":
        return lambda b: np.asarray(np.equal(b, None), dtype=np.bool_)
    return None


def _host_nan_fn(col):
    """vaex.functions.isnan of a column the device programs do not read: object values (x != x) and arrow floats (not null)"""
    if isinstance(col, np.ndarray) and not _is_masked(col) and col.dtype.kind == "O":
        return lambda b: np.asarray(np.not_equal(b, b), dtype=np.bool_)
    if _is_arrow(col):
        import pyarrow as pa
        if pa.types.is_floating(col.type):
            return lambda b: np.asarray(b.is_nan().fill_null(False).to_numpy(zero_copy_only=False), dtype=np.bool_)
    return None


class _Resolver:
    """turns one frame's selections into SelectionMask objects; `memo` gives every name one object within a call"""

    def __init__(self, frame, memo):
        self.frame, self.memo = frame, memo
        self.counter = 0

    def fresh(self, kind):
        self.counter += 1
        return f"__selection_{kind}{self.counter}"

    def name(self, name, stack):
        if name in stack:
            raise ValueError(f"selection {name!r} refers to itself: {' -> '.join(list(stack) + [name])}")
        if name not in self.memo:
            selection = self.frame.get_selection(name) if self.frame._has_history(name) else None
            if selection is None:
                raise KeyError(f"no selection named {name!r} on this frame")
            self.memo[name] = self.selection(selection, stack + (name,))
        return self.memo[name]

    def selection(self, selection, stack=()):
        chain = []
        while selection is not None:
            chain.append(selection)
            selection = selection.previous_selection
        out = SelectionMask(self.frame.length)
        text = None
        for step in reversed(chain):
            text = self.step(out, step, text, stack)
        self.finish(out, text)
        return out

    def expression_text(self, out, text, stack):
        """a selection expression with the selections it names as bool inputs, virtual columns expanded"""
        frame = self.frame
        names = {n for n in _names(text) if n not in frame.columns and n not in frame.variables and frame._has_history(n)}
        if names:
            subst = {}
            for n in sorted(names):
                sub = self.name(n, stack)
                key = self.fresh("named")
                out.named.append((key, sub))
                for c in sub.columns:
                    out._read(c)
                subst[n] = key

            class Sub(ast.NodeTransformer):
                def visit_Name(self, node):
                    return ast.copy_location(ast.Name(subst[node.id], node.ctx), node) if node.id in subst else node
            text = ast.unparse(Sub().visit(ast.parse(text, mode="eval")))
        return frame._expand(text)

    def inputs(self, out, extra=()):
        """the columns a program may read: the frame's real columns and the bool inputs made so far (zero-length placeholders give
        the compiler their dtype)"""
        from . import expression as _expr
        cols = {k: v for k, v in self.frame.columns.items() if not isinstance(v, _expr.DeviceExpression)}
        for key in [k for k, _ in out.named] + [k for k, _, _ in out.host_masks] + [k for k, _ in out.lassos] + [k for k, _, _ in out.programs] + list(extra):
            cols[key] = np.zeros(0, np.bool_)
        return cols

    def data_inputs(self, out):
        """the same for typing a program that reads masked columns through their data (only the lasso's coordinates and the NaN
        tests do that): a zero-length placeholder of the native dtype stands for a host column in the other byte order, which the
        compiler cannot type; the chunks themselves are byte-swapped by DeviceExpression.run"""
        return {k: (np.zeros(0, v.dtype.newbyteorder("=")) if isinstance(v, np.ndarray) and not v.dtype.isnative else v)
                for k, v in self.data_columns(out).items()}

    def data_columns(self, out):
        """the columns a program's chunks are read from: masked columns through their data, no copies"""
        return {k: (v.data if _is_masked(v) else v) for k, v in self.inputs(out).items()}

    def host_mask(self, out, fn, col):
        key = self.fresh("mask")
        out.host_masks.append((key, fn, col))
        out._read(col)
        return key

    def step(self, out, step, text, stack):
        from . import expression as _expr
        from .frame import _boolean_selection
        exclude = None
        if isinstance(step, SelectionExpression):
            cur = self.expression_text(out, step.boolean_expression, stack)
            # the expression on its own: a boolean over unmasked columns, or the one refusal every selection gives
            _boolean_selection(_expr.DeviceExpression(cur, self.inputs(out), self.frame.variables))
        elif isinstance(step, SelectionInvert):
            if text is None:
                raise ValueError("select_inverse of no selection")
            return self.join(out, "~({0})", [text])
        elif isinstance(step, SelectionLasso):
            cur, exclude = self.lasso(out, step)
        elif isinstance(step, SelectionDropNa):
            cur = self.dropna(out, step)
        else:
            raise TypeError(f"not a selection: {step!r}")
        combined = self.join(out, "{0}", [cur]) if text is None else self.join(out, _COMBINE.get(step.mode, "{1}"), [text, cur])
        if exclude is not None:  # the lasso's masked rows are dropped after the combine (vaex/selections.py:199-200)
            combined = self.join(out, "({0}) & ~({1})", [combined, self.any_of(out, exclude)])
        return combined

    def fits(self, out, text):
        return _fits(self.compile(out, text))

    def join(self, out, form, parts):
        """form.format(*parts) as a text that one b200_eval program can run: while it reads more than 8 inputs or runs more than 64
        ops, the part that reads the most becomes a program of its own and the text reads that program's mask instead.  A part that
        does not fit on its own is a single expression over too many columns, which program() refuses."""
        parts = list(parts)
        while True:
            text = form.format(*parts)
            if self.fits(out, text):
                return text
            sizes = [(len(e.program.inputs) + len(e.program.strcalls), len(e.program.ops)) for e in (self.compile(out, p) for p in parts)]
            k = max((i for i, p in enumerate(parts) if not (p.isidentifier() and p.startswith("__selection_"))), key=lambda i: sizes[i], default=None)
            if k is None:
                raise RuntimeError(f"the selection program {text!r} does not fit in one b200_eval call")
            parts[k] = self.program(out, parts[k])

    def any_of(self, out, terms):
        """`t1 | t2 | ...` over terms that each fit one program, packed into as few programs as it takes"""
        text = None
        for t in terms:
            text = self.join(out, "{0}", [t]) if text is None else self.join(out, "({0}) | ({1})", [text, t])
        return text

    def compile(self, out, text):
        from . import expression as _expr
        return _expr.DeviceExpression(text, self.data_inputs(out), self.frame.variables)

    def program(self, out, text):
        expr = self.compile(out, text)
        if not _fits(expr):
            p = expr.program
            raise NotImplementedError(f"{text!r} reads {len(p.inputs) + len(p.strcalls)} columns and string calls in {len(p.ops)} operations: one "
                                      f"expression is evaluated by one device program of at most {_MAX_INPUTS} inputs and {_MAX_OPS} operations")
        key = self.fresh("program")
        cols = self.data_columns(out)
        for k in list(expr.program.inputs) + [c for call in expr.program.strcalls for c in call.columns]:
            if not k.startswith("__selection_"):
                out._read(self.frame.columns[k])
        out.programs.append((key, expr, cols))
        return key

    def finish(self, out, text):
        if text is None:
            raise ValueError("an empty selection chain")
        self.program(out, text)

    def lasso(self, out, step):
        from . import expression as _expr
        frame = self.frame
        masks = []
        sources = []
        for e in (step.boolean_expression_x, step.boolean_expression_y):
            e = str(e)
            col = frame.columns.get(e)
            if col is not None and _lib.is_device(col) and _lib.dtype_of(col) == np.float64 and _lib.dtype_of(col).isnative:
                sources.append(col)
                out._read(col)
                continue
            text = frame._expand("(%s).astype('float64')" % e)
            expr = _expr.DeviceExpression(text, self.data_inputs(out), frame.variables)
            for k in expr.program.inputs:
                c = frame.columns[k]
                out._read(c)
                if _is_masked(c) and not any(c is m for m in masks):
                    masks.append(c)
            sources.append((expr, self.data_columns(out)))
        key = self.fresh("lasso")
        out.lassos.append((key, _Lasso(LassoPlan(step.xseq, step.yseq), *sources)))
        exclude = [self.host_mask(out, np.ma.getmaskarray, m) for m in masks] or None
        return key, exclude

    def dropna(self, out, step):
        """SelectionDropNa (vaex/selections.py:78-100): the rows with no NaN (drop_nan) and no missing value (drop_masked) in any of
        the expressions; a masked row is not NaN (vaex.functions.isnan)"""
        from . import expression as _expr
        frame = self.frame
        terms = []
        for e in step.expressions:
            col = frame.columns[e]
            if isinstance(col, _expr.DeviceExpression):
                raise NotImplementedError(f"select_non_missing of the virtual column {e!r}")
            missing = _missing_fn(col)
            mkey = self.host_mask(out, missing, col) if missing is not None else None
            nan = None
            if step.drop_nan:
                hostnan = _host_nan_fn(col)
                if hostnan is not None:
                    nan = self.host_mask(out, hostnan, col)
                elif not _is_arrow(col) and _lib.dtype_of(col).kind == "f":
                    nan = "((%s) != (%s))" % (e, e)
                    if _is_masked(col):
                        nan = "(%s & ~(%s))" % (nan, mkey)
            if nan is not None:
                terms.append(nan)
            if step.drop_masked and mkey is not None:
                terms.append(mkey)
        if not terms:
            return self.host_mask(out, lambda b: np.ones(len(b), np.bool_), frame.columns[step.expressions[0]] if step.expressions else np.zeros(frame.length, np.bool_))
        return self.join(out, "~({0})", [self.any_of(out, terms)])


def resolve(frame, selection, memo=None, stack=()):
    """a selection object of `frame` -> SelectionMask"""
    return _Resolver(frame, {} if memo is None else memo).selection(selection, stack)


def names_selection(frame, text):
    """whether `text` names a selection of `frame` that is neither a column nor a variable"""
    return any(n not in frame.columns and n not in frame.variables and frame._has_history(n) for n in _names(text))


def resolve_text(frame, text, memo=None):
    """a selection argument string of `frame` -> the selection it names (KeyError naming it when there is none), or a SelectionMask
    of the expression with the selections it names as inputs"""
    text = str(text)
    r = _Resolver(frame, {} if memo is None else memo)
    if text.isidentifier() and text not in frame.columns and text not in frame.variables:
        return r.name(text, ())
    return r.selection(SelectionExpression(text, None, "replace"))
