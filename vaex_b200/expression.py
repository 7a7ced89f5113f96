"""Device-side evaluation of simple expressions: virtual columns, filters and selections of the chunk-feed loop.

Reference: every chunk, ``_BlockScope.evaluate`` runs Python ``eval(expression, expression_namespace, scope)`` over the numpy
blocks (packages/vaex-core/vaex/scopes.py:108-128); the pre-filter mask compresses every dependent column
(vaex/execution.py:516-522); selections are expressions evaluated the same way (:539, :551).  Here the expression is compiled
ONCE from its Python AST into a postfix program for ``b200_eval`` (csrc/expr.cu).  numpy decides the dtype of every node — the
compiler asks numpy itself (zero-length arrays, so NEP 50's weak Python scalars are honoured) — and the device performs exactly one
correctly rounded operation per node in that dtype, which makes the results bit-identical to the reference's numpy evaluation.

Supported: column names, numeric literals, ``+ - * /``, unary ``-``, ``abs() sqrt()``, ``< <= > >= == !=`` (not chained: numpy rejects `a < b < c` on arrays too), ``& | ~``
on booleans, ``.astype('dtype')`` and ``_ordinal_values(x, hash_map_unique)`` (vaex/functions.py:2454-2463).  Anything else raises
``NotImplementedError`` when the expression is compiled — never a silent CPU evaluation.

String columns are read only by vaex's string predicates and measures: ``str_equals / str_notequals`` (also as ``s == 'lit'``,
``s != t``), ``str_startswith``, ``str_endswith``, ``str_contains``, ``str_count``, ``str_find``, ``str_rfind``, ``str_len`` and
``str_byte_length``.  Each such call is run over the chunk by ``b200_str_eval`` (csrc/strexpr.cu) into a device column first; the
program reads that column as an ordinary input.
"""
import ast
import ctypes as C
import inspect

import numpy as np

from . import _lib

(EX_INPUT, EX_CONST_F64, EX_CONST_I64, EX_ADD, EX_SUB, EX_MUL, EX_DIV, EX_NEG, EX_ABS, EX_SQRT, EX_LT, EX_LE, EX_GT, EX_GE, EX_EQ, EX_NE, EX_AND, EX_OR, EX_NOT,
 EX_CAST, EX_ORDINAL) = range(21)
# the string calls of b200_str_eval, numbered after the program opcodes (include/b200agg.h)
(EX_STR_EQUALS, EX_STR_EQUALS2, EX_STR_STARTSWITH, EX_STR_ENDSWITH, EX_STR_CONTAINS, EX_STR_COUNT, EX_STR_FIND, EX_STR_RFIND, EX_STR_LEN,
 EX_STR_BYTE_LENGTH) = range(21, 31)
# I64_U64 / U64_I64: comparisons of a signed integer with a uint64 by exact value, the operands in the order of the name
EXC_F64, EXC_F32, EXC_I64, EXC_U64, EXC_BOOL, EXC_I64_U64, EXC_U64_I64 = range(7)

_BINOPS = {ast.Add: (EX_ADD, np.add), ast.Sub: (EX_SUB, np.subtract), ast.Mult: (EX_MUL, np.multiply), ast.Div: (EX_DIV, np.true_divide)}
_CMPOPS = {ast.Lt: EX_LT, ast.LtE: EX_LE, ast.Gt: EX_GT, ast.GtE: EX_GE, ast.Eq: EX_EQ, ast.NotEq: EX_NE}


# the signatures of vaex's string functions (vaex/functions.py), used to bind the arguments of a call
def str_equals(x, y): pass
def str_notequals(x, y): pass
def str_startswith(x, pat): pass
def str_endswith(x, pat): pass
def str_contains(x, pattern, regex=True): pass
def str_count(x, pat, regex=False): pass
def str_find(x, sub, start=0, end=None): pass
def str_rfind(x, sub, start=0, end=None): pass
def str_len(x): pass
def str_byte_length(x): pass


_STR_FUNCS = {f.__name__: f for f in (str_equals, str_notequals, str_startswith, str_endswith, str_contains, str_count, str_find, str_rfind, str_len,
                                      str_byte_length)}
_STR_OPS = {"str_startswith": EX_STR_STARTSWITH, "str_endswith": EX_STR_ENDSWITH, "str_contains": EX_STR_CONTAINS, "str_count": EX_STR_COUNT,
            "str_find": EX_STR_FIND, "str_rfind": EX_STR_RFIND, "str_len": EX_STR_LEN, "str_byte_length": EX_STR_BYTE_LENGTH}
_REGEX_META = set(".^$*+?()[]{}|\\")
_MAX_INPUTS = 8  # b200_eval's input limit
_INT64_MAX = (1 << 63) - 1


class StrCall:
    """one string call of a program: b200_str_eval's opcode, the string column(s) it reads, the pattern as UTF-8 bytes and the
    code-point window of find / rfind (end = INT64_MAX: to the end of the row)"""

    def __init__(self, op, columns, pattern=b"", start=0, end=_INT64_MAX):
        self.op, self.columns, self.pattern, self.start, self.end = op, tuple(columns), bytes(pattern), int(start), int(end)
        self.dtype = np.dtype(np.int64 if op in (EX_STR_COUNT, EX_STR_FIND, EX_STR_RFIND, EX_STR_LEN, EX_STR_BYTE_LENGTH) else np.bool_)

    def key(self):
        return (self.op, self.columns, self.pattern, self.start, self.end)


def _cls(dtype):
    dtype = np.dtype(dtype)
    if dtype == np.float64:
        return EXC_F64
    if dtype == np.float32:
        return EXC_F32
    if dtype == np.bool_:
        return EXC_BOOL
    if dtype.kind == "i":
        return EXC_I64
    if dtype.kind == "u":
        return EXC_U64
    raise NotImplementedError(f"dtype {dtype} is not supported in device expressions")


def _i64(v):
    """an integer constant's 64-bit pattern as a signed int (uint64 values >= 2^63 wrap)"""
    return v - (1 << 64) if v >= 1 << 63 else v


class _Node:
    """value on the compile-time stack: a typed array expression, or a weak Python scalar (NEP 50) that takes the other
    operand's dtype"""

    def __init__(self, dtype=None, scalar=None):
        self.dtype = None if dtype is None else np.dtype(dtype)
        self.scalar = scalar

    @property
    def weak(self):
        return self.dtype is None

    def probe(self):
        return self.scalar if self.weak else np.zeros(0, self.dtype)


class Program:
    """A compiled expression: postfix ops + the column names it reads + the hash maps it probes."""

    def __init__(self, expression, dtypes, variables=None, strings=()):
        """strings: the names of the string columns (their dtype in `dtypes` is object, like any column without a numpy dtype)"""
        self.expression = str(expression)
        self.ops = []
        self.inputs = []    # column names, in input-index order
        self.strcalls = []  # StrCall: their results are the inputs after `inputs`, in this order
        self.sets = []      # ordered sets (superutils objects) probed by _ordinal_values
        self._dtypes = dtypes
        self._strings = set(strings)
        self._variables = dict(variables or {})
        tree = ast.parse(self.expression, mode="eval")
        top = self._emit(tree.body)
        if top.weak:  # a bare constant: give it numpy's default type
            top = self._materialise(top, np.result_type(top.scalar))
        self.dtype = top.dtype
        if self.strcalls:  # a string call's input index is known once every column input is
            if len(self.inputs) + len(self.strcalls) > _MAX_INPUTS:
                raise NotImplementedError(f"{self.expression!r} reads more than {_MAX_INPUTS} columns and string calls: not supported in device expressions")
            self.ops = [(op, cls, len(self.inputs) - arg - 1 if op == EX_INPUT and arg < 0 else arg, f, i) for op, cls, arg, f, i in self.ops]

    # ---- emit helpers -------------------------------------------------------------------------------------------------
    def _op(self, op, cls=0, arg=0, f=0.0, i=0):
        self.ops.append((op, cls, arg, float(f), int(i)))

    def _materialise(self, node, dtype):
        """push-time resolution of a weak scalar: it becomes a constant of `dtype`"""
        dtype = np.dtype(dtype)
        if dtype.kind == "f" and isinstance(node.scalar, int):
            # numpy converts a Python int to a double first (OverflowError beyond it), then to the float type: two roundings
            value = np.float64(float(node.scalar)).astype(dtype)
        else:
            value = np.asarray(node.scalar).astype(dtype)[()]  # numpy's own conversion of the literal
        c = _cls(dtype)
        pos = node.slot
        if c in (EXC_F64, EXC_F32):
            self.ops[pos] = (EX_CONST_F64, c, 0, float(value), 0)
        else:
            self.ops[pos] = (EX_CONST_I64, c, 0, 0.0, _i64(int(value)))
        return _Node(dtype)

    def _cast(self, node, dtype):
        dtype = np.dtype(dtype)
        if node.dtype != dtype:
            self._op(EX_CAST, _cls(node.dtype), _lib.DTYPE_CODE[dtype.name])
        return _Node(dtype)

    def _emit(self, n):
        if isinstance(n, ast.Name):
            if n.id in self._strings:
                raise NotImplementedError(f"column {n.id!r} is a string column: only the str_* functions and == / != against a string read it; "
                                          "other uses are not supported in device expressions")
            if n.id not in self._dtypes:
                raise KeyError(f"column {n.id!r} not found (expression {self.expression!r})")
            dt = np.dtype(self._dtypes[n.id])
            if dt.kind in "mM" or dt.name not in _lib.DTYPE_CODE:
                raise NotImplementedError(f"column {n.id!r} has dtype {dt}: not supported in device expressions")
            if n.id not in self.inputs:
                self.inputs.append(n.id)
            self._op(EX_INPUT, _cls(dt), self.inputs.index(n.id))
            return _Node(dt)
        if isinstance(n, ast.Constant):
            if isinstance(n.value, bool) or not isinstance(n.value, (int, float)):
                raise NotImplementedError(f"literal {n.value!r} is not supported in device expressions")
            node = _Node(scalar=n.value)
            node.slot = len(self.ops)
            self._op(EX_CONST_F64)  # placeholder, typed when its partner is known
            return node
        if isinstance(n, ast.UnaryOp):
            if isinstance(n.op, ast.USub):
                if isinstance(n.operand, ast.Constant) and isinstance(n.operand.value, (int, float)) and not isinstance(n.operand.value, bool):
                    return self._emit(ast.copy_location(ast.Constant(-n.operand.value), n))
                a = self._emit(n.operand)
                if a.dtype.kind == "b":
                    raise NotImplementedError("numpy has no negative of a boolean")
                self._op(EX_NEG, _cls(a.dtype))
                return self._wrap(a.dtype)
            if isinstance(n.op, ast.Invert):
                a = self._emit(n.operand)
                if a.dtype != np.bool_:
                    raise NotImplementedError("~ is only supported on boolean expressions")
                self._op(EX_NOT, EXC_BOOL)
                return a
            if isinstance(n.op, ast.UAdd):
                return self._emit(n.operand)
            raise NotImplementedError(ast.dump(n.op))
        if isinstance(n, ast.BinOp):
            if isinstance(n.op, (ast.BitAnd, ast.BitOr)):
                a, b = self._emit(n.left), self._emit(n.right)
                if a.weak or b.weak or a.dtype != np.bool_ or b.dtype != np.bool_:
                    raise NotImplementedError("& and | are only supported on boolean expressions")
                self._op(EX_AND if isinstance(n.op, ast.BitAnd) else EX_OR, EXC_BOOL)
                return _Node(np.bool_)
            if type(n.op) not in _BINOPS:
                raise NotImplementedError(f"operator {type(n.op).__name__} is not supported in device expressions")
            opcode, ufunc = _BINOPS[type(n.op)]
            a = self._emit(n.left)
            mark = len(self.ops)
            b = self._emit(n.right)
            return self._binary(opcode, ufunc, a, b, mark)
        if isinstance(n, ast.Compare):
            if len(n.ops) != 1:
                raise NotImplementedError("chained comparisons are not supported in device expressions (numpy rejects them too)")
            if isinstance(n.ops[0], (ast.Eq, ast.NotEq)) and (self._is_string(n.left) or self._is_string(n.comparators[0])):
                # vaex turns s == 'lit' / s != t into str_equals / str_notequals (vaex/expression.py:115-132)
                return self._str_equals(n.left, n.comparators[0], isinstance(n.ops[0], ast.NotEq))
            if type(n.ops[0]) not in _CMPOPS:
                raise NotImplementedError(type(n.ops[0]).__name__)
            start = len(self.ops)
            left = self._emit(n.left)
            mark = len(self.ops)
            right = self._emit(n.comparators[0])
            return self._compare(_CMPOPS[type(n.ops[0])], left, right, start, mark)
        if isinstance(n, ast.Call):
            return self._call(n)
        if isinstance(n, ast.Attribute):
            raise NotImplementedError("attribute access is only supported as .astype(...)")
        raise NotImplementedError(f"{type(n).__name__} is not supported in device expressions")

    def _wrap(self, dtype):
        """integer results narrower than 64 bits wrap like numpy's"""
        dtype = np.dtype(dtype)
        if dtype.kind in "iu" and dtype.itemsize < 8:
            self._op(EX_CAST, _cls(dtype), _lib.DTYPE_CODE[dtype.name])
        return _Node(dtype)

    def _promote(self, a, b, mark, ufunc):
        """numpy's input dtype for `ufunc(a, b)`; inserts the casts.  `mark` = index of the first op of b's code."""
        if a.weak and b.weak:
            raise NotImplementedError("constant folding of two literals is not supported: write the value")
        # ask numpy: the loop it selects tells both the computation dtype and the output dtype
        out = ufunc(a.probe(), b.probe())
        if ufunc in (np.less,):
            common = np.result_type(*(x.probe() for x in (a, b)))
        else:
            common = out.dtype
        if a.weak:
            a = self._materialise(a, common)
        elif a.dtype != common:  # cast a: its code ends right before `mark`
            self.ops.insert(mark, (EX_CAST, _cls(a.dtype), _lib.DTYPE_CODE[np.dtype(common).name], 0.0, 0))
            if getattr(b, "slot", None) is not None and b.weak:
                b.slot += 1
            a = _Node(common)
        if b.weak:
            b = self._materialise(b, common)
        elif b.dtype != common:
            b = self._cast(b, common)
        return a, b, np.dtype(common)

    def _compare(self, opcode, a, b, start, mark):
        """a comparison; `start` / `mark` = index of the first op of a's / b's code"""
        lit, col = (a, b) if a.weak else (b, a)
        if lit.weak and not col.weak and col.dtype.kind in "iu" and isinstance(lit.scalar, int):
            return self._compare_int_literal(opcode, a, b, start)
        if not a.weak and not b.weak and {a.dtype.kind, b.dtype.kind} == {"i", "u"} and np.dtype(np.uint64) in (a.dtype, b.dtype):
            # numpy compares a signed integer with a uint64 by exact value (its qQ / Qq loops), not through float64
            self._op(opcode, EXC_I64_U64 if a.dtype.kind == "i" else EXC_U64_I64)
            return _Node(np.bool_)
        a, b, common = self._promote(a, b, mark, np.less)
        self._op(opcode, _cls(common))
        return _Node(np.bool_)

    def _compare_int_literal(self, opcode, a, b, start):
        """integer column against a Python int: numpy compares by the literal's value, whatever the column's width"""
        lit, col = (a, b) if a.weak else (b, a)
        v = lit.scalar
        if v >= 1 << 64 or v < -(1 << 63):
            # beyond every 64-bit value: the answer does not depend on the row, so the operand's code is dropped
            less = (v > 0) == (b is lit)  # a < b on every row
            result = {EX_LT: less, EX_LE: less, EX_GT: not less, EX_GE: not less, EX_EQ: False, EX_NE: True}[opcode]
            del self.ops[start:]
            self._op(EX_CONST_I64, EXC_BOOL, i=int(result))
            return _Node(np.bool_)
        col_signed = col.dtype.kind == "i"
        lit_signed = col_signed if 0 <= v < 1 << 63 else v < 0
        self.ops[lit.slot] = (EX_CONST_I64, EXC_I64 if lit_signed else EXC_U64, 0, 0.0, _i64(v))
        if lit_signed == col_signed:
            cls = EXC_I64 if col_signed else EXC_U64
        else:
            cls = EXC_I64_U64 if (col_signed if a is col else lit_signed) else EXC_U64_I64
        self._op(opcode, cls)
        return _Node(np.bool_)

    def _binary(self, opcode, ufunc, a, b, mark):
        a, b, common = self._promote(a, b, mark, ufunc)
        if common == np.bool_:
            raise NotImplementedError("arithmetic on booleans is not supported in device expressions")
        if opcode == EX_DIV and common.kind not in "f":
            raise NotImplementedError("unexpected integer true-division loop")
        self._op(opcode, _cls(common))
        return self._wrap(common)

    def _call(self, n):
        # x.astype('float64')
        if isinstance(n.func, ast.Attribute) and n.func.attr == "astype":
            a = self._emit(n.func.value)
            if len(n.args) != 1 or not isinstance(n.args[0], ast.Constant) or not isinstance(n.args[0].value, str):
                raise NotImplementedError("astype takes one dtype string")
            dt = np.dtype(n.args[0].value)
            if dt.name not in _lib.DTYPE_CODE:
                raise NotImplementedError(f"astype({dt})")
            if a.weak:  # Python evaluates it too: an int or float has no .astype
                raise AttributeError(f"{type(a.scalar).__name__!r} object has no attribute 'astype'")
            return self._cast(a, dt)
        if not isinstance(n.func, ast.Name):
            raise NotImplementedError("only plain function names can be called in device expressions")
        name = n.func.id
        if name in _STR_FUNCS:
            return self._string_call(name, n)
        if name in ("abs", "sqrt"):
            if len(n.args) != 1:
                raise TypeError(f"{name}() takes one argument")
            a = self._emit(n.args[0])
            if a.weak:
                raise NotImplementedError(f"{name}() of a literal: write the value")
            if name == "abs":
                if a.dtype.kind in "bu":
                    return a
                self._op(EX_ABS, _cls(a.dtype))
                return self._wrap(a.dtype)
            out = np.sqrt(a.probe()).dtype  # ints -> float64, float32 stays
            if out not in (np.float64, np.float32):
                raise NotImplementedError(f"sqrt of {a.dtype}")
            a = self._cast(a, out)
            self._op(EX_SQRT, _cls(out))
            return _Node(out)
        if name == "_ordinal_values":
            if len(n.args) != 2 or not isinstance(n.args[1], ast.Name):
                raise NotImplementedError("_ordinal_values(expression, hash_map_unique_variable)")
            hm = self._variables.get(n.args[1].id)
            if hm is None:
                raise KeyError(f"variable {n.args[1].id!r} not found")
            internal = getattr(hm, "_internal", hm)
            a = self._emit(n.args[0])
            key_dtype = np.dtype(internal._np_dtype())
            if a.weak:
                a = self._materialise(a, key_dtype)
            a = self._cast(a, key_dtype)  # the set is probed with keys of its own dtype
            if internal not in self.sets:
                self.sets.append(internal)
            self._op(EX_ORDINAL, _cls(key_dtype), self.sets.index(internal))
            # ordered_set::map_ordinal picks the narrowest signed type that holds the set (src/hash_primitives.hpp:611-623)
            count = len(internal)
            out = np.dtype("int8") if count < 2 ** 7 else np.dtype("int16") if count < 2 ** 15 else np.dtype("int32") if count < 2 ** 31 else np.dtype("int64")
            return self._cast(_Node(np.int64), out)
        raise NotImplementedError(f"function {name}() is not supported in device expressions")

    # ---- string calls ---------------------------------------------------------------------------------------------------
    def _is_string(self, n):
        return isinstance(n, ast.Name) and n.id in self._strings

    def _str_input(self, call):
        """the program reads a string call's result like a column: EX_INPUT with a placeholder index, numbered after `inputs` once
        the whole expression is compiled"""
        keys = [c.key() for c in self.strcalls]
        if call.key() not in keys:
            self.strcalls.append(call)
            keys.append(call.key())
        self._op(EX_INPUT, _cls(call.dtype), -1 - keys.index(call.key()))
        return _Node(call.dtype)

    def _str_literal(self, n, what):
        if not (isinstance(n, ast.Constant) and isinstance(n.value, str)):
            raise NotImplementedError(f"{what} must be a string literal in device expressions")
        return n.value.encode("utf8")

    def _int_literal(self, n, what):
        if isinstance(n, ast.UnaryOp) and isinstance(n.op, ast.USub):
            return -self._int_literal(n.operand, what)
        if not (isinstance(n, ast.Constant) and isinstance(n.value, int) and not isinstance(n.value, bool)):
            raise NotImplementedError(f"{what} must be an integer literal in device expressions")
        if not -(1 << 63) <= n.value <= _INT64_MAX:
            raise OverflowError(f"{what} {n.value} does not fit in int64")
        return n.value

    def _str_equals(self, x, y, negate):
        """str_equals(x, y) / str_notequals(x, y) (= ~str_equals, vaex/functions.py:1015-1060) with either side a string column"""
        if not self._is_string(x):
            x, y = y, x  # 'lit' == s
        if not self._is_string(x):
            raise NotImplementedError("str_equals / str_notequals take a string column: not supported in device expressions")
        if self._is_string(y):
            node = self._str_input(StrCall(EX_STR_EQUALS2, (x.id, y.id)))
        else:
            node = self._str_input(StrCall(EX_STR_EQUALS, (x.id,), self._str_literal(y, "the other side of a string comparison")))
        if negate:
            self._op(EX_NOT, EXC_BOOL)
        return node

    def _string_call(self, name, n):
        try:
            args = inspect.signature(_STR_FUNCS[name]).bind(*n.args, **{k.arg: k.value for k in n.keywords})
        except TypeError as e:
            raise TypeError(f"{name}(): {e}") from None
        args.apply_defaults()
        a = args.arguments
        if name in ("str_equals", "str_notequals"):  # either argument may be the string column
            return self._str_equals(a["x"], a["y"], name == "str_notequals")
        if not self._is_string(a["x"]):
            raise NotImplementedError(f"{name}() of anything but a string column is not supported in device expressions")
        op = _STR_OPS[name]
        col = (a["x"].id,)
        if op in (EX_STR_LEN, EX_STR_BYTE_LENGTH):
            return self._str_input(StrCall(op, col))
        pattern = self._str_literal(a.get("pat", a.get("pattern", a.get("sub"))), f"the pattern of {name}()")
        if "regex" in a:
            regex = a["regex"]
            if isinstance(regex, ast.AST):
                if not (isinstance(regex, ast.Constant) and isinstance(regex.value, bool)):
                    raise NotImplementedError(f"regex= of {name}() must be True or False")
                regex = regex.value
            if regex and _REGEX_META & set(pattern.decode("utf8")):
                raise NotImplementedError(f"{name}(): the regex {pattern.decode('utf8')!r} is not supported in device expressions (there is no device "
                                          "regex engine); a pattern without any of .^$*+?()[]{}|\\ is searched as a literal")
        if op == EX_STR_COUNT and not pattern:
            # the reference's literal count never ends on it; its regex count gives len + 1 empty matches.  Neither is computed here.
            raise ValueError("str_count() of an empty pattern is not supported: vaex's literal count never ends on it")
        if op in (EX_STR_FIND, EX_STR_RFIND):
            start = a["start"] if isinstance(a["start"], int) else self._int_literal(a["start"], f"start of {name}()")
            end = a["end"]
            if isinstance(end, ast.Constant) and end.value is None:
                end = None
            end = _INT64_MAX if end is None else self._int_literal(end, f"end of {name}()")
            return self._str_input(StrCall(op, col, pattern, start, end))
        return self._str_input(StrCall(op, col, pattern))

    # ---- run ----------------------------------------------------------------------------------------------------------
    def c_ops(self):
        arr = (_lib.ExprOp * len(self.ops))()
        for k, (op, cls, arg, f, i) in enumerate(self.ops):
            arr[k].op, arr[k].cls, arr[k].arg, arr[k].f, arr[k].i = op, cls, arg, f, i
        return arr


class DeviceExpression:
    """A virtual column / filter / selection evaluated on the device chunk by chunk (the executor calls
    ``chunk(thread_index, i1, i2)`` on the worker's slot; the consumer runs on the same slot, i.e. the same stream)."""

    device_virtual = True

    def __init__(self, expression, columns, variables=None):
        from .hash import is_string_column
        self.expression = str(expression)
        self._columns = columns
        # an arrow column has no numpy dtype, so no device expression reads it as a number (a join's gathered strings are arrow);
        # string columns are read by the string calls only
        dtypes = {k: _lib.dtype_of(v) if hasattr(v, "dtype") else np.dtype("O") for k, v in columns.items()}
        self.program = Program(expression, dtypes, variables, strings=[k for k, v in columns.items() if is_string_column(v)])
        self.dtype = self.program.dtype
        strings = list(dict.fromkeys(name for call in self.program.strcalls for name in call.columns))
        # the executor looks here to decide host / device feeding
        self.columns = [columns[name] for name in self.program.inputs] + [columns[name] for name in strings]
        for name, col in zip(self.program.inputs, self.columns):
            if getattr(col, "device_virtual", False):
                raise NotImplementedError(f"{name!r} is itself a device-evaluated column: nest the expressions textually instead")
            if isinstance(col, np.ndarray) and np.ma.isMaskedArray(col):
                raise NotImplementedError(f"column {name!r} is masked: masked inputs are not supported in device expressions")
        self._ops = self.program.c_ops()
        self._buffers = {}
        self._ctx_cached = None

    def __len__(self):
        return len(self.columns[0]) if self.columns else 0

    @property
    def _ctx(self):
        if self._ctx_cached is None:
            self._ctx_cached = _lib.context()
        return self._ctx_cached

    def _buffer(self, thread_index, n, key=None, dtype=None):
        """the slot-local device buffer of the result (key None) or of a string call's column"""
        import torch
        nbytes = max(n, 1) * (dtype or self.dtype).itemsize
        buf = self._buffers.get((thread_index, key))
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(nbytes + 16, dtype=torch.uint8, device=f"cuda:{self._ctx.device}")
            self._buffers[(thread_index, key)] = buf
        return buf

    def _string_calls(self, thread_index, i1, i2):
        """run the program's string calls over rows [i1, i2) on the slot: one device column each, in program input order.  The
        string buffers are copied to the device on the slot's stream (b200_str_eval reads device memory only); allocated under that
        stream, they go back to torch's cache only once the stream is past the calls that read them."""
        import torch
        from .join import _string_source
        n = int(i2 - i1)
        slot = self._ctx.slot(thread_index)
        device = f"cuda:{self._ctx.device}"
        staged = {}
        outs = []
        with torch.cuda.stream(torch.cuda.ExternalStream(self._ctx.stream(slot), device=device)):

            def stage(a):
                return torch.from_numpy(np.ascontiguousarray(a)).to(device, non_blocking=False) if a is not None and len(a) else None

            def column(name, nulls):
                if name not in staged:
                    offsets, isz, data, first, mask = _string_source(self._columns[name][i1:i2])
                    nbytes = int(offsets[-1]) - first
                    staged[name] = [stage(offsets), isz, stage(data) if nbytes else None, first, nbytes, mask, None]
                col = staged[name]
                if nulls and col[5] is not None and col[6] is None:
                    col[6] = stage(col[5])
                off, isz, data, first, nbytes, _, mask = col
                # the device pointer the offsets index: the staged range starts at offset value `first`
                return off.data_ptr(), isz, (data.data_ptr() - first) if data is not None else None, mask.data_ptr() if nulls and mask is not None else None, nbytes

            pat = {}
            for k, call in enumerate(self.program.strcalls):
                nulls = call.op in (EX_STR_EQUALS, EX_STR_EQUALS2)
                off, isz, data, mask, nbytes = column(call.columns[0], nulls)
                off2, isz2, data2, mask2, _ = column(call.columns[1], nulls) if len(call.columns) > 1 else (None, 0, None, None, 0)
                if call.pattern and call.pattern not in pat:
                    pat[call.pattern] = stage(np.frombuffer(call.pattern, np.uint8))
                out = self._buffer(thread_index, n, k, call.dtype)
                _lib.check(_lib.lib().b200_str_eval(self._ctx._h, slot, call.op, off, isz, data, mask, off2, isz2, data2, mask2,
                                                    pat[call.pattern].data_ptr() if call.pattern else None, len(call.pattern), call.start, call.end, n,
                                                    nbytes, out.data_ptr()))
                outs.append((out, call.dtype))
        return outs

    def chunk(self, thread_index, i1, i2):
        return self.run(thread_index, i1, i2, [self._columns[name][i1:i2] for name in self.program.inputs])

    def run(self, thread_index, i1, i2, parts):
        """the program over rows [i1, i2) with `parts` as the blocks of its column inputs, in program.inputs order (a selection feeds
        the masks it computes this way, vaex_b200/selections.py)"""
        n = int(i2 - i1)
        raw = self._buffer(thread_index, n)
        out = DeviceArray(raw.data_ptr(), n, self.dtype, keep=raw)
        if n == 0:
            return out
        nin = len(self.program.inputs) + len(self.program.strcalls)
        inputs = (_lib.ExprInput * max(nin, 1))()
        keep = []
        for k, part in enumerate(parts):
            if isinstance(part, np.ndarray) and not part.dtype.isnative:
                part = part.astype(part.dtype.newbyteorder("="))
            c = _lib.column(part)
            keep.append(c)
            inputs[k].data, inputs[k].dtype = c.ptr, c.code
        if self.program.strcalls:
            for k, (buf, dtype) in enumerate(self._string_calls(thread_index, i1, i2), start=len(self.program.inputs)):
                c = _lib.column(DeviceArray(buf.data_ptr(), n, dtype, keep=buf))
                keep.append(c)
                inputs[k].data, inputs[k].dtype = c.ptr, c.code
        sets = (C.c_void_p * max(len(self.program.sets), 1))(*[s._h for s in self.program.sets])
        _lib.check(_lib.lib().b200_eval(self._ctx._h, self._ctx.slot(thread_index), self._ops, len(self.program.ops), inputs, nin, sets, len(self.program.sets), n,
                                        _lib.memspace(*keep), _lib.DTYPE_CODE[self.dtype.name], raw.data_ptr()))
        return out

    def evaluate(self, i1=0, i2=None, thread_index=0):
        """host copy of the values (tests, small results)"""
        i2 = len(self) if i2 is None else i2
        return self.chunk(thread_index, i1, i2).to_numpy()


class DeviceArray:
    """A typed view of device memory (``__cuda_array_interface__``), what the device evaluators hand to the task parts."""

    def __init__(self, ptr, length, dtype, keep=None):
        self.ptr, self.length, self.dtype, self._keep = int(ptr), int(length), np.dtype(dtype), keep
        self.__cuda_array_interface__ = {"shape": (self.length,), "typestr": self.dtype.str, "data": (self.ptr, False), "version": 3, "strides": None}

    def __len__(self):
        return self.length

    def __getitem__(self, s):
        if not isinstance(s, slice):
            raise TypeError("only slices")
        a, b, step = s.indices(self.length)
        if step != 1:
            raise ValueError("only contiguous slices")
        return DeviceArray(self.ptr + a * self.dtype.itemsize, max(b - a, 0), self.dtype, keep=self._keep)

    def to_numpy(self):
        import torch
        _lib.context().sync()  # the producing kernel runs on a slot's stream, torch copies on its own
        out = np.empty(self.length, self.dtype)
        if self.length:
            t = torch.as_tensor(self, device="cuda")
            out[:] = t.cpu().numpy().view(self.dtype) if self.dtype.kind == "u" and self.dtype.itemsize > 1 else t.cpu().numpy()
        return out


def compact(thread_index, keep_mask, columns, ctx=None):
    """Filter compaction on the device (vaex/execution.py:516-522 `filter(v, filter_mask)`): returns (count, [device arrays]) with
    the rows of every column where keep_mask is non-zero, in order.  Columns may be host (numpy) or device arrays.  A string column
    (arrow or numpy object) comes back as a large_string arrow array: the kept row numbers are compacted with the other columns
    and the strings gathered by them (b200_take_strings)."""
    import torch
    from .hash import is_string_column
    ctx = ctx or _lib.context()
    n = len(keep_mask)
    strings = [k for k, c in enumerate(columns) if is_string_column(c)]
    fixed = [c for c in columns if not is_string_column(c)] + ([np.arange(n, dtype=np.int64)] if strings else [])
    cols = [_lib.column(c.astype(c.dtype.newbyteorder("=")) if isinstance(c, np.ndarray) and not c.dtype.isnative else c) for c in fixed]
    km = _lib.mask_column(keep_mask)
    ncols = len(cols)
    bufs = [torch.empty(max(n, 1) * c.dtype.itemsize + 16, dtype=torch.uint8, device=f"cuda:{ctx.device}") for c in cols]
    cptr = (C.c_void_p * max(ncols, 1))(*[c.ptr for c in cols])
    optr = (C.c_void_p * max(ncols, 1))(*[b.data_ptr() for b in bufs])
    dts = (C.c_int32 * max(ncols, 1))(*[c.code for c in cols])
    count = C.c_int64(0)
    _lib.check(_lib.lib().b200_compact(ctx._h, ctx.slot(thread_index), km.ptr, ncols, cptr, dts, n, _lib.memspace(km, *cols), optr, C.byref(count)))
    out = [DeviceArray(b.data_ptr(), count.value, c.dtype, keep=b) for b, c in zip(bufs, cols)]
    if not strings:
        return count.value, out
    from .join import take_strings
    rows = out.pop()
    it = iter(out)
    return count.value, [take_strings(rows, c, thread_index)[0] if k in strings else next(it) for k, c in enumerate(columns)]
