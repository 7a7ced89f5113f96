"""A plain-Python restatement of csrc/expr.cu's interpreter: runs ``expression.Program(...).ops`` row by row with the semantics the
device is meant to have, so that the compiler can be checked without a GPU and the device against a reference that does not
depend on numpy's undefined cases.

- integer classes hold Python ints, wrapped explicitly to 64 bits (and to the target width by the casts the compiler emits);
- every float operation is one numpy scalar operation in the class dtype;
- integer -> float casts round the exact integer once; float -> integer casts follow numpy's x86-64 loops, stated with exact
  integers: the 64-bit cvttsd2si for int64 / uint32, gcc's two-step sequence for uint64, the 32-bit cvttsd2si for the narrower
  types, then the wrap to the target width (DESIGN §3).

``_ordinal_values`` is not restated here: its reference is ``oracle.OrderedSet``."""
import numpy as np

from helpers import M64, f64_to_i64_x86, f64_to_u64_x86
from vaex_b200 import _lib
from vaex_b200 import expression as X

DTYPES = ["float64", "float32", "int64", "int32", "int16", "int8", "uint64", "uint32", "uint16", "uint8", "bool"]
assert DTYPES == list(_lib.DTYPES)


def f64_to_i32_x86(x):
    """the 32-bit cvttsd2si: NaN and values outside [-2^31, 2^31) -> INT32_MIN"""
    return int(x) if -2.0 ** 31 <= x < 2.0 ** 31 else -(1 << 31)


def wrap(v, dtype):
    """an exact integer wrapped to `dtype` (numpy's overflow behaviour); bool -> v != 0"""
    d = np.dtype(dtype)
    if d == np.bool_:
        return int(v != 0)
    bits = 8 * d.itemsize
    v &= (1 << bits) - 1
    if d.kind == "i" and v >= 1 << (bits - 1):
        v -= 1 << bits
    return v


def int_to_f32(v):
    """an exact integer rounded once (to nearest, ties to even) to float32"""
    m = abs(v)
    if m < 1 << 24:
        return np.float32(v)
    shift = m.bit_length() - 24
    q, r = divmod(m, 1 << shift)
    half = 1 << (shift - 1)
    if r > half or (r == half and q & 1):
        q += 1
    return np.float32(float((q << shift) * (1 if v > 0 else -1)))  # <= 25 significant bits: exact in a double


def cast(v, cls, dtype):
    """astype(dtype) of the value `v` of class `cls`"""
    d = np.dtype(dtype)
    isfloat = cls in (X.EXC_F64, X.EXC_F32)
    if d == np.float64:
        return np.float64(v) if isfloat else np.float64(float(v))  # float(int) rounds the exact integer once
    if d == np.float32:
        return np.float32(v) if isfloat else int_to_f32(int(v))
    if d == np.bool_:
        return int(bool(v != 0))
    if not isfloat:
        return wrap(int(v), d)
    x = float(v)
    if d == np.uint64:
        return f64_to_u64_x86(x)
    if d in (np.int64, np.uint32):
        return wrap(f64_to_i64_x86(x), d)
    return wrap(f64_to_i32_x86(x), d)


def _load(col, row, cls):
    x = col[row]
    if cls == X.EXC_F64:
        return np.float64(x)
    if cls == X.EXC_F32:
        return np.float32(x)
    return int(x)


def _const(op):
    _, cls, _, f, i = op
    if op[0] == X.EX_CONST_F64:
        return np.float32(f) if cls == X.EXC_F32 else np.float64(f)
    if cls == X.EXC_U64:
        return i & M64
    if cls == X.EXC_BOOL:
        return int(i != 0)
    return i


_DTYPE_OF_CLS = {X.EXC_I64: np.int64, X.EXC_U64: np.uint64}


def _arith(op, cls, a, b):
    if cls in (X.EXC_F64, X.EXC_F32):
        return {X.EX_ADD: np.add, X.EX_SUB: np.subtract, X.EX_MUL: np.multiply, X.EX_DIV: np.true_divide}[op](a, b)
    if op == X.EX_DIV:
        raise AssertionError("integer true division has no device loop")
    r = a + b if op == X.EX_ADD else a - b if op == X.EX_SUB else a * b
    return wrap(r, _DTYPE_OF_CLS[cls])


def _compare(op, a, b):
    # floats: IEEE comparisons of the numpy scalars (NaN compares unequal); integers of every class, the mixed-sign ones
    # included: by exact value
    return int({X.EX_LT: a < b, X.EX_LE: a <= b, X.EX_GT: a > b, X.EX_GE: a >= b, X.EX_EQ: a == b, X.EX_NE: a != b}[op])


def run(program, columns):
    """evaluate `program` (an expression.Program) over `columns` (name -> numpy array) row by row; returns an array of
    program.dtype"""
    cols = [np.asarray(columns[name]) for name in program.inputs]
    n = len(cols[0]) if cols else 0
    out = []
    with np.errstate(all="ignore"):
        for row in range(n):
            st = []
            for op in program.ops:
                code, cls, arg = op[0], op[1], op[2]
                if code == X.EX_INPUT:
                    st.append(_load(cols[arg], row, cls))
                elif code in (X.EX_CONST_F64, X.EX_CONST_I64):
                    st.append(_const(op))
                elif code == X.EX_CAST:
                    st[-1] = cast(st[-1], cls, _lib.DTYPES[arg])
                elif code == X.EX_NEG:
                    st[-1] = -st[-1] if cls in (X.EXC_F64, X.EXC_F32) else wrap(-st[-1], _DTYPE_OF_CLS[cls])
                elif code == X.EX_ABS:
                    if cls in (X.EXC_F64, X.EXC_F32):
                        st[-1] = np.abs(st[-1])
                    elif cls == X.EXC_I64:
                        st[-1] = wrap(abs(st[-1]), np.int64)
                elif code == X.EX_SQRT:
                    st[-1] = np.sqrt(st[-1])
                elif code == X.EX_NOT:
                    st[-1] = int(st[-1] == 0)
                elif code == X.EX_ORDINAL:
                    raise NotImplementedError("_ordinal_values: use oracle.OrderedSet")
                else:
                    b = st.pop()
                    a = st[-1]
                    if code in (X.EX_ADD, X.EX_SUB, X.EX_MUL, X.EX_DIV):
                        st[-1] = _arith(code, cls, a, b)
                    elif code == X.EX_AND:
                        st[-1] = int(a != 0 and b != 0)
                    elif code == X.EX_OR:
                        st[-1] = int(a != 0 or b != 0)
                    else:
                        st[-1] = _compare(code, a, b)
            assert len(st) == 1, program.ops
            out.append(st[0])
    dt = program.dtype
    if dt.kind == "f":
        return np.array(out, dt) if out else np.zeros(0, dt)
    return np.array(out, dtype=object).astype(dt) if out else np.zeros(0, dt)


def evaluate(expression, columns):
    """compile `expression` for these columns' dtypes and run it"""
    return run(X.Program(expression, {k: np.asarray(v).dtype for k, v in columns.items()}), columns)


# ---- the edge corpus ---------------------------------------------------------------------------------------------------------
# short column names, one column per dtype
NAMES = {"float64": "f8", "float32": "f4", "int64": "i8", "int32": "i4", "int16": "i2", "int8": "i1", "uint64": "u8", "uint32": "u4",
         "uint16": "u2", "uint8": "u1", "bool": "b"}

# floats at the integer conversion bounds, halfway values of the float32 rounding, subnormal operands and results
FLOAT_BOUNDS = [2.0 ** 24 - 1, 2.0 ** 24, 2.0 ** 24 + 1, 2.0 ** 24 + 2, 2.0 ** 60 + 2.0 ** 36, 2.0 ** 53 - 1, 2.0 ** 53, 2.0 ** 53 + 2,
                127.5, -128.5, 255.5, 65535.9, -0.5, 0.5, 1.5, 2.5, 3e9 + 1, -3e9, 1e10, 1.5e19, 2.0 ** 63 + 6144, 1e-300, 1e-10,
                1.5 * 2.0 ** -1022, 1e-20, 1e-38, 3e-39, 0.1]
for _b in (2.0 ** 31, -2.0 ** 31, 2.0 ** 32, 2.0 ** 63, -2.0 ** 63, 2.0 ** 64, -2.0 ** 31 - 1):
    FLOAT_BOUNDS += [_b, float(np.nextafter(_b, -np.inf)), float(np.nextafter(_b, np.inf))]

# integers at the float32 / float64 rounding bounds (halfway values, either side of them), the 32- and 64-bit limits
INT_BOUNDS = [2, 3, 7, -2, 100, 2 ** 24 - 1, 2 ** 24, 2 ** 24 + 1, 2 ** 24 + 3, 2 ** 31 - 1, 2 ** 31, 2 ** 31 + 1, 2 ** 32 - 1, 2 ** 32,
              2 ** 32 + 1, 2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 2 ** 53 + 3, 2 ** 60 + 2 ** 36, 2 ** 60 + 3 * 2 ** 36, 2 ** 60 + 2 ** 36 + 1,
              2 ** 63 - 1, 2 ** 63, 2 ** 63 + 2 ** 10, 2 ** 63 + 2 ** 10 + 1, 2 ** 63 + 3 * 2 ** 10, 2 ** 63 + 2 ** 39, 2 ** 64 - 2 ** 10,
              2 ** 64 - 1, -(2 ** 24) - 1, -(2 ** 31) - 1, -(2 ** 53) - 1, -(2 ** 60) - 2 ** 36, -(2 ** 63) + 2 ** 10]

# the same integers at the start of every column (clipped to the dtype), so that pairs such as int64 2^63-1 / uint64 2^63 meet
ALIGNED = [0, 1, -1, 2 ** 24 + 1, 2 ** 31 - 1, 2 ** 31, 2 ** 32, 2 ** 53, 2 ** 53 + 1, 2 ** 63 - 1, 2 ** 63, 2 ** 64 - 1, -(2 ** 63),
           127, 128, 255, 256, -128, -129]


def edge_pool(dtype):
    """helpers.edge_values(dtype) plus the conversion bounds above that the dtype holds"""
    from helpers import edge_values
    d = np.dtype(dtype)
    base = edge_values(d)
    if d.kind == "f":
        with np.errstate(all="ignore"):
            extra = np.array(FLOAT_BOUNDS).astype(d)
        return np.concatenate([base, extra])
    if d.kind == "b":
        return base
    info = np.iinfo(d)
    return np.concatenate([base, np.array([v for v in INT_BOUNDS if info.min <= v <= info.max], dtype=object).astype(d)])


def aligned(dtype):
    d = np.dtype(dtype)
    if d.kind == "b":
        return np.array([v != 0 for v in ALIGNED])
    if d.kind == "f":
        return np.array([float(v) for v in ALIGNED]).astype(d)
    info = np.iinfo(d)
    return np.array([min(max(v, int(info.min)), int(info.max)) for v in ALIGNED], dtype=object).astype(d)


def edge_columns(n=128, seed=0):
    """one column per dtype: the aligned block, then the dtype's edge pool tiled and shuffled (a different order per dtype, so
    that every binary expression meets many pairs of edges)"""
    rng = np.random.default_rng(seed)
    out = {}
    for dt in DTYPES:
        head = aligned(dt)
        out[NAMES[dt]] = np.concatenate([head, rng.permutation(np.resize(edge_pool(dt), n - len(head)))]).astype(dt)
    return out


UNARY = ["-{}", "abs({})", "sqrt({})", "~{}"]
BINARY = ["+", "-", "*", "/", "<", "<=", ">", ">=", "==", "!="]
COMMON_LITERALS = [2 ** 63, 2 ** 64, -(2 ** 63) - 1, 1e40, 1e-50, 0.1, 16777217, -0.0, 2 ** 60 + 2 ** 36 + 1]


def literals(dtype):
    """literals at the dtype's bounds (min-1, min, max, max+1) and the common ones"""
    d = np.dtype(dtype)
    if d.kind == "f":
        big = float(np.finfo(d).max)
        bounds = [big, -big] + ([3.5e38] if d.itemsize == 4 else [])
    elif d.kind == "b":
        bounds = [-1, 0, 1, 2]
    else:
        info = np.iinfo(d)
        bounds = [int(info.min) - 1, int(info.min), int(info.max), int(info.max) + 1]
    return bounds + COMMON_LITERALS


def random_expression(rng, depth=0):
    """a seeded random nested expression over the corpus columns"""
    names = list(NAMES.values())
    r = rng.random()
    if depth >= 4 or r < 0.25:
        if rng.random() < 0.8:
            return names[int(rng.integers(len(names)))]
        return repr([2, -3, 0.5, 1e-300, 255, 2 ** 40, -1.5][int(rng.integers(7))])
    if r < 0.4:
        op = UNARY[int(rng.integers(3))]
        return op.format("(" + random_expression(rng, depth + 1) + ")")
    if r < 0.5:
        t = [d for d in DTYPES if d != "uint32"][int(rng.integers(len(DTYPES) - 1))]  # numpy's uint32 casts are not one rule
        return "(" + random_expression(rng, depth + 1) + ").astype('" + t + "')"
    if r < 0.6:
        a, b = random_expression(rng, depth + 1), random_expression(rng, depth + 1)
        return "((%s) %s (%s)) %s ((%s) %s (%s))" % (a, BINARY[4 + int(rng.integers(6))], b, "&|"[int(rng.integers(2))], b,
                                                      BINARY[4 + int(rng.integers(6))], a)
    return "(%s) %s (%s)" % (random_expression(rng, depth + 1), BINARY[int(rng.integers(10))], random_expression(rng, depth + 1))


def corpus_expressions(nrandom=300, seed=1):
    """every unary op on every dtype, every binary op on every ordered pair of dtypes, astype from every dtype to every dtype,
    comparisons and arithmetic with literals at the bounds (either side), and seeded random nested expressions that fit the
    device's limits (stack depth 12, 64 ops)"""
    out = []
    for dt in DTYPES:
        out += [u.format(NAMES[dt]) for u in UNARY]
    for a in DTYPES:
        for b in DTYPES:
            out += ["%s %s %s" % (NAMES[a], op, NAMES[b]) for op in BINARY]
    for a in DTYPES:
        out += ["%s.astype('%s')" % (NAMES[a], t) for t in DTYPES]
    for dt in DTYPES:
        for lit in literals(dt):
            for op in BINARY:
                out += ["%s %s %r" % (NAMES[dt], op, lit), "%r %s %s" % (lit, op, NAMES[dt])]
    rng = np.random.default_rng(seed)
    dtypes = {NAMES[d]: np.dtype(d) for d in DTYPES}
    made = 0
    while made < nrandom:
        e = random_expression(rng)
        try:
            p = X.Program(e, dtypes)
        except Exception:
            continue
        if p.inputs and len(p.ops) <= 64 and stack_depth(p.ops) <= 12:
            out.append(e)
            made += 1
    return out


def stack_depth(ops):
    depth = deepest = 0
    for op in ops:
        code = op[0]
        if code in (X.EX_INPUT, X.EX_CONST_F64, X.EX_CONST_I64):
            depth += 1
        elif code not in (X.EX_CAST, X.EX_NEG, X.EX_ABS, X.EX_SQRT, X.EX_NOT, X.EX_ORDINAL):
            depth -= 1
        deepest = max(deepest, depth)
    return deepest


# DESIGN §3: what the compiler refuses although numpy evaluates it: sqrt with a float16 result (int8, uint8, bool), arithmetic on
# booleans, ~ on integers
UNSUPPORTED = ("sqrt of", "boolean")


def numpy_eval(expression, columns):
    """numpy's evaluation of the expression over the columns (what the reference does per chunk)"""
    with np.errstate(all="ignore"):
        return np.asarray(eval(expression, {"abs": np.abs, "sqrt": np.sqrt}, dict(columns)))


def numpy_comparable(expression, columns, n):
    """rows where numpy's answer is one rule: numpy's float -> uint32 casts differ between its scalar and vector loops for NaN
    and for values outside (-2^31, 2^32), so those rows of `<float column>.astype('uint32')` are left out (DESIGN §3)"""
    keep = np.ones(n, bool)
    for src in ("f8", "f4"):
        if expression == "%s.astype('uint32')" % src:
            x = np.asarray(columns[src], np.float64)
            keep &= (x > -2.0 ** 31) & (x < 2.0 ** 32)
    return keep
