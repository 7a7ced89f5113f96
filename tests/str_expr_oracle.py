"""A plain-Python restatement, over bytes, of the string calls of device expressions (csrc/strexpr.cu, DESIGN.md §1 "String calls"):
what vaex's StringSequenceBase methods compute for every row read through its offsets (view(i)), null or not.

Pinned against the compiled reference by tests/test_str_expr_oracle_cpu.py (oracle/ref_strfunc_shim.cpp); `contains` and `count`
come from src/strings.cpp, which needs pcre and boost, so they are restated here and pinned against bytes.find / bytes.count."""
import numpy as np

INT64_MAX = (1 << 63) - 1


def step(c):
    """the bytes a UTF-8 lead byte steps over (src/string_utils.hpp:310-326); >= 0xF8 steps one byte (the reference does not end)"""
    return 1 if c < 0x80 else 2 if c < 0xE0 else 3 if c < 0xF0 else 4 if c < 0xF8 else 1


def str_len(s):
    p = n = 0
    while p < len(s):
        p += step(s[p])
        n += 1
    return n


def index_to_byte(s, index):
    """utf8_index_to_byte_offset (src/superstring.hpp:77-95): may pass len(s) when the row ends inside a sequence"""
    p = 0
    while p < len(s) and index > 0:
        p += step(s[p])
        index -= 1
    return p


def find(s, pat, start=0, end=INT64_MAX, last=False):
    """StringSequenceBase::find (src/superstring.hpp:161-197): the byte offset inside the window, not Python's character index"""
    bs = index_to_byte(s, start)
    if end > len(s):
        be = len(s)
    elif end < 0:
        be = index_to_byte(s, str_len(s) + end)
    else:
        be = index_to_byte(s, end)
    if not (bs < len(s) and be > bs):
        return -1
    window = s[bs:be]
    return window.rfind(pat) if last else window.find(pat)


def count(s, pat):
    """the literal branch of StringSequenceBase::count (src/strings.cpp:56-66): non-overlapping, each match advances by len(pat)"""
    assert pat, "the reference never ends on an empty pattern"
    n = off = 0
    while True:
        f = s.find(pat, off)
        if f < 0:
            return n
        n += 1
        off = f + len(pat)


def contains(s, pat):
    """the literal branch of StringSequenceBase::search (src/strings.cpp:103-107): string_view::find != npos"""
    return s.find(pat) >= 0


def evaluate(name, rows, nulls=None, pattern=b"", start=0, end=INT64_MAX, rows2=None, nulls2=None):
    """one string call over `rows` (list of bytes, a null row's slot included) -> numpy bool / int64 array"""
    n = len(rows)
    nulls = np.zeros(n, bool) if nulls is None else np.asarray(nulls, bool)
    if name == "equals":
        return np.array([not nulls[i] and rows[i] == pattern for i in range(n)], bool)
    if name == "equals2":
        nulls2 = np.zeros(n, bool) if nulls2 is None else np.asarray(nulls2, bool)
        return np.array([(nulls[i] and nulls2[i]) if (nulls[i] or nulls2[i]) else rows[i] == rows2[i] for i in range(n)], bool)
    if name == "notequals":
        return ~evaluate("equals", rows, nulls, pattern)
    fn = {"startswith": lambda s: s.startswith(pattern), "endswith": lambda s: s.endswith(pattern), "contains": lambda s: contains(s, pattern),
          "count": lambda s: count(s, pattern), "find": lambda s: find(s, pattern, start, end), "rfind": lambda s: find(s, pattern, start, end, True),
          "len": str_len, "byte_length": len}[name]
    dtype = bool if name in ("startswith", "endswith", "contains") else np.int64
    return np.array([fn(s) for s in rows], dtype)


def arrow_rows(arr):
    """the bytes of every row of an arrow string / large_string array read through its offsets (null rows' slots included), and
    the null mask"""
    import pyarrow as pa
    isz = 8 if pa.types.is_large_string(arr.type) else 4
    validity, off_buf, data_buf = arr.buffers()
    off = np.frombuffer(off_buf, dtype=np.int64 if isz == 8 else np.int32, count=len(arr) + 1, offset=arr.offset * isz)
    data = bytes(data_buf) if data_buf is not None else b""
    rows = [data[off[i]:off[i + 1]] for i in range(len(arr))]
    return rows, np.asarray(arr.is_null().to_numpy(zero_copy_only=False), bool)


# ---- the edge corpus of the string-call tests --------------------------------------------------------------------------------
# rows: empty, ASCII, 2-, 3- and 4-byte UTF-8, sequences cut off at the end of the row, continuation bytes in lead position, repeats
# for count; no lead byte >= 0xF8 (the reference never ends on one: see ROWS_F8)
ROWS = [b"", b"a", b"ab", b"abc", b"aaaa", b"abab", b"ababab", b"banana", b"Amsterdam", b"Hamburg", b"burg", b"NL", b"nl",
        "café".encode(), "été".encode(), "€100".encode(), "x€y€".encode(), "\U0001F600 smile".encode(),
        "a\U0001F600b\U0001F600".encode(), b"ab\xe2\x82", b"\xf0\x9f\x98", b"\xc3", b"\x80\x80abc", b"a" * 40, (b"xy" * 37) + b"needle",
        "é".encode() * 20, b" lead", b"trail ", b"a\x00b"]
# the null rows: some with an empty slot, some with bytes in their slot (arrow allows both)
NULLS = [i in (0, 3, 11, 19) for i in range(len(ROWS))]
PATTERNS = [b"", b"a", b"ab", b"aa", b"b", b"burg", b"NL", "é".encode(), "€".encode(), "\U0001F600".encode(), b"\xe2\x82", b"needle",
            b"a" * 41, b"\x00"]
WINDOWS = [(0, None), (1, None), (-2, None), (3, None), (100, None), (0, -1), (1, -1), (0, -100), (2, 4), (1, 2), (0, 0), (0, 100), (3, -2),
           (5, 6)]
# rows with a lead byte >= 0xF8: where the reference never ends, the device steps one byte (checked against the restatement only)
ROWS_F8 = [b"\xf8", b"a\xf9b", b"\xff\xfe", b"\xf8\xe2\x82\xac"]


def second_column(rows=ROWS, nulls=NULLS):
    """the other column of equals2: the rows rotated by one, a few of them changed, its own nulls (null meets null and value)"""
    rows2 = rows[1:] + rows[:1]
    rows2 = [r + b"!" if i % 5 == 2 else r for i, r in enumerate(rows2)]
    rows2[4] = rows[4]
    return rows2, [i in (0, 4, 7, 19) for i in range(len(rows))]


def buffers(rows, nulls=None, slack=b"#"):
    """rows -> (int64 offsets, uint8 bytes, uint8 nulls or None); a null row keeps its bytes in its slot"""
    offsets = np.zeros(len(rows) + 1, np.int64)
    offsets[1:] = np.cumsum([len(r) for r in rows])
    data = np.frombuffer(b"".join(rows) + slack, np.uint8).copy()
    return offsets, data, None if nulls is None else np.asarray(nulls, np.uint8)


def calls():
    """every (name, pattern, start, end) of the corpus; end None = to the end of the row"""
    out = [("len", b"", 0, None), ("byte_length", b"", 0, None), ("equals2", b"", 0, None)]
    for p in PATTERNS:
        out += [("equals", p, 0, None), ("notequals", p, 0, None), ("startswith", p, 0, None), ("endswith", p, 0, None), ("contains", p, 0, None)]
        if p:
            out.append(("count", p, 0, None))
        out += [(f, p, s, e) for f in ("find", "rfind") for s, e in WINDOWS]
    return out


def key(name, pattern, start, end):
    return f"{name}|{pattern.hex()}|{start}|{end}"
