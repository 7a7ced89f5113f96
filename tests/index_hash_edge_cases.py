"""Edge corpus for index_hash_<T> (vaex_b200.superutils.index_hash_<T>), built on the ordered-set corpus of set_cases.

A case is dict(dtype, nmaps, updates=[(keys, mask or None, start_index)], merges=[[(keys, mask, start_index)], ...], lookup,
lookup_mask or None, dup_start), the layout of tests/golden/make_golden_index_hash.py, whose `run` drives it.

* `sequential(...)` stays where the compiled reference is sequential (tests/index_hash_oracle.py): one update at start_index 0 with
  NaN and masks, several updates at increasing start_index without NaN or null, merges in row order.  The restatement is pinned on
  all of them against the compiled classes, and tests/golden/index_hash_edges_golden.npz stores the reference's answers for a rotation
  of them (two nmaps per dtype and kind).
* `unordered(...)` leaves those conditions and is compared with the restatement only: chunks out of order, negative start_index and
  start_index past 2^40, row spans of exactly 255 / 256 / 65535 / 65536 (where index_sort's row bytes change), the sentinel key (the
  key whose canonical pattern is the table's empty marker) with duplicates also in merged indexes only, and NaN / null seen only in a
  later call or a merged index.

Every dtype of set_cases.DTYPES and every nmaps of set_cases.NMAPS; lookups are set_cases.queries (every edge value, every NaN
payload, keys never inserted) plus inserted keys, with and without a lookup mask."""
import numpy as np

import set_cases as S

DTYPES = S.DTYPES
NMAPS = S.NMAPS
SPANS = [255, 256, 65535, 65536]
FAR = 2 ** 40 - 7  # rows of one call cross 2^40


def strip(keys, mask=None):
    """the rows of `keys` that are neither NaN nor masked"""
    keep = np.ones(len(keys), bool) if mask is None else ~np.asarray(mask, bool)
    if keys.dtype.kind == "f":
        keep &= ~np.isnan(keys)
    return keys[keep]


def _u8(mask):
    return None if mask is None else np.asarray(mask).astype(np.uint8)


def _columns(dtype, nmaps, zeros, n):
    return {name: (k, m) for name, k, m in S.columns(dtype, seed=NMAPS.index(nmaps), zeros=zeros, n=n)}


def _lookup(dtype, zeros, extra, rng, masked):
    look = np.concatenate([S.queries(dtype, zeros), extra]).astype(dtype)
    return look, ((rng.random(len(look)) < 0.15).astype(np.uint8) if masked else None)


def sequential(dtype, nmaps, zeros=False, n=100):
    """{name: case}: "one_", "calls_" and "merge_" cases of one dtype and nmaps, all inside the reference's sequential conditions"""
    cols = _columns(dtype, nmaps, zeros, n)
    rng = np.random.default_rng([7, DTYPES.index(dtype), nmaps])
    out = {}
    k, m = cols["mixed"]
    masked = (NMAPS.index(nmaps) - DTYPES.index(dtype)) % len(NMAPS) % 2 == 1  # each dtype's two stored nmaps: one of each
    look, lmask = _lookup(dtype, zeros, k[:20], rng, masked)
    out[f"one_{dtype}_{nmaps}"] = dict(dtype=dtype, nmaps=nmaps, updates=[(k, _u8(m), 0)], merges=[], lookup=look, lookup_mask=lmask, dup_start=1000)
    # several calls at increasing start_index (with gaps), no NaN / null: the sentinel's long run, every key once, late first rows
    ups, start = [], 0
    for name in ("run", "distinct", "late"):
        keys = strip(*cols[name])
        ups.append((keys, None, start))
        start += len(keys) + int(rng.integers(0, 4))
    look, _ = _lookup(dtype, zeros, strip(*cols["late"])[:10], rng, False)
    out[f"calls_{dtype}_{nmaps}"] = dict(dtype=dtype, nmaps=nmaps, updates=ups, merges=[], lookup=look, lookup_mask=None, dup_start=-3)
    # merges in row order: each merged index holds later rows than everything before it
    mixed = strip(k, m)
    parts, start = [], 0
    for keys in (mixed[: len(mixed) // 2], strip(*cols["run"])[-40:], mixed[len(mixed) // 2:]):
        parts.append([(keys, None, start)])
        start += len(keys)
    look, _ = _lookup(dtype, zeros, mixed[:10], rng, False)
    out[f"merge_{dtype}_{nmaps}"] = dict(dtype=dtype, nmaps=nmaps, updates=parts[0], merges=parts[1:], lookup=look, lookup_mask=None, dup_start=0)
    return out


def unordered(dtype, zeros=True, n=100):
    """{name: case}: the cases outside the reference's sequential conditions (compared with the restatement only); nmaps cycles
    through NMAPS"""
    dt = np.dtype(dtype)
    rng = np.random.default_rng([11, DTYPES.index(dtype)])
    nm = iter(NMAPS * 4)
    out = {}

    def case(name, updates, merges=(), dup_start=0, extra=(), masked=True):
        nmaps = next(nm)
        look, lmask = _lookup(dtype, zeros, np.asarray(extra, dt), rng, masked)
        out[f"{name}_{dtype}_{nmaps}"] = dict(dtype=dtype, nmaps=nmaps, updates=list(updates), merges=[list(m) for m in merges], lookup=look,
                                             lookup_mask=lmask, dup_start=dup_start)

    cols = _columns(dtype, 1, zeros, n)
    k, m = cols["mixed"]
    m = _u8(m)
    # chunks out of order, NaN and masks in every chunk
    b = [0, len(k) // 5, len(k) // 5 + 1, 2 * len(k) // 3, len(k)]
    chunks = [(k[b[j]:b[j + 1]], m[b[j]:b[j + 1]], b[j]) for j in range(4)]
    case("order", [chunks[2], chunks[0], chunks[3], chunks[1]], extra=k[:10], dup_start=7)
    case("reversed", chunks[::-1], dup_start=-1)
    # negative start_index, then rows that cross 2^40
    case("negstart", [(k[:60], m[:60], -len(k) - 1000), (k[60:], m[60:], -(10 ** 9))], extra=k[50:70], dup_start=-5)
    case("far", [(k, m, FAR), (k[:40], None, 3)], dup_start=FAR)
    # row spans of exactly 255 / 256 / 65535 / 65536 (row_max - row_min), from row 0 and from a negative first row
    run = strip(*cols["run"])
    for span in SPANS:
        for base in (0, -(span // 3) - 1):
            second = np.concatenate([run[:3], k[:5]])
            case(f"span{span}{'neg' if base else ''}", [(k[:80], m[:80], base), (second, None, base + span - len(second) + 1)], extra=second, dup_start=base)
    # the sentinel (or the largest value) with duplicates: across merged indexes merged out of row order, and only in a merged index
    head = S.sentinel(dt) if S.sentinel(dt) is not None else S.edge_values(dt)[-1]
    rest = strip(k, m)
    a = np.concatenate([rest[:5], [head], rest[5:8], [head]]).astype(dt)
    case("sentdup", [(a, None, 10)], merges=[[(np.array([head, head], dt), None, 2)], [(np.concatenate([[head], rest[8:20]]).astype(dt), None, 100)]],
         extra=[head], dup_start=3)
    case("sentmerged", [(rest[:30], None, 0)], merges=[[(np.array([head], dt), None, 50)], [(np.array([head, rest[0], head], dt), None, 40)]],
         extra=[head], dup_start=0)
    # NaN / null seen only in a later call, and only in a merged index
    nans = S.nan_values(dt)
    late = np.concatenate([S.edge_values(dt, zeros), nans]).astype(dt)
    lmask = np.zeros(len(late), np.uint8)
    lmask[[1, -1]] = 1
    case("speclater", [(rest[:40], None, 0), (late, lmask, 500)], extra=late, dup_start=0)
    case("specmerged", [(rest[:40], None, 0)], merges=[[(late, lmask, 30)], [(late[::-1].copy(), lmask[::-1].copy(), 5000)]], extra=late, dup_start=1)
    return out


def all_sequential(zeros=False):
    out = {}
    for dtype in DTYPES:
        for nmaps in NMAPS:
            out.update(sequential(dtype, nmaps, zeros))
    return out


def all_unordered(zeros=True):
    out = {}
    for dtype in DTYPES:
        out.update(unordered(dtype, zeros))
    return out
