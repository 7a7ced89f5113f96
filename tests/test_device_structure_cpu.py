"""The device code makes three low-level decisions in one place each: how a sort runs its radix passes (radix_sort in
vaex_b200/csrc/radix.cuh), how one 1/2/4/8-byte element is read or written as raw bits (load1_raw, ldcs1_raw and store1_raw in
vaex_b200/csrc/device_utils.cuh), and how the key table of the ordered sets, counters and indexes places and probes a key
(vaex_b200/csrc/settable.cuh, with one host loop that grows the table and redoes an insert pass in hashset.cu).  The scans below keep
hand-written copies from coming back."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "vaex_b200", "csrc")

# a pointer of each element width cast and then indexed (p[i]) or offset (p + i): one element is read or written
_TYPES = {1: r"char|uint8_t|int8_t", 2: r"short|uint16_t|int16_t", 4: r"unsigned|int|uint32_t|int32_t", 8: r"long long|uint64_t|int64_t"}
ELEMENT = {w: re.compile(r"_cast<\s*(?:const\s+)?(?:\w+\s+)*?(?:%s)\s*\*\s*>\s*\([^()]*\)\s*[\[+]" % t) for w, t in _TYPES.items()}
# reads that sign-extend on purpose: not raw bits (the gather's index column)
SIGN_EXTENDING = {("take.cu", "load_index")}


def sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh")):
            text = open(os.path.join(CSRC, name)).read()
            yield name, re.sub(r"//[^\n]*|/\*.*?\*/", "", text, flags=re.S)


def enclosing_definition(text, pos):
    """(name, first line) of the function whose definition starts on the last line at column 0 before `pos` that names one"""
    for line in reversed(text[:pos].split("\n")):
        if re.match(r"[A-Za-z_]", line) and not re.match(r"(template|struct|namespace|constexpr|using|extern)\b", line):
            names = [n for n in re.findall(r"\b(\w+)\s*\(", line) if n != "__launch_bounds__"]
            if names:
                return names[0], line
    return None, ""


def enclosing_function(text, pos):
    return enclosing_definition(text, pos)[0]


def switches(text):
    """(enclosing function, body) of every switch statement"""
    for m in re.finditer(r"\bswitch\s*\(", text):
        start = text.index("{", m.end())
        depth, i = 0, start
        while True:
            depth += {"{": 1, "}": -1}.get(text[i], 0)
            if depth == 0:
                break
            i += 1
        yield enclosing_function(text, m.start()), text[start:i + 1]


def width_switches(text):
    """(enclosing function, body) of every switch on an element width: at least three of its labels are 1, 2, 4 or 8"""
    return [(fn, body) for fn, body in switches(text) if len(set(re.findall(r"\bcase\s+([1248])\s*:", body))) >= 3]


def element_switches():
    """(file, function) of every switch on an element width that reads or writes one element in at least three of the widths"""
    out = []
    for name, text in sources():
        for fn, body in width_switches(text):
            if sum(bool(ELEMENT[w].search(body)) for w in ELEMENT) >= 3:
                out.append((name, fn))
    return out


def test_radix_passes_are_launched_only_by_the_driver():
    launches = {name: len(re.findall(r"\bk_radix_(?:hist|scatter)\s*<<<", text)) for name, text in sources()}
    assert launches.pop("radix.cuh") == 2
    stray = {name: n for name, n in launches.items() if n}
    assert not stray, stray


def test_element_access_switch_lives_only_in_device_utils():
    found = element_switches()
    helpers = {fn for name, fn in found if name == "device_utils.cuh"}
    assert {"load1_raw", "ldcs1_raw", "store1_raw"} <= helpers, helpers
    stray = [site for site in found if site[0] != "device_utils.cuh" and site not in SIGN_EXTENDING]
    assert not stray, stray


def test_scan_tells_element_access_from_width_dispatch():
    """the vectorised row loads and the fill-kernel dispatch switch on the width too, but do not touch one element"""
    found = element_switches()
    texts = dict(sources())
    assert "launch_fill_elems" in [fn for fn, _ in width_switches(texts["binby.cu"])]
    assert ("binby.cu", "launch_fill_elems") not in found
    vec_branch = next(body for fn, body in width_switches(texts["device_utils.cuh"]) if fn == "load4_raw" and "ldcs128" in body)
    assert not any(ELEMENT[w].search(vec_branch) for w in ELEMENT)
    assert ("take.cu", "load_index") in found  # the scan sees the signed index read; it is exempt by name, not missed


# the key table's probe rule: a home slot hash64(key) & mask, a linear step (h + 1) & mask, a claim of a free slot by CAS
HOME_SLOT = re.compile(r"\bhash64\((?:[^()]|\([^()]*\))*\)\s*&\s*[\w.\[\]>-]*mask\b")
PROBE_STEP = re.compile(r"\(\s*\w+\s*\+\s*1\s*\)\s*&\s*[\w.\[\]>-]*mask\b")
SLOT_CLAIM = re.compile(r"\batomicCAS\(\s*&[^,;]*\.key\s*,\s*SET_EMPTY\b")
# nunique.cu's table of 128-bit (cell, value) pairs: another layout, claimed with a 128-bit CAS
OTHER_TABLES = {("nunique.cu", "pair_insert")}


def sites(pattern):
    return [(name, enclosing_function(text, m.start())) for name, text in sources() for m in pattern.finditer(text)]


def test_key_table_is_probed_only_in_settable():
    for pattern in (HOME_SLOT, PROBE_STEP, SLOT_CLAIM):
        found = sites(pattern)
        stray = [site for site in found if site[0] != "settable.cuh" and site not in OTHER_TABLES]
        assert not stray, (pattern.pattern, stray)
        assert any(name == "settable.cuh" for name, _ in found), pattern.pattern


def test_probe_scans_see_the_pair_table():
    """nunique.cu's pair table steps and hashes like the key table: it is exempt by name, not missed"""
    assert ("nunique.cu", "pair_insert") in sites(HOME_SLOT)
    assert ("nunique.cu", "pair_insert") in sites(PROBE_STEP)


def test_host_reads_the_overflow_flag_in_one_function():
    """only the insert-pass driver (set_insert_pass) reads CTR_OVERFLOW on the host, grows the table and redoes the pass"""
    host = set()
    for name, text in sources():
        for m in re.finditer(r"\bCTR_OVERFLOW\b", text):
            fn, line = enclosing_definition(text, m.start())
            if fn and not re.search(r"__global__|__device__", line):
                host.add((name, fn))
    assert host == {("hashset.cu", "set_insert_pass")}, host
