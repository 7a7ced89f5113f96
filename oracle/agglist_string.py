"""AggListString (src/agg_list.cpp:122-222) restated in plain Python — TEST INFRASTRUCTURE ONLY, next to the oracle's other
restatements (oracle.py); pinned against the compiled reference by tests/golden/agglist_string_golden.npz."""
import numpy as np


def agg_list_string(cells, strings, ncells=None, dropnan=False, dropnull=False, mask=None):
    """AggListString (src/agg_list.cpp:183-197 aggregate, :141-181 get_result) restated: per cell of the flat grid the strings of the
    rows in arrival order; a null string (None) is pushed as a null AT ITS ARRIVAL POSITION (:191-195, StringList::push_null pushes
    an empty string and clears its validity bit, src/superstring.hpp:729-734) unless dropnull.  `dropnan` has no effect (never read
    in AggListString).  `mask`, the data mask, is accepted and IGNORED: AggBaseString::set_data_mask stores it and nothing reads it
    (src/agg_base.hpp:192-199) — a reference quirk kept like AggList's mask[r % 1024].  The order of the bin() calls is the arrival
    order, so no call ranges are needed.  Returns the arrow large_list<large_string> buffers: (list offsets int64[ncells + 1],
    string offsets int64[total + 1], bytes uint8, validity uint8[total] (1 = string, 0 = null))."""
    del dropnan, mask
    cells = np.asarray(cells, dtype=np.int64)
    ncells = int(cells.max()) + 1 if ncells is None else int(ncells)
    lists = [[] for _ in range(ncells)]
    for c, s in zip(cells.tolist(), strings):
        if s is not None:
            lists[c].append(s.encode("utf8") if isinstance(s, str) else bytes(s))
        elif not dropnull:
            lists[c].append(None)
    list_offsets = np.zeros(ncells + 1, np.int64)
    list_offsets[1:] = np.cumsum([len(lst) for lst in lists])
    flat = [s for lst in lists for s in lst]
    str_offsets = np.zeros(len(flat) + 1, np.int64)
    str_offsets[1:] = np.cumsum([0 if s is None else len(s) for s in flat])
    data = np.frombuffer(b"".join(s for s in flat if s is not None), dtype=np.uint8).copy()
    valid = np.array([s is not None for s in flat], np.uint8)
    return list_offsets, str_offsets, data, valid
