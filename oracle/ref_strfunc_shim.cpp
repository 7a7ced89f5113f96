// oracle/ref_strfunc_shim.cpp — TEST INFRASTRUCTURE ONLY.
// glue only: calls the inline string predicates and measures of the reference's StringSequenceBase (src/superstring.hpp, unmodified,
// included from where it lies) on a StringList64 built from plain numpy buffers: startswith, endswith, find (left and right), equals,
// equals2, len and byte_length.  search and count live in src/strings.cpp, which needs pcre and boost; tests/str_expr_oracle.py
// restates them.
#include "superstring.hpp"
namespace py = pybind11;

// (int64 offsets[n + 1] as they are, bytes, uint8 null mask or None: 1 = null) -> StringList64
static std::shared_ptr<StringList64> make_list(py::array_t<int64_t> offsets, py::array_t<uint8_t> bytes, py::object mask) {
    const int64_t n = offsets.shape(0) - 1;
    const int64_t nbytes = bytes.shape(0);
    auto sl = std::make_shared<StringList64>(nbytes, n);
    std::copy(bytes.data(), bytes.data() + nbytes, (uint8_t *)sl->bytes);
    for (int64_t i = 0; i <= n; i++)
        sl->indices[i] = offsets.at(i);
    if (!mask.is_none()) {
        py::array_t<uint8_t> m = mask.cast<py::array_t<uint8_t>>();
        sl->ensure_null_bitmap();
        for (int64_t i = 0; i < n; i++)
            if (m.at(i))
                sl->set_null(i);
    }
    return sl;
}

PYBIND11_MODULE(strfunc_shim, m) {
    m.def("startswith", [](py::array_t<int64_t> o, py::array_t<uint8_t> b, py::object mk, py::bytes p) { return make_list(o, b, mk)->startswith(p); });
    m.def("endswith", [](py::array_t<int64_t> o, py::array_t<uint8_t> b, py::object mk, py::bytes p) { return make_list(o, b, mk)->endswith(p); });
    // end = None: to the end of the row (vaex/functions.py str_find passes till_end)
    m.def("find", [](py::array_t<int64_t> o, py::array_t<uint8_t> b, py::object mk, py::bytes p, int64_t start, py::object end, bool left) {
        return make_list(o, b, mk)->find(p, start, end.is_none() ? 0 : end.cast<int64_t>(), end.is_none(), left);
    });
    m.def("equals", [](py::array_t<int64_t> o, py::array_t<uint8_t> b, py::object mk, py::bytes p) { return make_list(o, b, mk)->equals(p); });
    m.def("equals2", [](py::array_t<int64_t> o, py::array_t<uint8_t> b, py::object mk, py::array_t<int64_t> o2, py::array_t<uint8_t> b2, py::object mk2) {
        auto other = make_list(o2, b2, mk2);
        return make_list(o, b, mk)->equals2(other.get());
    });
    m.def("len", [](py::array_t<int64_t> o, py::array_t<uint8_t> b, py::object mk) { auto sl = make_list(o, b, mk);
        return static_cast<StringSequenceBase *>(sl.get())->len(); });
    m.def("byte_length", [](py::array_t<int64_t> o, py::array_t<uint8_t> b, py::object mk) { auto sl = make_list(o, b, mk);
        return static_cast<StringSequenceBase *>(sl.get())->byte_length(); });
}
