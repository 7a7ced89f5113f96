// oracle/ref_strlist_shim.cpp — TEST INFRASTRUCTURE ONLY.
// glue only: registers the reference's StringSequence / StringList64 (src/superstring.hpp, unmodified, included from where it lies)
// with pybind11, so that the compiled, unmodified superagg module (oracle/_ref) accepts this module's string lists in
// AggList_string_int64.set_data and hands its get_result() StringList64 back to Python.  The reference binds these classes in its
// superstrings module, which needs pcre and is not built here; pybind11 shares registered types between modules built with the same
// pybind11 and compiler, which is what makes the hand-over work.
#include "superstring.hpp"
namespace py = pybind11;


PYBIND11_MODULE(strlist_shim, m) {
    py::class_<StringSequence, std::shared_ptr<StringSequence>>(m, "StringSequence");
    py::class_<StringList64, std::shared_ptr<StringList64>, StringSequence>(m, "StringList64");
    // (int64 offsets[n + 1], bytes, uint8 null mask or None: 1 = null) -> StringList64, offsets taken as they are (absolute)
    m.def("make", [](py::array_t<int64_t> offsets, py::array_t<uint8_t> bytes, py::object mask) {
        const int64_t n = offsets.shape(0) - 1;
        const int64_t nbytes = bytes.shape(0);
        auto sl = std::make_shared<StringList64>(nbytes, n);
        std::copy(bytes.data(), bytes.data() + nbytes, (uint8_t *)sl->bytes);
        for (int64_t i = 0; i <= n; i++)
            sl->indices[i] = offsets.at(i);
        if (!mask.is_none()) {
            py::array_t<uint8_t> mk = mask.cast<py::array_t<uint8_t>>();
            sl->ensure_null_bitmap();
            for (int64_t i = 0; i < n; i++)
                if (mk.at(i))
                    sl->set_null(i);
        }
        return sl;
    });
    // StringList64 -> (int64 offsets[n + 1] from 0, bytes, uint8 validity: 1 = string)
    m.def("buffers", [](std::shared_ptr<StringList64> sl) {
        const int64_t n = sl->length;
        py::array_t<int64_t> off(n + 1);
        for (int64_t i = 0; i <= n; i++)
            off.mutable_at(i) = sl->indices[i] - sl->indices[0];
        const int64_t nb = sl->indices[n] - sl->indices[0];
        py::array_t<uint8_t> by(nb);
        std::copy(sl->bytes + sl->indices[0] - sl->offset, sl->bytes + sl->indices[0] - sl->offset + nb, (char *)by.mutable_data());
        py::array_t<uint8_t> valid(n);
        for (int64_t i = 0; i < n; i++)
            valid.mutable_at(i) = !sl->is_null(i);
        return py::make_tuple(off, by, valid);
    });
}
