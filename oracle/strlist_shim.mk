# oracle/strlist_shim.mk — TEST INFRASTRUCTURE ONLY.  Builds oracle/_ref/strlist_shim*.so: the reference's StringSequence /
# StringList64 (src/superstring.hpp, unmodified, included where it lies) registered with pybind11 by ref_strlist_shim.cpp, so that
# the compiled superagg's AggList_string_int64 can be fed and read from Python (tests/golden/make_golden_agglist_string.py).
# Flags, paths and the string_utils object come from the main recipe (Makefile).  Only built where $(REF) exists.
#
# usage:  make -C oracle ref && make -C oracle -f strlist_shim.mk
include Makefile

.DEFAULT_GOAL := strlist_shim

strlist_shim: _ref/strlist_shim$(EXT)

_ref/strlist_shim$(EXT): ref_strlist_shim.cpp _ref/obj/utl_string_utils.o $(REF)/src/superstring.hpp
	$(CXX) $(REF_CXXFLAGS) -I$(REF)/src -shared -o $@ ref_strlist_shim.cpp _ref/obj/utl_string_utils.o

.PHONY: strlist_shim
