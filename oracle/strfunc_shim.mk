# oracle/strfunc_shim.mk — TEST INFRASTRUCTURE ONLY.  Builds oracle/_ref/strfunc_shim*.so: the reference's inline string predicates
# and measures (src/superstring.hpp, unmodified, included where it lies) called on numpy buffers by ref_strfunc_shim.cpp, the checker
# of tests/str_expr_oracle.py and the source of tests/golden/str_expr_golden.npz.  Flags, paths and the string_utils object come from
# the main recipe (Makefile).  Only built where $(REF) exists.
#
# usage:  make -C oracle ref && make -C oracle -f strfunc_shim.mk
include Makefile

.DEFAULT_GOAL := strfunc_shim

strfunc_shim: _ref/strfunc_shim$(EXT)

_ref/strfunc_shim$(EXT): ref_strfunc_shim.cpp _ref/obj/utl_string_utils.o $(REF)/src/superstring.hpp
	$(CXX) $(REF_CXXFLAGS) -I$(REF)/src -shared -o $@ ref_strfunc_shim.cpp _ref/obj/utl_string_utils.o

.PHONY: strfunc_shim
