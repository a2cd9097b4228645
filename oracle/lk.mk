# Pyramidal Lucas-Kanade test infrastructure, built after the main recipe (make -C oracle -f lk.mk):
#
#   _ref/libsrl_lk_ref.so   the reference's own LKOpticalFlowKernel: src/lkpyramid.cpp compiled unmodified from where it lies, over
#                           the OpenCV stand-in of shim_lk/ (ahead of shim/ on this library's include path only), +
#                           srl_lk_harness.cpp (the C entry points, tests/lk_ref.py)
#                           (only when the reference tree is present; a prebuilt library is kept otherwise)
include Makefile
.DEFAULT_GOAL := lk

LK_FLAGS = -std=c++14 -O3 -fPIC -pthread -ffp-contract=off -w -include shim_lk/srl_lk_prelude.h -Ishim_lk -Ishim -I. -I$(REF_ROOT)/include
LK_DEPS = shim_lk/srl_lk_cv.h shim_lk/srl_lk_prelude.h srl_lk_harness.cpp

lk:
	@if [ -f $(REF_ROOT)/src/lkpyramid.cpp ]; then \
	  mkdir -p _ref && \
	  if [ ! -f _ref/libsrl_lk_ref.so ] || [ $(REF_ROOT)/src/lkpyramid.cpp -nt _ref/libsrl_lk_ref.so ] || [ $(REF_ROOT)/include/lkpyramid.h -nt _ref/libsrl_lk_ref.so ] || \
	     [ -n "$$(find $(LK_DEPS) shim_lk -newer _ref/libsrl_lk_ref.so -type f | head -1)" ]; then \
	    echo "$(CXX) $(REF_ROOT)/src/lkpyramid.cpp + srl_lk_harness.cpp -> _ref/libsrl_lk_ref.so" && \
	    $(CXX) $(LK_FLAGS) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL -o _ref/libsrl_lk_ref.so $(REF_ROOT)/src/lkpyramid.cpp srl_lk_harness.cpp || exit 1 ; \
	  fi ; \
	else echo "lk: reference tree absent: keeping prebuilt _ref/libsrl_lk_ref.so (if any)"; fi

.PHONY: lk
