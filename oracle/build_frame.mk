# buildFrame test infrastructure, built after the main recipe (make -C oracle; make -C oracle -f build_frame.mk):
#
#   _ref/libsrl_shuffle_probe.so       std::shuffle as this compiler's libstdc++ draws (Lemire's 128-bit multiply)
#   _ref/libsrl_shuffle_probe_div.so   the same compiled with -U__SIZEOF_INT128__ (libstdc++'s division downscale)
#   _ref/libsrl_build_frame_ref.so     the reference's own lioOptimization::buildFrame: the reference objects the main recipe
#                                      compiled into _ref/obj/ + srl_reference_harness.cpp + srl_build_frame_harness.cpp
#                                      (only when the reference tree is present; a prebuilt library is kept otherwise)
include Makefile
.DEFAULT_GOAL := build_frame

build_frame: shuffle_probe build_frame_ref

shuffle_probe: _ref/libsrl_shuffle_probe.so _ref/libsrl_shuffle_probe_div.so
_ref/libsrl_shuffle_probe.so: srl_shuffle_probe.cpp
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -o $@ srl_shuffle_probe.cpp
_ref/libsrl_shuffle_probe_div.so: srl_shuffle_probe.cpp
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -U__SIZEOF_INT128__ -o $@ srl_shuffle_probe.cpp

build_frame_ref:
	@if [ -f $(REF_ROOT)/src/optimize.cpp ] && [ -f _ref/libsrl_reference.so ]; then \
	  if [ ! -f _ref/libsrl_build_frame_ref.so ] || [ _ref/libsrl_reference.so -nt _ref/libsrl_build_frame_ref.so ] || [ srl_build_frame_harness.cpp -nt _ref/libsrl_build_frame_ref.so ]; then \
	    echo "$(CXX) reference objects + srl_reference_harness.cpp + srl_build_frame_harness.cpp -> _ref/libsrl_build_frame_ref.so" && \
	    $(CXX) $(REF_FLAGS) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL -o _ref/libsrl_build_frame_ref.so srl_reference_harness.cpp srl_build_frame_harness.cpp \
	      $(addprefix _ref/obj/,$(addsuffix .o,$(REF_SRCS))) ; \
	  fi ; \
	else echo "build_frame_ref: reference tree absent: keeping prebuilt _ref/libsrl_build_frame_ref.so (if any)"; fi

.PHONY: build_frame shuffle_probe build_frame_ref
