# Projection-selection test infrastructure, built after the main recipe (make -C oracle; make -C oracle -f tracker.mk):
#
#   _build/libsrl_tracker_oracle.so  the oracle of the map tracker's selection: srl_oracle.cpp as it is + the entry points of
#                                    srl_tracker_oracle.cpp (orc_color_select, orc_color_gather); always buildable
#   _ref/libsrl_tracker_ref.so       the reference's own selectPointsForProjection / refreshPointsForProjection: the unmodified
#                                    reference objects the main recipe compiled into _ref/obj/, srl_reference_harness.cpp and
#                                    srl_tracker_harness.cpp (the C entry points)
#                                    (only when the reference tree is present; a prebuilt library is kept otherwise)
include Makefile
.DEFAULT_GOAL := tracker

TRK_OBJS = $(addprefix _ref/obj/,$(addsuffix .o,$(REF_SRCS)))

tracker: _build/libsrl_tracker_oracle.so tracker_ref

_build/libsrl_tracker_oracle.so: srl_tracker_oracle.cpp srl_oracle.cpp srl_oracle.h
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -o $@ srl_tracker_oracle.cpp

tracker_ref:
	@if [ -f $(REF_ROOT)/src/rgbMapTracker.cpp ] && [ -f _ref/libsrl_reference.so ]; then \
	  if [ ! -f _ref/libsrl_tracker_ref.so ] || [ _ref/libsrl_reference.so -nt _ref/libsrl_tracker_ref.so ] || [ srl_tracker_harness.cpp -nt _ref/libsrl_tracker_ref.so ]; then \
	    echo "$(CXX) reference objects + srl_reference_harness.cpp + srl_tracker_harness.cpp -> _ref/libsrl_tracker_ref.so" && \
	    $(CXX) $(REF_FLAGS) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL -o _ref/libsrl_tracker_ref.so srl_reference_harness.cpp srl_tracker_harness.cpp \
	      $(TRK_OBJS) || exit 1 ; \
	  fi ; \
	else echo "tracker_ref: reference tree absent: keeping prebuilt _ref/libsrl_tracker_ref.so (if any)"; fi

.PHONY: tracker tracker_ref
