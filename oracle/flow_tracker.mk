# Optical-flow tracker bookkeeping test infrastructure, built after the main recipe (make -C oracle -f flow_tracker.mk):
#
#   _ref/libsrl_flow_tracker_ref.so   the reference's own opticalFlowTracker: src/opticalFlowTracker.cpp compiled unmodified over
#                                     shim/ with shim_ft/srl_flow_tracker_prelude.h force-included, the unmodified reference
#                                     objects the main recipe compiled into _ref/obj/, srl_reference_harness.cpp (imageProcessing's
#                                     stand-ins) and srl_flow_tracker_harness.cpp (the stand-ins for LKOpticalFlowKernel and the two
#                                     RANSACs, and the C entry points tests/flow_tracker_ref.py loads)
#                                     (only when the reference tree is present; a prebuilt library is kept otherwise)
include Makefile
.DEFAULT_GOAL := flow_tracker

FT_OBJS = $(addprefix _ref/obj/,$(addsuffix .o,$(REF_SRCS)))

flow_tracker:
	@if [ -f $(REF_ROOT)/src/opticalFlowTracker.cpp ] && [ -f _ref/libsrl_reference.so ]; then \
	  if [ ! -f _ref/libsrl_flow_tracker_ref.so ] || [ _ref/libsrl_reference.so -nt _ref/libsrl_flow_tracker_ref.so ] || \
	     [ srl_flow_tracker_harness.cpp -nt _ref/libsrl_flow_tracker_ref.so ] || [ shim_ft/srl_flow_tracker_prelude.h -nt _ref/libsrl_flow_tracker_ref.so ] || \
	     [ $(REF_ROOT)/src/opticalFlowTracker.cpp -nt _ref/libsrl_flow_tracker_ref.so ]; then \
	    mkdir -p _ref/obj_ft && \
	    $(CXX) $(REF_FLAGS) -include shim_ft/srl_flow_tracker_prelude.h -c $(REF_ROOT)/src/opticalFlowTracker.cpp -o _ref/obj_ft/opticalFlowTracker.o && \
	    $(CXX) $(REF_FLAGS) -c srl_reference_harness.cpp -o _ref/obj_ft/srl_reference_harness.o && \
	    echo "$(CXX) opticalFlowTracker.cpp + reference objects + srl_reference_harness.o + srl_flow_tracker_harness.cpp -> _ref/libsrl_flow_tracker_ref.so" && \
	    $(CXX) $(REF_FLAGS) -include shim_ft/srl_flow_tracker_prelude.h -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL -Wl,-z,defs \
	      -o _ref/libsrl_flow_tracker_ref.so srl_flow_tracker_harness.cpp _ref/obj_ft/srl_reference_harness.o _ref/obj_ft/opticalFlowTracker.o $(FT_OBJS) || exit 1 ; \
	  fi ; \
	else echo "flow_tracker: reference tree or _ref/libsrl_reference.so absent: keeping prebuilt _ref/libsrl_flow_tracker_ref.so (if any)"; fi

.PHONY: flow_tracker
