# cloudProcessing test infrastructure, built after the main recipe (make -C oracle -f cloud_processing.mk):
#
#   _ref/libsrl_sort_probe.so               std::sort's permutation as this compiler's libstdc++ leaves it (srl_sort_probe.cpp)
#   _ref/libsrl_cloud_processing_ref.so     the reference's own cloudProcessing: src/cloudProcessing.cpp compiled unmodified over
#                                           shim/ with shim_cp/srl_cloud_processing_prelude.h force-included (pcl::fromROSMsg and
#                                           the registered point fields), the reference's utility.o from the main recipe (the
#                                           time_list comparators) and srl_cloud_processing_harness.cpp (C entry points).  A library
#                                           of its own: srl_reference_harness.cpp stubs cloudProcessing's methods.
#                                           (only when the reference tree is present; a prebuilt library is kept otherwise)
include Makefile
.DEFAULT_GOAL := cloud_processing

cloud_processing: sort_probe cloud_processing_ref

sort_probe: _ref/libsrl_sort_probe.so
_ref/libsrl_sort_probe.so: srl_sort_probe.cpp
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -o $@ srl_sort_probe.cpp

CP_FLAGS = $(REF_FLAGS) -include shim_cp/srl_cloud_processing_prelude.h
cloud_processing_ref:
	@if [ -f $(REF_ROOT)/src/cloudProcessing.cpp ] && [ -f _ref/obj/utility.o ]; then \
	  if [ ! -f _ref/libsrl_cloud_processing_ref.so ] || [ _ref/obj/utility.o -nt _ref/libsrl_cloud_processing_ref.so ] || \
	     [ srl_cloud_processing_harness.cpp -nt _ref/libsrl_cloud_processing_ref.so ] || [ shim_cp/srl_cloud_processing_prelude.h -nt _ref/libsrl_cloud_processing_ref.so ] || \
	     [ $(REF_ROOT)/src/cloudProcessing.cpp -nt _ref/libsrl_cloud_processing_ref.so ]; then \
	    mkdir -p _ref/obj_cp && \
	    $(CXX) $(CP_FLAGS) -c $(REF_ROOT)/src/cloudProcessing.cpp -o _ref/obj_cp/cloudProcessing.o && \
	    echo "$(CXX) cloudProcessing.cpp + utility.o + srl_cloud_processing_harness.cpp -> _ref/libsrl_cloud_processing_ref.so" && \
	    $(CXX) $(CP_FLAGS) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL -Wl,-z,defs -o _ref/libsrl_cloud_processing_ref.so \
	      srl_cloud_processing_harness.cpp _ref/obj_cp/cloudProcessing.o _ref/obj/utility.o || exit 1 ; \
	  fi ; \
	else echo "cloud_processing_ref: reference tree or _ref/obj/utility.o absent: keeping prebuilt _ref/libsrl_cloud_processing_ref.so (if any)"; fi

.PHONY: cloud_processing sort_probe cloud_processing_ref
