# Publication test infrastructure, built after the main recipe (make -C oracle; make -C oracle -f publish.mk):
#
#   _build/libsrl_publish_oracle.so  the oracle of the published maps: srl_oracle.cpp as it is + the entry points of
#                                    srl_publish_oracle.cpp (orc_map_add_points_published, orc_color_export); always buildable
#   _ref/libsrl_publish_ref.so       the reference's own addPointsToMap / pubColorPoints / saveColorPoints with the clouds they
#                                    publish and save observable: src/lioOptimization.cpp compiled unmodified with
#                                    srl_publish_capture.h force-included (pcl::toROSMsg / pcl::io::savePCDFileBinary of the
#                                    stand-in specialized for the published cloud types), the other reference objects the main
#                                    recipe compiled into _ref/obj/, srl_reference_harness.cpp and srl_publish_harness.cpp (the
#                                    specializations and the C entry points)
#                                    (only when the reference tree is present; a prebuilt library is kept otherwise)
include Makefile
.DEFAULT_GOAL := publish

PUB_OBJS = $(addprefix _ref/obj/,$(addsuffix .o,$(filter-out lioOptimization,$(REF_SRCS)))) _ref/obj_publish/lioOptimization.o
PUB_FLAGS = $(REF_FLAGS) -include srl_publish_capture.h

publish: _build/libsrl_publish_oracle.so publish_ref

_build/libsrl_publish_oracle.so: srl_publish_oracle.cpp srl_oracle.cpp srl_oracle.h
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -o $@ srl_publish_oracle.cpp

publish_ref:
	@if [ -f $(REF_ROOT)/src/lioOptimization.cpp ] && [ -f _ref/libsrl_reference.so ]; then \
	  mkdir -p _ref/obj_publish && \
	  if [ ! -f _ref/obj_publish/lioOptimization.o ] || [ _ref/obj/lioOptimization.o -nt _ref/obj_publish/lioOptimization.o ] || [ srl_publish_capture.h -nt _ref/obj_publish/lioOptimization.o ]; then \
	    echo "$(CXX) -include srl_publish_capture.h lioOptimization.cpp -> _ref/obj_publish/lioOptimization.o" && \
	    $(CXX) $(PUB_FLAGS) -c $(REF_ROOT)/src/lioOptimization.cpp -o _ref/obj_publish/lioOptimization.o || exit 1 ; \
	  fi ; \
	  if [ ! -f _ref/libsrl_publish_ref.so ] || [ _ref/obj_publish/lioOptimization.o -nt _ref/libsrl_publish_ref.so ] || [ _ref/libsrl_reference.so -nt _ref/libsrl_publish_ref.so ] || [ srl_publish_harness.cpp -nt _ref/libsrl_publish_ref.so ]; then \
	    echo "$(CXX) reference objects (lioOptimization capturing clouds) + srl_reference_harness.cpp + srl_publish_harness.cpp -> _ref/libsrl_publish_ref.so" && \
	    $(CXX) $(PUB_FLAGS) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL -o _ref/libsrl_publish_ref.so srl_reference_harness.cpp srl_publish_harness.cpp \
	      $(PUB_OBJS) ; \
	  fi ; \
	else echo "publish_ref: reference tree absent: keeping prebuilt _ref/libsrl_publish_ref.so (if any)"; fi

.PHONY: publish publish_ref
