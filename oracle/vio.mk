# Camera-update test infrastructure, built after the main recipe (make -C oracle; make -C oracle -f vio.mk):
#
#   _ref/libsrl_vio_ref.so   the reference's own imageProcessing::vioEsikf / vioPhotometric: src/imageProcessing.cpp compiled
#                            unmodified over shim/ with shim_vio/srl_vio_prelude.h force-included (the OpenCV calls of its image
#                            steps, which the tests never run, and Eigen's 1 x 1 product to scalar), the unmodified reference
#                            objects the main recipe compiled into _ref/obj/, srl_reference_harness.cpp with its stand-ins for
#                            imageProcessing's members made weak (objcopy), and srl_vio_harness.cpp (the C entry points)
#                            (only when the reference tree is present; a prebuilt library is kept otherwise)
include Makefile
.DEFAULT_GOAL := vio

VIO_OBJS = $(addprefix _ref/obj/,$(addsuffix .o,$(REF_SRCS)))

vio:
	@if [ -f $(REF_ROOT)/src/imageProcessing.cpp ] && [ -f _ref/libsrl_reference.so ] && command -v objcopy >/dev/null; then \
	  if [ ! -f _ref/libsrl_vio_ref.so ] || [ _ref/libsrl_reference.so -nt _ref/libsrl_vio_ref.so ] || [ srl_vio_harness.cpp -nt _ref/libsrl_vio_ref.so ] || \
	     [ shim_vio/srl_vio_prelude.h -nt _ref/libsrl_vio_ref.so ] || [ $(REF_ROOT)/src/imageProcessing.cpp -nt _ref/libsrl_vio_ref.so ]; then \
	    mkdir -p _ref/obj_vio && \
	    $(CXX) $(REF_FLAGS) -include shim_vio/srl_vio_prelude.h -c $(REF_ROOT)/src/imageProcessing.cpp -o _ref/obj_vio/imageProcessing.o && \
	    $(CXX) $(REF_FLAGS) -c srl_reference_harness.cpp -o _ref/obj_vio/srl_reference_harness.o && \
	    syms=$$(nm _ref/obj_vio/srl_reference_harness.o | awk '$$2=="T" && $$3 ~ /15imageProcessing/ {printf "--weaken-symbol=%s ", $$3}') && \
	    objcopy $$syms _ref/obj_vio/srl_reference_harness.o && \
	    echo "$(CXX) imageProcessing.cpp + reference objects + srl_reference_harness.o (imageProcessing weakened) + srl_vio_harness.cpp -> _ref/libsrl_vio_ref.so" && \
	    $(CXX) $(REF_FLAGS) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL -o _ref/libsrl_vio_ref.so srl_vio_harness.cpp \
	      _ref/obj_vio/srl_reference_harness.o _ref/obj_vio/imageProcessing.o $(VIO_OBJS) || exit 1 ; \
	  fi ; \
	else echo "vio: reference tree, _ref/libsrl_reference.so or objcopy absent: keeping prebuilt _ref/libsrl_vio_ref.so (if any)"; fi

.PHONY: vio
