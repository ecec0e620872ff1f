# oracle/iqcorr.mk -- the I/Q correction checkers (HackRF, FUNcube).  TEST INFRASTRUCTURE, NOT PRODUCT.
#
#   _ref/libka9qiqcorr.so         the reference's OWN hackrf.c and funcube.c, #included unmodified from where they lie
#                                 by ref_hackrf.c and ref_funcube.c, compiled with the reference's flags, on the filter
#                                 path objects oracle/Makefile leaves in _ref/ (not sched.o: the scheduling helpers are
#                                 no-op stubs here)
#   _ref/iqcorr_driver_refhdr.so  tests/abi/iqcorr_driver.c against the reference's own src/filter.h, linked to
#                                 libka9qgpu.so: a driver that declares the extensions itself, as a patched radiod would
#
# Built by __graft_entry__.build() after oracle/Makefile; only where the reference sources exist.  The .so files are
# git-ignored and travel with the tree.
REFERENCE ?= /root/reference
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CC ?= gcc
KGPU := $(HERE)../ka9q_radio_b200/libka9qgpu.so

REF_CFLAGS = -std=gnu11 -D_GNU_SOURCE=1 -O3 -DNDEBUG=1 -march=native -funsafe-math-optimizations \
             -fno-math-errno -freciprocal-math -fno-trapping-math -ffp-contract=fast -fcx-limited-range \
             -fPIC -pthread -w
REF_OBJS = $(addprefix $(HERE)_ref/,filter.o window.o misc.o sincospi.o sincospif.o osc.o gauss.o fftw_shim.o fft_cpu.o)

ifneq ($(wildcard $(REFERENCE)/src/hackrf.c),)
all: $(HERE)_ref/libka9qiqcorr.so $(HERE)_ref/iqcorr_driver_refhdr.so
$(HERE)_ref/ref_hackrf.o: $(HERE)ref_hackrf.c $(REFERENCE)/src/hackrf.c $(HERE)stubs/libhackrf/hackrf.h
	@mkdir -p $(HERE)_ref
	$(CC) $(REF_CFLAGS) -I$(HERE)stubs -iquote $(REFERENCE)/src -c -o $@ $<
$(HERE)_ref/ref_funcube.o: $(HERE)ref_funcube.c $(REFERENCE)/src/funcube.c $(HERE)stubs/portaudio.h
	@mkdir -p $(HERE)_ref
	$(CC) $(REF_CFLAGS) -I$(HERE)stubs -iquote $(REFERENCE)/src -c -o $@ $<
$(HERE)_ref/ref_iqcorr_stubs.o: $(HERE)ref_iqcorr_stubs.c
	@mkdir -p $(HERE)_ref
	$(CC) -std=gnu11 -O1 -fPIC -c -o $@ $<
$(HERE)_ref/libka9qiqcorr.so: $(HERE)_ref/ref_hackrf.o $(HERE)_ref/ref_funcube.o $(HERE)_ref/ref_iqcorr_stubs.o $(REF_OBJS)
	$(CC) -shared -pthread -Wl,--no-undefined -o $@ $^ -lm -ldl
$(HERE)_ref/iqcorr_driver_refhdr.so: $(HERE)../tests/abi/iqcorr_driver.c $(REFERENCE)/src/filter.h $(KGPU)
	@mkdir -p $(HERE)_ref
	$(CC) -std=gnu11 -O2 -fPIC -shared -pthread -w -DFILTER_HEADER='"filter.h"' -I$(HERE)stubs -iquote $(REFERENCE)/src \
	    -o $@ $< -L$(HERE)../ka9q_radio_b200 -lka9qgpu -Wl,-rpath,'$$ORIGIN/../../ka9q_radio_b200'
else
all:
	@echo "oracle: $(REFERENCE) not present; keeping prebuilt _ref/ (if any)"
endif
.PHONY: all
