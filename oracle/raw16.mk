# oracle/raw16.mk -- the raw 16-bit ingest checkers (HydraSDR int16 / uint16, bladeRF SC16 Q11, SDRplay's planar I/Q).
# TEST INFRASTRUCTURE, NOT PRODUCT.
#
#   _ref/libka9qraw16.so         the reference's OWN hydrasdr.c and bladerf.c, #included unmodified from where they lie
#                                by ref_hydrasdr.c and ref_bladerf.c, compiled with the reference's flags, on the filter
#                                path objects oracle/Makefile leaves in _ref/ (not sched.o: the scheduling helpers are
#                                no-op stubs here)
#   _ref/raw16_driver_refhdr.so  tests/abi/raw16_driver.c against the reference's own src/filter.h, linked to
#                                libka9qgpu.so: a driver that declares the extensions itself, as a patched radiod would
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
REF_OBJS = $(addprefix $(HERE)_ref/,filter.o window.o misc.o sincospi.o sincospif.o osc.o gauss.o airspy-unpack.o \
                                    fftw_shim.o fft_cpu.o)

ifneq ($(wildcard $(REFERENCE)/src/hydrasdr.c),)
all: $(HERE)_ref/libka9qraw16.so $(HERE)_ref/raw16_driver_refhdr.so
$(HERE)_ref/ref_hydrasdr.o: $(HERE)ref_hydrasdr.c $(REFERENCE)/src/hydrasdr.c $(HERE)stubs/libhydrasdr/hydrasdr.h
	@mkdir -p $(HERE)_ref
	$(CC) $(REF_CFLAGS) -I$(HERE)stubs -iquote $(REFERENCE)/src -c -o $@ $<
$(HERE)_ref/ref_bladerf.o: $(HERE)ref_bladerf.c $(REFERENCE)/src/bladerf.c $(HERE)stubs/libbladeRF.h
	@mkdir -p $(HERE)_ref
	$(CC) $(REF_CFLAGS) -I$(HERE)stubs -iquote $(REFERENCE)/src -c -o $@ $<
$(HERE)_ref/ref_raw16_stubs.o: $(HERE)ref_raw16_stubs.c
	@mkdir -p $(HERE)_ref
	$(CC) -std=gnu11 -O1 -fPIC -c -o $@ $<
$(HERE)_ref/libka9qraw16.so: $(HERE)_ref/ref_hydrasdr.o $(HERE)_ref/ref_bladerf.o $(HERE)_ref/ref_raw16_stubs.o $(REF_OBJS)
	$(CC) -shared -pthread -Wl,--no-undefined -o $@ $^ -lm -ldl
$(HERE)_ref/raw16_driver_refhdr.so: $(HERE)../tests/abi/raw16_driver.c $(REFERENCE)/src/filter.h $(KGPU)
	@mkdir -p $(HERE)_ref
	$(CC) -std=gnu11 -O2 -fPIC -shared -pthread -w -DFILTER_HEADER='"filter.h"' -I$(HERE)stubs -iquote $(REFERENCE)/src \
	    -o $@ $< -L$(HERE)../ka9q_radio_b200 -lka9qgpu -Wl,-rpath,'$$ORIGIN/../../ka9q_radio_b200'
else
all:
	@echo "oracle: $(REFERENCE) not present; keeping prebuilt _ref/ (if any)"
endif
.PHONY: all
