# oracle/float.mk -- the float ingest checkers (AirspyHF+, Fobos, HydraSDR FLOAT32_REAL / FLOAT32_IQ).
# TEST INFRASTRUCTURE, NOT PRODUCT.
#
#   _ref/libka9qfloat.so         the reference's OWN airspyhf.c, fobos.c and hydrasdr.c, #included unmodified from where
#                                they lie by ref_airspyhf.c, ref_fobos.c and ref_hydrasdr_float.c, compiled with the
#                                reference's flags, on the filter path objects oracle/Makefile leaves in _ref/ (not
#                                sched.o: the scheduling helpers are no-op stubs here)
#   _ref/float_driver_refhdr.so  tests/abi/float_driver.c against the reference's own src/filter.h, linked to
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
SHIMS = airspyhf fobos hydrasdr_float

ifneq ($(wildcard $(REFERENCE)/src/airspyhf.c),)
all: $(HERE)_ref/libka9qfloat.so $(HERE)_ref/float_driver_refhdr.so
$(HERE)_ref/ref_airspyhf.o: $(HERE)ref_airspyhf.c $(REFERENCE)/src/airspyhf.c $(HERE)stubs/libairspyhf/airspyhf.h
$(HERE)_ref/ref_fobos.o: $(HERE)ref_fobos.c $(REFERENCE)/src/fobos.c $(HERE)stubs/fobos.h
$(HERE)_ref/ref_hydrasdr_float.o: $(HERE)ref_hydrasdr_float.c $(REFERENCE)/src/hydrasdr.c $(HERE)stubs/libhydrasdr/hydrasdr.h
$(addprefix $(HERE)_ref/ref_,$(addsuffix .o,$(SHIMS))): $(HERE)_ref/ref_%.o:
	@mkdir -p $(HERE)_ref
	$(CC) $(REF_CFLAGS) -I$(HERE)stubs -iquote $(REFERENCE)/src -c -o $@ $(HERE)ref_$*.c
$(HERE)_ref/ref_float_stubs.o: $(HERE)ref_float_stubs.c
	@mkdir -p $(HERE)_ref
	$(CC) -std=gnu11 -O1 -fPIC -c -o $@ $<
$(HERE)_ref/libka9qfloat.so: $(addprefix $(HERE)_ref/ref_,$(addsuffix .o,$(SHIMS))) $(HERE)_ref/ref_float_stubs.o $(REF_OBJS)
	$(CC) -shared -pthread -Wl,--no-undefined -o $@ $^ -lm -ldl
$(HERE)_ref/float_driver_refhdr.so: $(HERE)../tests/abi/float_driver.c $(HERE)../tests/abi/raw_driver.c $(REFERENCE)/src/filter.h $(KGPU)
	@mkdir -p $(HERE)_ref
	$(CC) -std=gnu11 -O2 -fPIC -shared -pthread -w -DFILTER_HEADER='"filter.h"' -I$(HERE)stubs -iquote $(REFERENCE)/src \
	    -o $@ $< -L$(HERE)../ka9q_radio_b200 -lka9qgpu -Wl,-rpath,'$$ORIGIN/../../ka9q_radio_b200'
else
all:
	@echo "oracle: $(REFERENCE) not present; keeping prebuilt _ref/ (if any)"
endif
.PHONY: all
