# oracle/siggen_mod.mk -- the modulated (AM / DSB) signal generator checker.  TEST INFRASTRUCTURE, NOT PRODUCT.
#
#   _ref/libka9qsiggenmod.so          the reference's OWN sig_gen.c, #included unmodified from where it lies by
#                                     ref_siggen_mod.c, whose stand-ins script the envelope libsamplerate would produce;
#                                     compiled with the reference's flags, on the filter path objects oracle/Makefile
#                                     leaves in _ref/ and the stubs siggen.mk builds; linked -Bsymbolic like libka9qsiggen.so
#   _ref/siggen_mod_driver_refhdr.so  tests/abi/siggen_mod_driver.c against the reference's own src/filter.h, linked to
#                                     libka9qgpu.so: a driver that declares the extensions itself, as a patched radiod would
#
# Built by __graft_entry__.build() after oracle/Makefile and siggen.mk; only where the reference sources exist.  The .so
# files are git-ignored and travel with the tree.
REFERENCE ?= /root/reference
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CC ?= gcc
KGPU := $(HERE)../ka9q_radio_b200/libka9qgpu.so

REF_CFLAGS = -std=gnu11 -D_GNU_SOURCE=1 -O3 -DNDEBUG=1 -march=native -funsafe-math-optimizations \
             -fno-math-errno -freciprocal-math -fno-trapping-math -ffp-contract=fast -fcx-limited-range \
             -fPIC -pthread -w
REF_OBJS = $(addprefix $(HERE)_ref/,filter.o window.o misc.o sincospi.o sincospif.o osc.o gauss.o fftw_shim.o fft_cpu.o \
             ref_siggen_stubs.o)

ifneq ($(wildcard $(REFERENCE)/src/sig_gen.c),)
all: $(HERE)_ref/libka9qsiggenmod.so $(HERE)_ref/siggen_mod_driver_refhdr.so
$(HERE)_ref/ref_siggen_mod.o: $(HERE)ref_siggen_mod.c $(REFERENCE)/src/sig_gen.c $(HERE)stubs/samplerate.h
	@mkdir -p $(HERE)_ref
	$(CC) $(REF_CFLAGS) -I$(HERE)stubs -iquote $(REFERENCE)/src -c -o $@ $<
$(HERE)_ref/libka9qsiggenmod.so: $(HERE)_ref/ref_siggen_mod.o $(REF_OBJS)
	$(CC) -shared -pthread -Wl,--no-undefined -Wl,-Bsymbolic -o $@ $^ -lm -ldl
$(HERE)_ref/siggen_mod_driver_refhdr.so: $(HERE)../tests/abi/siggen_mod_driver.c $(HERE)../tests/abi/raw_driver.c \
                                         $(REFERENCE)/src/filter.h $(KGPU)
	@mkdir -p $(HERE)_ref
	$(CC) -std=gnu11 -O2 -fPIC -shared -pthread -w -DFILTER_HEADER='"filter.h"' -I$(HERE)stubs -iquote $(REFERENCE)/src \
	    -o $@ $< -L$(HERE)../ka9q_radio_b200 -lka9qgpu -Wl,-rpath,'$$ORIGIN/../../ka9q_radio_b200'
else
all:
	@echo "oracle: $(REFERENCE) not present; keeping prebuilt _ref/ (if any)"
endif
.PHONY: all
