# oracle/narrowband.mk -- the narrowband spectrum analyzer's checkers.  TEST INFRASTRUCTURE, NOT PRODUCT.
#
#   libkanarrowband.so           our restatement of narrowband_poll and its ring (narrowband_oracle.c + fft_cpu.c)
#   _ref/libka9qnarrowband.so    the reference's OWN spectrum.c, #included unmodified from where it lies by
#                                ref_narrowband.c, with the FFTW shim, the filter path objects of Makefile and stubs
#
# Built by __graft_entry__.build() after oracle/Makefile and spectrum.mk; the _ref target needs $(REFERENCE) and the
# objects those leave in _ref/.
REFERENCE ?= /root/reference
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CC ?= gcc

REF_CFLAGS = -std=gnu11 -D_GNU_SOURCE=1 -O3 -DNDEBUG=1 -march=native -funsafe-math-optimizations \
             -fno-math-errno -freciprocal-math -fno-trapping-math -ffp-contract=fast -fcx-limited-range \
             -fPIC -pthread -w
# the restatement is compiled with the reference's flags so that its bin arithmetic is the reference's
NB_CFLAGS = -std=gnu11 -D_GNU_SOURCE=1 -O3 -march=native -fno-math-errno -ffp-contract=fast -fcx-limited-range -fPIC \
            -pthread -Wall -Wextra

all: $(HERE)libkanarrowband.so ref

$(HERE)libkanarrowband.so: $(HERE)narrowband_oracle.c $(HERE)fft_cpu.c $(HERE)fft_cpu.h $(HERE)fft_cpu_impl.h
	$(CC) $(NB_CFLAGS) -shared -o $@ $(HERE)narrowband_oracle.c $(HERE)fft_cpu.c -lm

REF_OBJS = $(addprefix $(HERE)_ref/,filter.o window.o misc.o sched.o sincospi.o sincospif.o osc.o gauss.o airspy-unpack.o \
           fftw_shim.o fft_cpu.o ref_spectrum_stubs.o)

ifneq ($(wildcard $(REFERENCE)/src/spectrum.c),)
ref: $(HERE)_ref/libka9qnarrowband.so
$(HERE)_ref/ref_narrowband.o: $(HERE)ref_narrowband.c $(REFERENCE)/src/spectrum.c
	@mkdir -p $(HERE)_ref
	$(CC) $(REF_CFLAGS) -I$(HERE)stubs -iquote $(REFERENCE)/src -c -o $@ $<
$(HERE)_ref/ref_spectrum_stubs.o: $(HERE)ref_spectrum_stubs.c
	@mkdir -p $(HERE)_ref
	$(CC) -std=gnu11 -O1 -fPIC -c -o $@ $<
$(HERE)_ref/libka9qnarrowband.so: $(HERE)_ref/ref_narrowband.o $(REF_OBJS)
	$(CC) -shared -pthread -Wl,--no-undefined -o $@ $^ -lm -ldl
else
ref:
	@echo "oracle: $(REFERENCE) not present; keeping prebuilt _ref/ (if any)"
endif

clean:
	rm -f $(HERE)libkanarrowband.so $(HERE)_ref/ref_narrowband.o $(HERE)_ref/libka9qnarrowband.so
.PHONY: all ref clean
