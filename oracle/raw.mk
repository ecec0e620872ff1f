# oracle/raw.mk -- tests/abi/raw_driver.c against the REFERENCE's own src/filter.h, linked to libka9qgpu.so, into
# _ref/raw_driver_refhdr.so: a driver that declares the raw-ingest extensions itself, as a patched radiod would, binds
# to the library (tests/test_gpu_raw_ingest.py).  TEST INFRASTRUCTURE, NOT PRODUCT.  Only where the reference sources
# exist; the .so is git-ignored and travels with the tree.
REFERENCE ?= /root/reference
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CC ?= gcc
KGPU := $(HERE)../ka9q_radio_b200/libka9qgpu.so

ifneq ($(wildcard $(REFERENCE)/src/filter.h),)
all: $(HERE)_ref/raw_driver_refhdr.so
$(HERE)_ref/raw_driver_refhdr.so: $(HERE)../tests/abi/raw_driver.c $(REFERENCE)/src/filter.h $(KGPU)
	@mkdir -p $(HERE)_ref
	$(CC) -std=gnu11 -O2 -fPIC -shared -pthread -w -DFILTER_HEADER='"filter.h"' -I$(HERE)stubs -iquote $(REFERENCE)/src \
	    -o $@ $< -L$(HERE)../ka9q_radio_b200 -lka9qgpu -Wl,-rpath,'$$ORIGIN/../../ka9q_radio_b200'
else
all:
	@echo "oracle: $(REFERENCE) not present; keeping prebuilt _ref/ (if any)"
endif
.PHONY: all
