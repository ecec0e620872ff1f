# oracle/small.mk -- the small-master checker.  TEST INFRASTRUCTURE, NOT PRODUCT.
#
#   _ref/small_driver_refhdr.so  tests/abi/small_driver.c (filter_driver.c's sessions, opened with
#                                create_filter_input_small) against the reference's own src/filter.h, linked to
#                                libka9qgpu.so: a driver that declares the extension itself, as a patched radiod would
#
# The reference's own filter.c these sessions are checked against is oracle/Makefile's _ref/libka9qref.so.  Built by
# __graft_entry__.build() after oracle/Makefile; only where the reference sources exist.  The .so is git-ignored and
# travels with the tree.
REFERENCE ?= /root/reference
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CC ?= gcc
KGPU := $(HERE)../ka9q_radio_b200/libka9qgpu.so

ifneq ($(wildcard $(REFERENCE)/src/filter.h),)
all: $(HERE)_ref/small_driver_refhdr.so
$(HERE)_ref/small_driver_refhdr.so: $(HERE)../tests/abi/small_driver.c $(HERE)../tests/abi/filter_driver.c \
                                    $(REFERENCE)/src/filter.h $(KGPU)
	@mkdir -p $(HERE)_ref
	$(CC) -std=gnu11 -O2 -fPIC -shared -pthread -w -DFILTER_HEADER='"filter.h"' -I$(HERE)stubs -iquote $(REFERENCE)/src \
	    -o $@ $< -L$(HERE)../ka9q_radio_b200 -lka9qgpu -Wl,-rpath,'$$ORIGIN/../../ka9q_radio_b200'
else
all:
	@echo "oracle: $(REFERENCE) not present; keeping prebuilt _ref/ (if any)"
endif
.PHONY: all
