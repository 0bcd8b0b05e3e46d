# make -C oracle -f flooding.mk  ->  oracle/_ref/libsmref_flooding.so (refharness/sweep_flood.cpp: libsmref.so plus the
# sweep-flood driver), compiled as the `ref` target of the Makefile compiles libsmref.so.  TEST INFRASTRUCTURE.
REFERENCE_ROOT ?= /root/reference
CXX ?= g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

all: $(HERE)_ref/libsmref_flooding.so

# -fno-gnu-unique: a process that loads libsmref.so too keeps two separate sets of the reference's globals
$(HERE)_ref/libsmref_flooding.so: $(HERE)refharness/sweep_flood.cpp $(HERE)refharness/harness.cpp $(HERE)refharness/stubs.h $(HERE)refharness/glm/glm.hpp
	@mkdir -p $(HERE)_ref
	$(CXX) -std=c++20 -O2 -w -fPIC -shared -fno-gnu-unique -I$(HERE)refharness -I$(REFERENCE_ROOT) \
	    $(HERE)refharness/sweep_flood.cpp -o $@

.PHONY: all
