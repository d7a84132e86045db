# Builds _ref/libgbref_lgc.so, the reference's own CPU checker of local graph
# clustering (ref_lgc.cpp), from the sources under $(REF) when that directory exists
# (elsewhere a file built earlier is kept).  Flags as the other reference checkers'
# (Makefile, target ref): no -march, so the host compiler emits no fused multiply-add,
# as in the reference's own build.
#   make -C oracle -f ref_lgc.mk
REF  ?= /root/reference
SHIM ?= ../graphblast_b200/csrc/shim
ORC_CXX := $(shell command -v /usr/bin/g++ || echo g++)

all:
	@if [ -d $(REF)/graphblas ]; then \
	  mkdir -p _ref && \
	  $(ORC_CXX) -O3 -fPIC -shared -std=c++14 -fpermissive -w -fvisibility=hidden -I $(REF) -I $(SHIM) \
	      -o _ref/libgbref_lgc.so ref_lgc.cpp && echo "built _ref/libgbref_lgc.so"; \
	else echo "reference sources not present: keeping prebuilt _ref/libgbref_lgc.so (if any)"; fi

.PHONY: all
