# TEST INFRASTRUCTURE ONLY.  Builds _ref/libdada2ref_filter.so: the reference's src/filter.cpp (C_matchRef, C_matrixEE),
# compiled UNMODIFIED against oracle/stub/Rcpp.h, plus filter_shim.cpp (C-ABI).  A library of its own, next to the
# Makefile's libdada2ref.so.  Only built when $(REF) exists; the .so is git-ignored and travels with the tree.
REF ?= /root/reference
CXX ?= g++
# -O2 like R's default Makevars; no -ffast-math, no -march (no FMA contraction on x86-64)
CXXFLAGS = -O2 -std=c++11 -fPIC -pthread -w

.PHONY: ref
ref:
	@if [ -d $(REF)/src ]; then $(MAKE) -f filter.mk _ref/libdada2ref_filter.so; else echo "no $(REF): keeping prebuilt _ref/libdada2ref_filter.so"; fi

_ref/libdada2ref_filter.so: filter_shim.cpp stub/Rcpp.h filter.mk
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -Istub -I$(REF)/src -c $(REF)/src/filter.cpp -o _ref/ref_filter.o
	$(CXX) $(CXXFLAGS) -Istub -I$(REF)/src -c filter_shim.cpp -o _ref/filter_shim.o
	$(CXX) -shared -pthread -o $@ _ref/ref_filter.o _ref/filter_shim.o -lm
