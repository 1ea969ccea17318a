# TEST INFRASTRUCTURE ONLY.  Builds _ref/libdada2ref_taxonomy.so: the reference's src/taxonomy.cpp (C_assign_taxonomy2),
# compiled UNMODIFIED against oracle/stub_tax/Rcpp.h (oracle/stub/Rcpp.h plus <cfloat> and an injectable Rcpp::runif),
# plus taxonomy_shim.cpp (C-ABI).  Only built when $(REF) exists; the .so is git-ignored and travels with the tree.
REF ?= /root/reference
CXX ?= g++
# -O2 like R's default Makevars; no -ffast-math, no -march (no FMA contraction on x86-64)
CXXFLAGS = -O2 -std=c++11 -fPIC -pthread -w

.PHONY: ref
ref:
	@if [ -d $(REF)/src ]; then $(MAKE) -f taxonomy.mk _ref/libdada2ref_taxonomy.so; else echo "no $(REF): keeping prebuilt _ref/libdada2ref_taxonomy.so"; fi

_ref/libdada2ref_taxonomy.so: taxonomy_shim.cpp stub_tax/Rcpp.h stub/Rcpp.h stub/RcppParallel.h taxonomy.mk
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -Istub_tax -Istub -I$(REF)/src -c $(REF)/src/taxonomy.cpp -o _ref/ref_taxonomy.o
	$(CXX) $(CXXFLAGS) -Istub_tax -Istub -I$(REF)/src -c taxonomy_shim.cpp -o _ref/taxonomy_shim.o
	$(CXX) -shared -pthread -o $@ _ref/ref_taxonomy.o _ref/taxonomy_shim.o -lm
