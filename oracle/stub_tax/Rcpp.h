// TEST INFRASTRUCTURE ONLY -- oracle/stub/Rcpp.h plus the two things src/taxonomy.cpp needs beyond it:
// FLT_MAX (<cfloat>) and Rcpp::runif, which returns the uniforms oracle/taxonomy_shim.cpp injects.
// Searched before oracle/stub by oracle/taxonomy.mk only, so the other reference builds see the stub unchanged.
#ifndef ORACLE_STUB_TAX_RCPP_H
#define ORACLE_STUB_TAX_RCPP_H
#include "../stub/Rcpp.h"
#include <cfloat>

namespace Rcpp {
NumericVector runif(size_t n);       // defined in taxonomy_shim.cpp
}
#endif
