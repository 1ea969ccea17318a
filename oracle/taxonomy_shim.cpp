// TEST INFRASTRUCTURE ONLY (parity oracle) -- never linked into the product.
//
// C-ABI wrapper around the reference's src/taxonomy.cpp, compiled UNMODIFIED (see oracle/taxonomy.mk):
//   ref_assign_taxonomy()  C_assign_taxonomy2 with the uniforms of Rcpp::runif injected by the caller.
// The reference's tie draw (std::random_device) stays random: callers compare only where the arg-max is strict.
#include <Rcpp.h>
#include <algorithm>
#include <atomic>
#include <string>
#include <vector>

Rcpp::List C_assign_taxonomy2(std::vector<std::string> seqs, std::vector<std::string> rcs, std::vector<std::string> refs,
                              std::vector<int> ref_to_genus, Rcpp::IntegerMatrix genusmat, bool try_rc, bool verbose);

static const double *g_unifs = nullptr;
static long long g_nunifs = 0;
static std::atomic<int> g_threads(1);

extern "C" int oracle_get_threads(void) { return g_threads.load(); }

namespace Rcpp {
NumericVector runif(size_t n) {
  if ((long long)n != g_nunifs) stop("oracle: runif(%zu) but %lld uniforms were injected", n, g_nunifs);
  NumericVector v(n);
  for (size_t i = 0; i < n; i++) v[i] = g_unifs[i];
  return v;
}
}  // namespace Rcpp

static std::vector<std::string> unpack(int n, const char *cat, const long long *off) {
  std::vector<std::string> v;
  for (int i = 0; i < n; i++) v.emplace_back(cat + off[i], (size_t)(off[i + 1] - off[i]));
  return v;
}

extern "C" {

// Sequences: n strings concatenated with int64 offsets (n + 1).  genusmat: [ngenus][nlevel] row-major.  tax: int32[nseq],
// boot: int32[nseq][nlevel], boot_tax: int32[nseq][100].  Returns 0, or 1 with the reference's message in err.
int ref_assign_taxonomy(int nseq, const char *seq_cat, const long long *seq_off, const char *rc_cat, const long long *rc_off, int nref,
                        const char *ref_cat, const long long *ref_off, const int *ref_to_genus, int ngenus, int nlevel, const int *genusmat,
                        int try_rc, const double *unifs, long long nunifs, int nthreads, int *tax, int *boot, int *boot_tax, char *err,
                        int errlen) {
  try {
    g_unifs = unifs; g_nunifs = nunifs;
    g_threads.store(std::max(1, nthreads));
    Rcpp::IntegerMatrix gm(ngenus, nlevel);
    for (int i = 0; i < ngenus; i++)
      for (int j = 0; j < nlevel; j++) gm(i, j) = genusmat[(size_t)i * nlevel + j];
    Rcpp::List r = C_assign_taxonomy2(unpack(nseq, seq_cat, seq_off), unpack(nseq, rc_cat, rc_off), unpack(nref, ref_cat, ref_off),
                                      std::vector<int>(ref_to_genus, ref_to_genus + nref), gm, try_rc != 0, false);
    const Rcpp::Any *t = r.get("tax"), *b = r.get("boot"), *bt = r.get("boot_tax");
    for (int i = 0; i < nseq; i++) tax[i] = (*t->iv)[i];
    for (int i = 0; i < nseq; i++)
      for (int j = 0; j < nlevel; j++) boot[(size_t)i * nlevel + j] = (*b->iv)[i + (size_t)nseq * j];
    for (int i = 0; i < nseq; i++)
      for (int j = 0; j < 100; j++) boot_tax[(size_t)i * 100 + j] = (*bt->iv)[i + (size_t)nseq * j];
    return 0;
  } catch (std::exception &e) {
    snprintf(err, errlen, "%s", e.what());
    return 1;
  }
}

}  // extern "C"
