// TEST INFRASTRUCTURE ONLY (parity oracle) -- never linked into the product.
//
// C-ABI wrapper around the reference's src/filter.cpp, compiled UNMODIFIED (see oracle/filter.mk):
//   ref_match_ref()  C_matchRef, the k-mer screen behind isPhiX;
//   ref_matrix_ee()  C_matrixEE, the expected errors of a quality matrix.
// Built as its own library (_ref/libdada2ref_filter.so) so that libdada2ref.so stays as it is.
#include <Rcpp.h>
#include <algorithm>
#include <string>
#include <vector>

Rcpp::IntegerVector C_matchRef(std::vector<std::string> seqs, std::string ref, unsigned int word_size, bool non_overlapping);
Rcpp::NumericVector C_matrixEE(Rcpp::IntegerMatrix inp);

extern "C" {

// seqs: n sequences concatenated with int64 offsets (n + 1); hits: int32[n].
int ref_match_ref(int n, const char *seq_concat, const long long *seq_off, const char *ref, int word_size, int non_overlapping, int *hits) {
  std::vector<std::string> seqs;
  for (int i = 0; i < n; i++) seqs.emplace_back(seq_concat + seq_off[i], (size_t)(seq_off[i + 1] - seq_off[i]));
  Rcpp::IntegerVector r = C_matchRef(seqs, std::string(ref), (unsigned)word_size, non_overlapping != 0);
  for (int i = 0; i < n; i++) hits[i] = r[i];
  return 0;
}

// quals: n reads concatenated with offsets as above, laid out as R's as(quality, "matrix"): NA beyond a read's end.
int ref_matrix_ee(int n, const unsigned char *qual_concat, const long long *seq_off, double *ee) {
  int ncol = 0;
  for (int i = 0; i < n; i++) ncol = std::max(ncol, (int)(seq_off[i + 1] - seq_off[i]));
  Rcpp::IntegerMatrix m(n, ncol);
  for (int i = 0; i < n; i++)
    for (int j = 0; j < ncol; j++) m(i, j) = j < seq_off[i + 1] - seq_off[i] ? (int)qual_concat[seq_off[i] + j] : NA_INTEGER;
  Rcpp::NumericVector r = C_matrixEE(m);
  for (int i = 0; i < n; i++) ee[i] = r[i];
  return 0;
}

}  // extern "C"
