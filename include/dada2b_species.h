/* dada2b_species.h -- C-ABI of the H100-native species assignment by exact matching (libdada2b.so).
 *
 * assignSpecies (R/taxonomy.R:240-289) looks for every query as an exact, contiguous substring of every reference of a
 * species fasta (Biostrings' vcountPDict, fixed=TRUE) and maps the hit references to genus and species labels.  Here the
 * references are 2-bit packed with a mask of their non-A/C/G/T positions and stay resident on the device
 * (dada2b_species_db); every call scans all of them once for all queries and reduces the hits to distinct labels on the
 * device.  The Rcpp shim is in INTEGRATION.md 2k; the contract is DESIGN.md 22.
 *
 * Contract (DESIGN.md 22):
 *   hit    query q hits reference r when q occurs in r as an exact substring; with try_rc also when revcomp(q) does.
 *          A reference position holding anything but A/C/G/T matches no query letter.  A reference counts once per query.
 *   labels ref_to_genus / ref_to_species are label ids chosen by the caller; 0 is NA and counts as a distinct label
 *   keep   a query's distinct-label list is returned when its length is at most keep (keep <= 0: always); otherwise
 *          only its length is
 *   queries must be non-empty and A/C/G/T only (refused with a message otherwise); any length, including longer than
 *          every reference, gives the exact answer
 * Results do not depend on the launch geometry, the hit buffer's size or the anchor choice.
 *
 * Environment (test hooks): DADA2B_SPECIES_HITCAP=<n> sets the initial hit-record capacity (the call grows the buffer and
 * scans again when it overflows); DADA2B_SPECIES_ANCHOR0=1 anchors every pattern at offset 0 instead of the least
 * shared of its candidate offsets.
 *
 * Returns 0 on success, non-zero with a message in errbuf; nothing throws across the ABI.  There is no CPU path.
 */
#ifndef DADA2B_SPECIES_H
#define DADA2B_SPECIES_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef DADA2B_ERRLEN
#define DADA2B_ERRLEN 256
#endif

#define DADA2B_SPECIES_ANCHOR 32       /* anchor length of queries of at least 32 nt (shorter queries anchor whole)    */

typedef struct {                       /* n strings concatenated, n + 1 offsets                                         */
  int32_t n, reserved;
  const char *seq_concat;
  const int64_t *seq_off;
} dada2b_species_seqs;

typedef struct dada2b_species_db dada2b_species_db;    /* opaque: the packed references and their labels on a device */

typedef struct {
  int32_t nref, reserved;
  int64_t nbases;                      /* reference bases                                                               */
  int64_t device_bytes;                /* resident bytes: packed bases, mask, reference starts and labels              */
  /* work counters and timings of the build (information only) */
  int64_t gpu_launches, h2d_bytes, d2h_bytes, kernel_bytes;
  double ms_h2d, ms_kernels, ms_d2h, ms_device, ms_total;
} dada2b_species_db_info;

typedef struct {
  int32_t nseq, reserved;
  int32_t *nhits;                      /* [nseq] distinct hit references                                                */
  int32_t *genus_n;                    /* [nseq] distinct genus ids among the hits (NA = 0 included)                   */
  int64_t *genus_off;                  /* [nseq + 1] CSR into genus_ids: empty for a query whose genus_n exceeds keep   */
  int32_t *genus_ids;                  /* ascending per query                                                           */
  int32_t *species_n, *species_ids;    /* the same for species                                                          */
  int64_t *species_off;
  int64_t *hit_off;                    /* test hook only (NULL otherwise): [nseq + 1] CSR into hit_refs                 */
  int32_t *hit_refs;                   /* test hook only: sorted 0-based distinct hit references                        */
  int64_t npatterns;                   /* queries, plus their reverse complements with try_rc                          */
  int64_t hit_records;                 /* occurrences recorded by the scan (before deduplication)                      */
  int64_t hit_capacity;                /* the hit buffer's final capacity                                               */
  int64_t distinct_hits;               /* distinct (query, reference) pairs                                             */
  int32_t scans, max_group;            /* scans of the references (> 1 after a hit-buffer overflow); most patterns
                                          sharing one anchor                                                            */
  int64_t gpu_launches, h2d_bytes, d2h_bytes, kernel_bytes;
  double ms_h2d, ms_scan, ms_reduce, ms_d2h, ms_device, ms_total;   /* ms_scan: the scan and verify kernel (events) */
} dada2b_species_out;

/* refs: the references (upper-case; any byte other than A/C/G/T matches nothing).  ref_to_genus / ref_to_species:
 * [nref] label ids >= 0 (0: NA).  The caller has already applied any relabelling (Escherichia/Shigella). */
int dada2b_species_db_build(const dada2b_species_seqs *refs, const int32_t *ref_to_genus, const int32_t *ref_to_species, int32_t device,
                            dada2b_species_db **db, char errbuf[DADA2B_ERRLEN]);
int dada2b_species_db_info_get(const dada2b_species_db *db, dada2b_species_db_info *info);
void dada2b_species_db_free(dada2b_species_db *db);

/* keep_genus / keep_species: see keep above (assignSpecies: 1 for the genus; 1, <= 0 for Inf, or an integer). */
int dada2b_species_assign(dada2b_species_db *db, const dada2b_species_seqs *seqs, int32_t try_rc, int32_t keep_genus, int32_t keep_species,
                          dada2b_species_out **out, char errbuf[DADA2B_ERRLEN]);
void dada2b_species_free(dada2b_species_out *out);

/* Test hook: dada2b_species_assign with keep <= 0 that also returns every query's distinct hit references (hit_off,
 * hit_refs), forward and reverse-complement hits combined. */
int dada2b_test_species_hits(dada2b_species_db *db, const dada2b_species_seqs *seqs, int32_t try_rc, dada2b_species_out **out,
                             char errbuf[DADA2B_ERRLEN]);

#ifdef __cplusplus
}
#endif
#endif
