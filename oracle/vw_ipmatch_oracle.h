/* vw_ipmatch_oracle.h -- CPU restatement of InterestPointMatcherSimple with L2NormMetric / HammingMetric and remove_duplicates
 * (InterestPoint/Matcher.h:415-509, Matcher.cc:33-195), loop for loop; the checker of K11.  Built with -ffp-contract=off. */
#ifndef VW_IPMATCH_ORACLE_H
#define VW_IPMATCH_ORACLE_H
#include <stddef.h>
#include <stdint.h>

/* L2NormMetric::operator()(ip1, ip2) with the default maxdist FLT_MAX: the loop breaks once dist > FLT_MAX */
float vwm_l2(const float* a, const float* b, int dim);
/* HammingMetric::operator()(ip1, ip2): bytes static_cast<uint8>(value), popcounts of 8-, 4- and 1-byte chunks summed in float.
 * Every value must lie in (-1, 256) (vwm_match checks). */
float vwm_hamming(const float* a, const float* b, int dim);
/* InterestPointMatcherSimple<Metric, NullConstraint>(threshold)::operator() over n1 x dim / n2 x dim descriptors (dense rows)
 * and polarity bytes (compared as bools): index[i] = the match of ip1[i] or -1; first / second (may be NULL) the double
 * first_pick / second_pick.  metric 0 L2, 1 Hamming.  Returns 0; -1 for a Hamming value outside (-1, 256) or NaN (*bad_list
 * 0 / 1 and *bad_elem = row * dim + k of the first such element, desc1 before desc2); -4 for a Hamming 8 dim > 2^24. */
int vwm_match(int metric, const float* d1, const uint8_t* p1, int n1, const float* d2, const uint8_t* p2, int n2, int dim, double threshold,
              int32_t* index, double* first, double* second, int* bad_list, long long* bad_elem);
/* remove_duplicates on n matched pairs' (x, y): keep[0 .. *n_kept) the kept indices in ascending order.  -1 on a NaN. */
int vwm_remove_duplicates(const float* xy1, const float* xy2, int n, int32_t* keep, int* n_kept);

#endif
