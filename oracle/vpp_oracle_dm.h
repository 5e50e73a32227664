/* vpp_oracle_dm.h — CPU restatement of the SAD descriptor matchers (descriptor_matcher/bruteforce_matcher.hh:11-47,
 * local_index1d_sad_descriptor_matcher.hh, grid_index.hh:11-88), part of libvpp_oracle.so.  TEST INFRASTRUCTURE ONLY, like
 * vpp_oracle.h, whose vo_img it uses.  Patch extraction is restated in numpy (tests/dm_cases.py). */
#ifndef VPP_ORACLE_DM_H_
#define VPP_ORACLE_DM_H_

#include "vpp_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Descriptors are the rows of q and t (elem 1 = unsigned char or 4 = int, one length); distance sum |q[k] - t[k]| in int.
 * Brute force: for every query the train of smallest distance, ties to the lowest train index; (-1, INT32_MAX) without trains.
 * Grid-local: over the trains whose cell (p.r / s, p.c / s), C division, lies in the query's window ((q - R) / s .. (q + R) / s),
 * the smallest distance, ties to the smallest (cell row, cell col, train index); (-1, INT32_MAX) when the window holds no train.
 * A train at a coordinate <= -s is never matched.  Positions are (row, col) int pairs.  Return 0, or -2 for a bad argument (s < 1,
 * R < 0, mismatched descriptors), writing nothing. */
int vo_match_bruteforce_sad(const vo_img* q, const vo_img* t, int32_t* idx, int32_t* dist);
int vo_match_local_sad(const vo_img* q, const vo_img* t, const int32_t* qpos, const int32_t* tpos, int32_t R, int32_t s, int32_t* idx,
                       int32_t* dist);

#ifdef __cplusplus
}
#endif
#endif /* VPP_ORACLE_DM_H_ */
