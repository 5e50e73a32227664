/* vpp_oracle_dt.h — CPU restatement of the chamfer distance transforms (distance_transforms.hh:86-152), part of
 * libvpp_oracle.so.  TEST INFRASTRUCTURE ONLY, like vpp_oracle.h, whose vo_img it uses. */
#ifndef VPP_ORACLE_DT_H_
#define VPP_ORACLE_DT_H_

#include "vpp_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* kind 0 = d4, 1 = d8, 2 = d3-4, 3 = d5-7-11 (VPPB_DT_*).  in: elem 1 (unsigned char) or 4 (int); out: int, same domain, border
 * >= 1 (>= 2 for d5-7-11), all of it written.  Returns 0, -2 (bad argument) or -3 (border too small), writing nothing on error. */
int vo_distance_transform(const vo_img* in, const vo_img* out, int kind);

#ifdef __cplusplus
}
#endif
#endif /* VPP_ORACLE_DT_H_ */
