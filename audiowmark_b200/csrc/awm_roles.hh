// awm_roles.hh -- what a FrameMod entry means: role code (include/awm_b200.h) x coded bit.  The host table builder
// (gen_frame_mod_ab) and the batched embed kernel (k_embed_batch) both form their entries here.
#pragma once
#include "../../include/awm_b200.h"

#ifdef __CUDACC__
#define AWM_HOST_DEVICE __host__ __device__
#else
#define AWM_HOST_DEVICE
#endif

/* FrameMod entry (0 keep, 1 up, 2 down) of a role in block ab (0 = A, 1 = B); coded_ab = that block's coded data bits (0 / nonzero) */
inline AWM_HOST_DEVICE uint8_t
role_frame_mod (uint16_t role, int ab, const uint8_t *coded_ab)
{
  if (!(role & AWM_ROLE_MARK))
    return 0;
  const int index = role >> AWM_ROLE_SHIFT;
  const int bit = (role & AWM_ROLE_SYNC) ? ((index + ab) & 1) : (coded_ab[index] != 0);
  return (bit ^ ((role & AWM_ROLE_DOWN) != 0)) ? 1 : 2;
}
