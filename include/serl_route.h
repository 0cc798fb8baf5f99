/* serl_b200 — which rollout kernel flies a uniform actor.  Part of the C-ABI of include/serl_b200.h (which includes this
 * header); same conventions: 0 or a positive count on success, a negative serl_status on failure.
 */
#ifndef SERL_ROUTE_H
#define SERL_ROUTE_H

#include <stdint.h>

#include "serl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The reference's Actor (base/core/genetic_agent.py:69-101) with num_layers = L is the width list [h] * (L + 1) with the
 * same genome.  Returns 0 when K1 (serl_rollout without widths) flies `shape`, or reports why it cannot: a shape outside
 * the PH-LAB task, num_layers = 0.  Otherwise K1's genome does not fit its kernels and the call writes [h] * (L + 1) to
 * widths_out and returns L + 1: pass them as serl_rollout_desc.widths to fly the actor on K1-TC (2 to 9 widths, h <= 320).
 * K1 keeps h = 32 up to L = 44, 64 up to 9, 72 up to 7, 96 up to 4 and 128 up to 3; at L = 3 it keeps h <= 100 and
 * h = 128, at L = 1 h <= 141.  SERL_ERR_ARG when widths_out holds fewer than cap = L + 1 entries.  Host only, no CUDA
 * call. */
int32_t serl_actor_tc_widths(const serl_actor_shape* shape, int32_t* widths_out, int32_t cap);

#ifdef __cplusplus
}
#endif
#endif
