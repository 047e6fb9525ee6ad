/*
 * apus_fence.h -- the decisions of a read fence (apus_read_fence, DESIGN.md section 2 "Read fences"), shared by the
 * fence kernel (apus_batch.cu: apus_read_fence_kernel) and by the CPU property test (tests/hostlogic/read_fence_props.c),
 * which is why it compiles as plain C as well.  They live in the public include/apus_fence_rule.h, so that a resident
 * reader (include/apus_reader.cuh) takes the very same rule.
 */
#ifndef APUS_FENCE_H
#define APUS_FENCE_H
#include "../../include/apus_fence_rule.h"
#endif
