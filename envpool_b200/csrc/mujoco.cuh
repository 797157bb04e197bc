// HalfCheetah (mujoco/gym) family: host-side queries of the two-lane physics kernel.
#pragma once
#include <cuda_runtime.h>

#include "common.cuh"

namespace epb {

int64_t mjc_model_blob(void* dst, int64_t cap);  // sizeof(hcm::HcModel); fills dst if it fits
// constraint rows per lane the two-lane kernel keeps in shared memory for a launch of n rows
int mjc_pair_rows(int n);

}  // namespace epb
