// Sizes fixed by the kernels that the host plan (plan.h) also needs.  Plain C++, so that plan.h compiles without CUDA.
#pragma once

namespace b200 {

constexpr int SEL_WARPS = 8;      // rows (one warp each) per block of the list re-score / merge kernels
constexpr int WIDE_MAX = 512;     // candidates per row rescore_wide_kernel holds (kp <= 128)
constexpr int WIDE_MAX_L = 4096;  // candidates per row rescore_wide_large_kernel holds (128 < kp <= 1024)
constexpr int LIST_SLOTS = 32;    // slots of each of the fused kernel's two candidate lists per subject row (K' <= 32)
// survivors large_k_select_kernel sorts in shared memory (2 buffers x 8 B each: 192 KiB, next to 34 KiB of static shared
// memory within the 227 KiB a CTA may have); rows with more sort through 16 B per entry of global scratch
constexpr int LK_SMEM_PAIRS = 12288;

}  // namespace b200
