// The compaction step shared by the meta-architectures' inference (sparseinst_infer.cu, detr_infer.cu): the kept rows of a [B][N] batch in
// compact order (image, then ascending query).  Bit 0 of keep[r] marks a kept row; bit 1 is a per-row error flag that is OR-ed into *status.
#pragma once

#include "sm90.cuh"

#include <stdint.h>

using yb::pdl_sync;

namespace {

// counts [B], exclusive offsets [B + 1], and per kept row its query index within the image, its score, its label as int64 and, when `box` is
// not null, its 4 box values.  status (may be null) = OR over all rows of keep >> 1.  One CTA; thread b owns image b.
__global__ void __launch_bounds__(256) infer_compact_kernel(const uint8_t* __restrict__ keep, const float* __restrict__ score,
                                                            const int32_t* __restrict__ label, const float* __restrict__ box, int B, int N,
                                                            int32_t* __restrict__ counts, int32_t* __restrict__ offsets, int32_t* __restrict__ kept_query,
                                                            float* __restrict__ kept_score, int64_t* __restrict__ kept_label, float* __restrict__ kept_box,
                                                            int32_t* __restrict__ status) {
  pdl_sync();
  __shared__ int s_flags;
  if (threadIdx.x == 0) s_flags = 0;
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    int c = 0, f = 0;
    for (int q = 0; q < N; ++q) {
      const int k = keep[static_cast<long long>(b) * N + q];
      c += k & 1;
      f |= k >> 1;
    }
    counts[b] = c;
    if (f) atomicOr(&s_flags, f);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int b = 0; b < B; ++b) offsets[b] = run, run += counts[b];
    offsets[B] = run;
    if (status) *status = s_flags;
  }
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    int j = offsets[b];
    for (int q = 0; q < N; ++q) {
      const long long r = static_cast<long long>(b) * N + q;
      if (!(keep[r] & 1)) continue;
      kept_query[j] = q;
      kept_score[j] = score[r];
      kept_label[j] = label[r];
      if (box)
        for (int i = 0; i < 4; ++i) kept_box[4LL * j + i] = box[4 * r + i];
      ++j;
    }
  }
}

}  // namespace
