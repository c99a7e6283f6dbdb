// Batched post-processing: confidence filter + per-class NMS for every image of the batch in one pass.
//
// Restates `postprocess` (yolov7/utils/boxes.py:171-210) + torchvision.ops.batched_nms with the per-class ("vanilla")
// semantics on un-offset fp32 coordinates (SURVEY.md par.0.3): candidates are ordered by (class, score descending, anchor
// index ascending) -- a stable descending sort as torchvision's nms -- then greedily suppressed with
// inter / (area_i + area_j - inter) > thr evaluated in explicitly rounded fp32; survivors are emitted by descending
// score (ties: lower anchor first).  No per-image host loop, no boolean-mask indexing, no host synchronisation.
#include <algorithm>

#include "host_common.cuh"
#include "sm90.cuh"

using namespace yb;

namespace {

constexpr int kNmsThreads = 1024;
constexpr unsigned long long kEmpty = ~0ull;
constexpr int kIdxBits = 16;  // anchors per image < 65536

// ---- stage 1: per anchor class max / score / filter, xyxy conversion, sort keys ----
__global__ void nms_prepare_kernel(float* __restrict__ pred, int num_anchors, int ch, int apad, float conf_thre, int mutate,
                                   float4* __restrict__ boxes, float4* __restrict__ meta, unsigned long long* __restrict__ keys) {
  pdl_sync();
  const int b = blockIdx.y;
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= apad) return;
  unsigned long long key = kEmpty;
  if (a < num_anchors) {
    float* p = pred + (1LL * b * num_anchors + a) * ch;
    const float cx = p[0], cy = p[1], w = p[2], h = p[3];
    float4 bx;
    bx.x = __fsub_rn(cx, __fmul_rn(w, 0.5f));  // prediction[:, :, 0] - prediction[:, :, 2] / 2   (boxes.py:173-176)
    bx.y = __fsub_rn(cy, __fmul_rn(h, 0.5f));
    bx.z = __fadd_rn(cx, __fmul_rn(w, 0.5f));
    bx.w = __fadd_rn(cy, __fmul_rn(h, 0.5f));
    float best = p[5];
    int arg = 0;
    for (int c = 1; c < ch - 5; ++c) {
      const float v = p[5 + c];
      if (v > best) { best = v; arg = c; }  // first maximum, as torch.max(dim)
    }
    const float obj = p[4];
    const float score = __fmul_rn(obj, best);  // image_pred[:, 4] * class_conf   (boxes.py:189)
    if (mutate) { p[0] = bx.x; p[1] = bx.y; p[2] = bx.z; p[3] = bx.w; }
    boxes[1LL * b * num_anchors + a] = bx;
    meta[1LL * b * num_anchors + a] = make_float4(obj, best, static_cast<float>(arg), score);
    if (score >= conf_thre) {
      const unsigned int sb = 0xFFFFFFFFu - __float_as_uint(score);  // scores are >= 0: bit pattern is monotonic
      key = (static_cast<unsigned long long>(arg) << (32 + kIdxBits)) | (static_cast<unsigned long long>(sb) << kIdxBits) |
            static_cast<unsigned long long>(a);
    }
  }
  keys[1LL * b * apad + a] = key;
}

__device__ __forceinline__ void bitonic_sort_smem(unsigned long long* k, int n) {
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < (n >> 1); t += blockDim.x) {
        const int i = ((t & ~(stride - 1)) << 1) | (t & (stride - 1));
        const int l = i | stride;
        const bool asc = (i & size) == 0;
        const unsigned long long x = k[i], y = k[l];
        if ((x > y) == asc) { k[i] = y; k[l] = x; }
      }
      __syncthreads();
    }
  }
}

__device__ __forceinline__ int lower_bound_smem(const unsigned long long* k, int n, unsigned long long v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (k[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// ---- stage 2: one block per image: sort, per-class greedy suppression, order survivors by score, emit ----
__global__ void __launch_bounds__(kNmsThreads)
nms_suppress_kernel(const unsigned long long* __restrict__ keys_in, const float4* __restrict__ boxes, const float4* __restrict__ meta,
                    int num_anchors, int num_classes, int apad, float nms_thre, float* __restrict__ det, int* __restrict__ det_count,
                    int* __restrict__ det_anchor, int* __restrict__ tie_count) {
  pdl_sync();
  extern __shared__ unsigned long long sk[];                          // [apad]
  unsigned char* sup = reinterpret_cast<unsigned char*>(sk + apad);   // [apad]
  __shared__ int s_n, s_keep, s_ties;
  const int b = blockIdx.x;
  const float4* bx = boxes + 1LL * b * num_anchors;
  for (int i = threadIdx.x; i < apad; i += blockDim.x) {
    sk[i] = keys_in[1LL * b * apad + i];
    sup[i] = 0;
  }
  if (threadIdx.x == 0) { s_keep = 0; s_ties = 0; }
  __syncthreads();
  bitonic_sort_smem(sk, apad);
  if (threadIdx.x == 0) s_n = lower_bound_smem(sk, apad, kEmpty);
  __syncthreads();
  const int n = s_n;
  const unsigned long long idx_mask = (1ull << kIdxBits) - 1;

  // per-class greedy NMS: one warp per class segment
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  // (staging a class segment's boxes in shared memory for the greedy chain was measured SLOWER: 3.59 vs 3.09 ms per 64 x 8400 call)
  for (int c = warp; c < num_classes; c += nwarps) {
    const int lo = lower_bound_smem(sk, n, static_cast<unsigned long long>(c) << (32 + kIdxBits));
    const int hi = lower_bound_smem(sk, n, static_cast<unsigned long long>(c + 1) << (32 + kIdxBits));
    for (int i = lo; i < hi; ++i) {
      if (sup[i]) continue;  // warp-uniform
      const float4 bi = bx[sk[i] & idx_mask];
      const float area_i = __fmul_rn(__fsub_rn(bi.z, bi.x), __fsub_rn(bi.w, bi.y));
      for (int j = i + 1 + lane; j < hi; j += 32) {
        if (sup[j]) continue;
        const float4 bj = bx[sk[j] & idx_mask];
        const float xx1 = fmaxf(bi.x, bj.x), yy1 = fmaxf(bi.y, bj.y), xx2 = fminf(bi.z, bj.z), yy2 = fminf(bi.w, bj.w);
        const float w = fmaxf(0.f, __fsub_rn(xx2, xx1)), h = fmaxf(0.f, __fsub_rn(yy2, yy1));
        const float inter = __fmul_rn(w, h);
        const float area_j = __fmul_rn(__fsub_rn(bj.z, bj.x), __fsub_rn(bj.w, bj.y));
        const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_i, area_j), inter));
        if (ovr > nms_thre) sup[j] = 1;
      }
      __syncwarp();
    }
  }
  __syncthreads();
  // survivors: re-key by (score descending, anchor ascending) and COMPACT them to the front, so that the second sort runs over the next power
  // of two above their number (a few hundred to a few thousand) instead of the whole padded array.  All reads of sk complete before the first write.
  unsigned long long mine[16];  // apad <= 16384 = 16 x kNmsThreads
  int kept = 0;
#pragma unroll
  for (int u = 0; u < 16; ++u) {
    const int i = threadIdx.x + u * kNmsThreads;
    if (i < n && !sup[i]) mine[kept++] = sk[i] & ((1ull << (32 + kIdxBits)) - 1);  // drop the class field
  }
  __syncthreads();
  const int pos = atomicAdd(&s_keep, kept);  // the order inside the compacted range is irrelevant: it is sorted next
#pragma unroll
  for (int u = 0; u < 16; ++u)
    if (u < kept) sk[pos + u] = mine[u];
  __syncthreads();
  const int nk = s_keep;
  int npad = 1;
  while (npad < nk) npad <<= 1;
  if (npad > apad) npad = apad;
  for (int i = nk + threadIdx.x; i < npad; i += blockDim.x) sk[i] = kEmpty;
  __syncthreads();
  bitonic_sort_smem(sk, npad);
  if (threadIdx.x == 0) det_count[b] = nk;
  const float4* mt = meta + 1LL * b * num_anchors;
  float* d = det + 1LL * b * num_anchors * 7;
  for (int r = threadIdx.x; r < nk; r += blockDim.x) {
    const int a = static_cast<int>(sk[r] & idx_mask);
    const float4 bb = bx[a];
    const float4 m = mt[a];
    float* o = d + 7LL * r;  // (x1, y1, x2, y2, obj_conf, class_conf, class_pred)   boxes.py:193
    o[0] = bb.x; o[1] = bb.y; o[2] = bb.z; o[3] = bb.w; o[4] = m.x; o[5] = m.y; o[6] = m.z;
    if (det_anchor) det_anchor[1LL * b * num_anchors + r] = a;
    if (tie_count && r + 1 < nk && (sk[r] >> kIdxBits) == (sk[r + 1] >> kIdxBits)) atomicAdd(&s_ties, 1);  // bit-identical scores
  }
  if (tie_count) {
    __syncthreads();
    if (threadIdx.x == 0) tie_count[b] = s_ties;
  }
}

int next_pow2(int v) { int p = 1; while (p < v) p <<= 1; return p; }
int64_t pad256(int64_t v) { return (v + 255) / 256 * 256; }

}  // namespace

extern "C" int64_t yb200_nms_workspace(int batch, int num_anchors) {
  if (batch <= 0 || num_anchors <= 0 || num_anchors >= (1 << kIdxBits)) return YB200_ERR_INVALID;
  const int64_t ba = 1LL * batch * num_anchors;
  return pad256(16 * ba) + pad256(16 * ba) + pad256(8LL * batch * next_pow2(num_anchors)) + 256;
}

extern "C" int yb200_postprocess_nms_indexed(float* prediction, int batch, int num_anchors, int num_classes, float conf_thre, float nms_thre,
                                             int mutate_prediction, void* workspace, float* detections, int32_t* det_count,
                                             int32_t* det_anchor, int32_t* tie_count, void* stream) {
  YB_REQUIRE(prediction && workspace && detections && det_count, YB200_ERR_INVALID, "postprocess_nms: null pointer");
  YB_REQUIRE(batch > 0 && num_anchors > 0 && num_anchors < (1 << kIdxBits) && num_classes > 0 && num_classes < (1 << 14), YB200_ERR_INVALID,
             "postprocess_nms: batch=%d anchors=%d classes=%d", batch, num_anchors, num_classes);
  const int apad = next_pow2(num_anchors);
  const size_t smem = static_cast<size_t>(apad) * 9;
  YB_REQUIRE(smem <= 220 * 1024, YB200_ERR_UNSUPPORTED, "postprocess_nms: %d anchors per image exceed the shared-memory sort (max 16384)", num_anchors);
  const int64_t ba = 1LL * batch * num_anchors;
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  float4* boxes = reinterpret_cast<float4*>(ws);
  float4* meta = reinterpret_cast<float4*>(ws + pad256(16 * ba));
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(ws + 2 * pad256(16 * ba));
  cudaStream_t st = as_stream(stream);
  launch_k(nms_prepare_kernel, dim3(ceil_div(apad, 256), batch), 256, 0, st, prediction, num_anchors, 5 + num_classes, apad, conf_thre, mutate_prediction,
                                                                      boxes, meta, keys);
  YB_CHECK_CUDA(cudaGetLastError());
  static PerDevice<int> smem_limit(0);
  YB_CHECK_CUDA(raise_smem_limit(smem_limit, static_cast<int>(smem), nms_suppress_kernel));
  launch_k(nms_suppress_kernel, batch, kNmsThreads, smem, st, keys, boxes, meta, num_anchors, num_classes, apad, nms_thre, detections, det_count,
                                                        det_anchor, tie_count);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_postprocess_nms(float* prediction, int batch, int num_anchors, int num_classes, float conf_thre, float nms_thre,
                                     int mutate_prediction, void* workspace, float* detections, int32_t* det_count, void* stream) {
  return yb200_postprocess_nms_indexed(prediction, batch, num_anchors, num_classes, conf_thre, nms_thre, mutate_prediction, workspace, detections,
                                       det_count, nullptr, nullptr, stream);
}
