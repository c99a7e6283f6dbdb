// Parameter update on the flat fp32 buffers (SURVEY.md par.8f rank 1): the step that follows the gradient all-reduce in
// detectron2's run_step.  One launch updates every parameter of the model; per-parameter hyper-parameters (weight decay,
// learning-rate multiplier: yolov7/optimizer/build.py:77-170) come from a sorted segment table, so the kernel is a single
// streaming pass: SGD reads p, g, m and writes p, m (20 B / parameter), AdamW reads p, g, m, v and writes p, m, v (28 B).
//   SGD    torch.optim.SGD as built at optimizer/build.py:234-245 (momentum, optional nesterov, dampening 0 by default)
//   AdamW  torch.optim.AdamW as built at optimizer/build.py:248-256 (decoupled decay, bias correction, no amsgrad)
//   clip   FullModelGradientClippingOptimizer, optimizer/build.py:206-223 = clip_grad_norm_(all params, max_norm)
// grad_scale folds the 1/world_size of the DDP mean into the same pass.
#include "host_common.cuh"
#include "sm90.cuh"
#include <math.h>

using namespace yb;

namespace {

constexpr int kOptThreads = 256;
constexpr int kNormBlocks = 592;  // 4 per SM

__device__ __forceinline__ int find_segment(const int64_t* __restrict__ seg_begin, int nseg, long long i) {
  int lo = 0, hi = nseg - 1;  // largest s with seg_begin[s] <= i
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (seg_begin[mid] <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ float clip_coef(const float* total_norm, float max_norm) {
  if (!total_norm || max_norm <= 0.f) return 1.f;
  const float c = max_norm / (*total_norm + 1e-6f);  // torch.nn.utils.clip_grad_norm_
  return c < 1.f ? c : 1.f;
}

// deterministic sum of squares: fixed grid, fixed in-block order, second stage in one block
__global__ void __launch_bounds__(kOptThreads) sqnorm_partial_kernel(const float* __restrict__ g, int64_t n, float scale, double* __restrict__ partial) {
  pdl_sync();
  __shared__ double s_w[kOptThreads / 32];
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * kOptThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kOptThreads) {
    const float v = g[i] * scale;
    acc += (double)v * v;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kOptThreads / 32; ++w) t += s_w[w];
    partial[blockIdx.x] = t;
  }
}
__global__ void sqnorm_final_kernel(const double* __restrict__ partial, int nparts, float* __restrict__ out_norm) {
  pdl_sync();
  __shared__ double s_w[32];
  double acc = 0.0;
  for (int i = threadIdx.x; i < nparts; i += blockDim.x) acc += partial[i];
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_w[w];
    *out_norm = (float)sqrt(t);
  }
}

struct SegTable {
  const int64_t* begin;
  const float* wd;
  const float* lr_mult;  // may be null
  int nseg;
};

template <bool NESTEROV>
__global__ void __launch_bounds__(kOptThreads) sgd_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, int64_t n, SegTable st,
                                                           float lr, float momentum, float dampening, int first_step, float grad_scale,
                                                           const float* __restrict__ total_norm, float max_norm) {
  pdl_sync();
  const long long i0 = ((long long)blockIdx.x * kOptThreads + threadIdx.x) * 4;
  if (i0 >= n) return;
  const float gs = grad_scale * clip_coef(total_norm, max_norm);
  int s = find_segment(st.begin, st.nseg, i0);
  float pv[4], gv[4], mv[4];
  const bool full = i0 + 4 <= n;
  if (full) {
    const float4 a = *reinterpret_cast<const float4*>(p + i0), b = *reinterpret_cast<const float4*>(g + i0);
    pv[0] = a.x; pv[1] = a.y; pv[2] = a.z; pv[3] = a.w;
    gv[0] = b.x; gv[1] = b.y; gv[2] = b.z; gv[3] = b.w;
    if (momentum != 0.f && !first_step) {
      const float4 c = *reinterpret_cast<const float4*>(m + i0);
      mv[0] = c.x; mv[1] = c.y; mv[2] = c.z; mv[3] = c.w;
    }
  } else {
    for (int j = 0; j < 4; ++j)
      if (i0 + j < n) { pv[j] = p[i0 + j]; gv[j] = g[i0 + j]; mv[j] = (momentum != 0.f && !first_step) ? m[i0 + j] : 0.f; }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long i = i0 + j;
    if (i >= n) break;
    while (s + 1 < st.nseg && st.begin[s + 1] <= i) ++s;
    const float wd = st.wd[s];
    const float lrs = st.lr_mult ? lr * st.lr_mult[s] : lr;
    float d = gv[j] * gs;
    if (wd != 0.f) d = d + wd * pv[j];
    if (momentum != 0.f) {
      const float buf = first_step ? d : momentum * mv[j] + (1.f - dampening) * d;
      mv[j] = buf;
      d = NESTEROV ? d + momentum * buf : buf;
    }
    pv[j] = pv[j] - lrs * d;
  }
  if (full) {
    *reinterpret_cast<float4*>(p + i0) = make_float4(pv[0], pv[1], pv[2], pv[3]);
    if (momentum != 0.f) *reinterpret_cast<float4*>(m + i0) = make_float4(mv[0], mv[1], mv[2], mv[3]);
  } else {
    for (int j = 0; j < 4; ++j)
      if (i0 + j < n) { p[i0 + j] = pv[j]; if (momentum != 0.f) m[i0 + j] = mv[j]; }
  }
}

__global__ void __launch_bounds__(kOptThreads) adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                                             int64_t n, SegTable st, float lr, float beta1, float beta2, float eps, float bc1,
                                                             float bc2_sqrt, float grad_scale, const float* __restrict__ total_norm, float max_norm) {
  pdl_sync();
  const long long i0 = ((long long)blockIdx.x * kOptThreads + threadIdx.x) * 4;
  if (i0 >= n) return;
  const float gs = grad_scale * clip_coef(total_norm, max_norm);
  int s = find_segment(st.begin, st.nseg, i0);
  for (int j = 0; j < 4; ++j) {
    const long long i = i0 + j;
    if (i >= n) break;
    while (s + 1 < st.nseg && st.begin[s + 1] <= i) ++s;
    const float wd = st.wd[s];
    const float lrs = st.lr_mult ? lr * st.lr_mult[s] : lr;
    const float gi = g[i] * gs;
    float pi = p[i];
    pi = pi * (1.f - lrs * wd);
    const float mi = m[i] + (gi - m[i]) * (1.f - beta1);
    const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    pi = pi - (lrs / bc1) * (mi / denom);
    p[i] = pi;
    m[i] = mi;
    v[i] = vi;
  }
}

int check_segments(const int64_t* seg_begin, const float* seg_wd, int nseg, const char* who) {
  YB_REQUIRE(seg_begin && seg_wd && nseg >= 1, YB200_ERR_INVALID, "%s: segment table missing (nseg=%d)", who, nseg);
  return 0;
}

}  // namespace

extern "C" int64_t yb200_grad_norm_workspace(void) { return kNormBlocks * sizeof(double); }

extern "C" int yb200_grad_norm(const float* grad, int64_t n, float grad_scale, void* workspace, float* out_norm, void* stream) {
  YB_REQUIRE(grad && workspace && out_norm && n >= 0, YB200_ERR_INVALID, "grad_norm: null pointer");
  cudaStream_t st = as_stream(stream);
  launch_k(sqnorm_partial_kernel, kNormBlocks, kOptThreads, 0, st, grad, n, grad_scale, static_cast<double*>(workspace));
  launch_k(sqnorm_final_kernel, 1, 256, 0, st, static_cast<const double*>(workspace), kNormBlocks, out_norm);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_sgd_step(float* param, const float* grad, float* momentum_buf, int64_t n, const int64_t* seg_begin, const float* seg_wd,
                              const float* seg_lr_mult, int nseg, float lr, float momentum, float dampening, int nesterov, int first_step,
                              float grad_scale, const float* total_norm, float max_norm, void* stream) {
  YB_REQUIRE(param && grad && n >= 0, YB200_ERR_INVALID, "sgd_step: null pointer");
  YB_REQUIRE(momentum == 0.f || momentum_buf, YB200_ERR_INVALID, "sgd_step: momentum %.3f needs a momentum buffer", momentum);
  // torch.optim.SGD raises ValueError for the same combination
  YB_REQUIRE(!nesterov || (momentum > 0.f && dampening == 0.f), YB200_ERR_INVALID, "sgd_step: nesterov requires momentum > 0 and zero dampening");
  if (int e = check_segments(seg_begin, seg_wd, nseg, "sgd_step")) return e;
  if (n == 0) return 0;
  const SegTable st{seg_begin, seg_wd, seg_lr_mult, nseg};
  const long long threads = (n + 3) / 4;
  const int blocks = static_cast<int>((threads + kOptThreads - 1) / kOptThreads);
  if (nesterov)
    launch_k(sgd_kernel<true>, blocks, kOptThreads, 0, as_stream(stream), param, grad, momentum_buf, n, st, lr, momentum, dampening, first_step, grad_scale, total_norm, max_norm);
  else
    launch_k(sgd_kernel<false>, blocks, kOptThreads, 0, as_stream(stream), param, grad, momentum_buf, n, st, lr, momentum, dampening, first_step, grad_scale, total_norm, max_norm);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_adamw_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, const int64_t* seg_begin,
                                const float* seg_wd, const float* seg_lr_mult, int nseg, float lr, float beta1, float beta2, float eps, int step,
                                float grad_scale, const float* total_norm, float max_norm, void* stream) {
  YB_REQUIRE(param && grad && exp_avg && exp_avg_sq && n >= 0, YB200_ERR_INVALID, "adamw_step: null pointer");
  YB_REQUIRE(step >= 1, YB200_ERR_INVALID, "adamw_step: step counts from 1 (got %d)", step);
  if (int e = check_segments(seg_begin, seg_wd, nseg, "adamw_step")) return e;
  if (n == 0) return 0;
  const SegTable st{seg_begin, seg_wd, seg_lr_mult, nseg};
  const float bc1 = static_cast<float>(1.0 - pow((double)beta1, (double)step));  // torch computes these in Python doubles
  const float bc2_sqrt = static_cast<float>(sqrt(1.0 - pow((double)beta2, (double)step)));
  const long long threads = (n + 3) / 4;
  const int blocks = static_cast<int>((threads + kOptThreads - 1) / kOptThreads);
  launch_k(adamw_kernel, blocks, kOptThreads, 0, as_stream(stream), param, grad, exp_avg, exp_avg_sq, n, st, lr, beta1, beta2, eps, bc1, bc2_sqrt, grad_scale,
                                                               total_norm, max_norm);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
