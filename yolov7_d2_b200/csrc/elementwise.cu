// HBM-bound kernels around the convolutions: image preprocessing (Focus layout), BatchNorm finalize / apply+SiLU /
// backward, SPP max-pooling, nearest upsampling.  All activations are NHWC bf16 views (see include/yb200.h); every
// thread moves 8 channels (16 bytes) per access so warps read and write whole 128-byte lines.
#include <algorithm>

#include <cuda_fp16.h>

#include "host_common.cuh"
#include "sm90.cuh"

using namespace yb;

namespace {

struct View {  // device-side copy of yb200_act with element strides resolved
  __nv_bfloat16* p;  // already offset by c_off
  int n, h, w, c, pitch;
};

View mk(const yb200_act* a) {
  View v;
  v.p = static_cast<__nv_bfloat16*>(a->ptr) + a->c_off;
  v.n = a->n; v.h = a->h; v.w = a->w; v.c = a->c; v.pitch = a->c_pitch;
  return v;
}

// streaming 16-byte load (read once: do not allocate in L1)
// YB200_L2_ORDER=1: element-wise passes walk their tensors in the direction that meets the producer's most recent (L2-resident) output first
static int l2_order() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("YB200_L2_ORDER");
    v = (e && e[0] == '1') ? 1 : 0;
  }
  return v;
}

__device__ __forceinline__ uint4 ldg_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ float2 h2f(uint32_t u) {
  __half2 h;
  *reinterpret_cast<uint32_t*>(&h) = u;
  return __half22float2(h);
}
__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
// the pre-BatchNorm tensor z is stored in fp16 (see conv_gemm.cuh); the view type only carries the 2-byte element size
__device__ __forceinline__ void unpack8_f16(const uint4& u, float* f) {
  const float2 a = h2f(u.x), b = h2f(u.y), c = h2f(u.z), d = h2f(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}
// sigmoid(u) = 0.5 tanh(u / 2) + 0.5 on MUFU.TANH: FMUL + MUFU + FFMA instead of FMUL + MUFU.EX2 + FADD + MUFU.RCP (+ FMUL).  These passes are
// bound by instruction issue (ncu: 60-72 % issue-slot utilisation at 4.3-5.4 TB/s), so every instruction per element counts; the absolute
// error of tanh.approx (2^-11) is below the bf16 resolution of everything these kernels store.
__device__ __forceinline__ float sigmoid_fast(float u) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * u));
  return fmaf(t, 0.5f, 0.5f);
}
__device__ __forceinline__ float silu_f(float u) { return u * sigmoid_fast(u); }

int grid_for(long long work, int threads) {
  long long b = (work + threads - 1) / threads;
  long long cap = 32LL * sm_count();
  return static_cast<int>(std::max<long long>(1, std::min(b, cap)));
}

// ------------------------------------------------------------------------------------------------
// preprocess: uint8 NCHW image batch -> Focus (space-to-depth) NHWC bf16 with 16 channels
//   channel = patch*3 + rgb, patch order (top-left, bottom-left, top-right, bottom-right)   wrappers.py:210-220
//   channels 12..15 are zero (pads K to the MMA granule); pixels beyond (h_valid[n], w_valid[n]) read as pad_value
//   (detectron2 ImageList.from_tensors with MODEL.PADDED_VALUE = 114, yolox.py:100-101).
// ------------------------------------------------------------------------------------------------
__global__ void preprocess_focus_kernel(const uint8_t* __restrict__ img, int n, int h, int w, const int* __restrict__ hw_valid,
                                        float pad_value, __nv_bfloat16* __restrict__ out, int pitch) {
  pdl_sync();
  const int oh = h / 2, ow = w / 2;
  const long long total = 1LL * n * oh * ow;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = static_cast<int>(i % ow);
    const int y = static_cast<int>((i / ow) % oh);
    const int b = static_cast<int>(i / (1LL * ow * oh));
    const int hv = hw_valid ? hw_valid[2 * b] : h;
    const int wv = hw_valid ? hw_valid[2 * b + 1] : w;
    float f[16];
#pragma unroll
    for (int patch = 0; patch < 4; ++patch) {
      const int yy = 2 * y + (patch & 1);   // patches 1 and 3 are the odd rows
      const int xx = 2 * x + (patch >> 1);  // patches 2 and 3 are the odd columns
      const bool in = yy < hv && xx < wv;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        f[patch * 3 + c] = in ? static_cast<float>(img[((1LL * b * 3 + c) * h + yy) * w + xx]) : pad_value;
    }
    f[12] = f[13] = f[14] = f[15] = 0.f;
    uint4* o = reinterpret_cast<uint4*>(out + i * pitch);
    o[0] = pack8(f);
    o[1] = pack8(f + 8);
  }
}

// ------------------------------------------------------------------------------------------------
// BatchNorm (training): finalize statistics
// ------------------------------------------------------------------------------------------------
__global__ void bn_finalize_kernel(double* __restrict__ ssum, double* __restrict__ ssq, int c, double count, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float eps, float momentum, float* __restrict__ running_mean,
                                   float* __restrict__ running_var, long long* __restrict__ num_batches, float* __restrict__ scale,
                                   float* __restrict__ shift, float* __restrict__ mean_out, float* __restrict__ invstd_out) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0 && num_batches) *num_batches += 1;
  if (i >= c) return;
  const double mean = ssum[i] / count;
  double var = ssq[i] / count - mean * mean;  // biased variance, used for normalisation (ATen batch_norm)
  if (var < 0) var = 0;
  const float invstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  const float g = gamma[i];
  scale[i] = g * invstd;
  shift[i] = beta[i] - static_cast<float>(mean) * g * invstd;
  mean_out[i] = static_cast<float>(mean);
  invstd_out[i] = invstd;
  if (running_mean) {
    const double unbiased = count > 1 ? var * count / (count - 1) : var;
    running_mean[i] = (1.f - momentum) * running_mean[i] + momentum * static_cast<float>(mean);
    running_var[i] = (1.f - momentum) * running_var[i] + momentum * static_cast<float>(unbiased);
  }
  ssum[i] = 0.0;  // ready for the next step
  ssq[i] = 0.0;
}

// eval mode: scale/shift from the running statistics (the fold of utils/checkpoint.py:11-43 applied as an epilogue)
__global__ void bn_eval_affine_kernel(int c, const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ rm,
                                      const float* __restrict__ rv, float eps, float* __restrict__ scale, float* __restrict__ shift) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c) return;
  const float s = gamma[i] / sqrtf(rv[i] + eps);
  scale[i] = s;
  shift[i] = beta[i] - rm[i] * s;
}

// Thread mapping of the BatchNorm kernels: blockDim = (channel vectors of 8, pixels), so a thread's channels are fixed
// (per-channel constants live in registers) and no integer division is needed to decode an element index; consecutive
// linear thread ids touch consecutive 16-byte chunks, i.e. warps read and write whole 128-byte lines.
constexpr int kEwThreads = 256;
constexpr int kEwIters = 8;  // pixels per thread (2 was measured slower in the real step: the per-channel constants are re-loaded per thread)

struct PixXY {
  int x, y, b;
};
__device__ __forceinline__ PixXY decode_pix(unsigned pix, int w, int h) {
  PixXY r;
  const unsigned row = pix / static_cast<unsigned>(w);
  r.x = static_cast<int>(pix - row * w);
  r.b = static_cast<int>(row / static_cast<unsigned>(h));
  r.y = static_cast<int>(row - static_cast<unsigned>(r.b) * h);
  return r;
}

// a = SiLU(z*scale + shift) [+ residual];  optionally also written 2x nearest-upsampled into a second view
// Training-mode finalize folded into the apply pass (fin.ssum != nullptr): every block derives scale / shift of its channels from the batch
// sums (a dozen fp64 operations per channel), block 0 additionally publishes scale / shift / mean / invstd for the backward pass and updates the
// running statistics -- one launch per BatchNorm instead of two.  The sums are NOT cleared here (the plan clears all accumulators once per step).
struct BnFinalize {
  const double* ssum;
  const double* ssq;
  double inv_count;  // 1 / count
  float unbias;      // count / (count - 1): running_var takes the unbiased variance
  const float* gamma;
  const float* beta;
  float eps, momentum;
  float* running_mean;
  float* running_var;
  float* scale_out;
  float* shift_out;
  float* mean_out;
  float* invstd_out;
};

__global__ void __launch_bounds__(kEwThreads)
bn_apply_silu_kernel(View z, View a, View res, View up, const float* __restrict__ scale, const float* __restrict__ shift, int has_res,
                     int has_up, unsigned npix, int rev, BnFinalize fin) {
  pdl_sync();
  const int c8 = threadIdx.x * 8;
  float s[8], t[8];
  if (fin.ssum != nullptr) {
    // one thread row derives the per-channel constants (fp64 only where the cancellation var = E[x^2] - mean^2 needs it; no fp64 division or
    // square root: the fp64 pipe is narrow) and hands them to the other rows through shared memory
    __shared__ float s_st[2][kEwThreads * 8];
    if (threadIdx.y == 0) {
      const bool publish = blockIdx.x == 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int c = c8 + k;
        const double mean = fin.ssum[c] * fin.inv_count;
        double var = fma(-mean, mean, fin.ssq[c] * fin.inv_count);  // biased variance, used for normalisation (ATen batch_norm)
        if (var < 0) var = 0;
        const float ve = static_cast<float>(var) + fin.eps;
        float invstd = rsqrtf(ve);
        invstd = invstd * (1.5f - 0.5f * ve * invstd * invstd);      // one Newton step: full fp32 accuracy
        const float g = fin.gamma[c];
        const float sc = g * invstd, sh = fin.beta[c] - static_cast<float>(mean) * g * invstd;
        s_st[0][c] = sc;
        s_st[1][c] = sh;
        if (publish) {
          fin.scale_out[c] = sc; fin.shift_out[c] = sh; fin.mean_out[c] = static_cast<float>(mean); fin.invstd_out[c] = invstd;
          if (fin.running_mean) {
            const float unbiased = static_cast<float>(var) * fin.unbias;
            fin.running_mean[c] = (1.f - fin.momentum) * fin.running_mean[c] + fin.momentum * static_cast<float>(mean);
            fin.running_var[c] = (1.f - fin.momentum) * fin.running_var[c] + fin.momentum * unbiased;
          }
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 8; ++k) { s[k] = s_st[0][c8 + k]; t[k] = s_st[1][c8 + k]; }
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) { s[k] = scale[c8 + k]; t[k] = shift[c8 + k]; }
  }
  // rev: walk the tensor from its end -- the convolution that produced z wrote its tail last, so the tail is what the L2 still holds
  const unsigned p0 = (rev ? gridDim.x - 1 - blockIdx.x : blockIdx.x) * (blockDim.y * kEwIters) + threadIdx.y;
  constexpr int U = 4;  // loads of U pixels are issued before any of them is consumed
#pragma unroll 1
  for (int it0 = 0; it0 < kEwIters; it0 += U) {
    uint4 zq[U], rq[U];
    unsigned pixs[U];
    bool oks[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned pix_raw = p0 + (it0 + u) * blockDim.y;
      oks[u] = pix_raw < npix;
      pixs[u] = oks[u] ? pix_raw : npix - 1;  // clamped: loads stay unconditional
      zq[u] = ldg_stream(z.p + static_cast<size_t>(pixs[u]) * z.pitch + c8);
      if (has_res) rq[u] = ldg_stream(res.p + static_cast<size_t>(pixs[u]) * res.pitch + c8);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned pix = pixs[u];
      float f[8];
      unpack8_f16(zq[u], f);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] = silu_f(fmaf(f[k], s[k], t[k]));
      if (has_res) {
        // residual is added to the *rounded* activation, as in the reference where y = conv2(...) is materialised first
        float r[8];
        unpack8(rq[u], r);
#pragma unroll
        for (int k = 0; k < 8; ++k) f[k] = bf16_round(f[k]) + r[k];
      }
      const uint4 o = pack8(f);
      if (!oks[u]) continue;
      *reinterpret_cast<uint4*>(a.p + static_cast<size_t>(pix) * a.pitch + c8) = o;
      if (has_up) {
        const PixXY q = decode_pix(pix, z.w, z.h);
        __nv_bfloat16* up_p = up.p + ((static_cast<size_t>(q.b) * up.h + 2 * q.y) * up.w + 2 * q.x) * up.pitch + c8;
        *reinterpret_cast<uint4*>(up_p) = o;
        *reinterpret_cast<uint4*>(up_p + up.pitch) = o;
        *reinterpret_cast<uint4*>(up_p + static_cast<size_t>(up.w) * up.pitch) = o;
        *reinterpret_cast<uint4*>(up_p + static_cast<size_t>(up.w + 1) * up.pitch) = o;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// BatchNorm + SiLU backward
//   u = z*scale + shift, a = silu(u);   du = da * sig(u) * (1 + u*(1-sig(u)))
//   pass 1: dbeta = sum du, dgamma = sum du * zhat        (zhat = (z-mean)*invstd)
//   pass 2: dz = gamma*invstd * (du - dbeta/M - zhat*dgamma/M)
// `da` may be the sum of up to two views (fan-out of the activation) and, for upsampled consumers, a third view that
// is 2x larger and gets 2x2 sum-pooled (backward of nn.Upsample(nearest), yolo_pafpn.py:28).
// ------------------------------------------------------------------------------------------------
struct DaSrc {
  View a, b, up;
  int has_b, has_up;
};

__device__ __forceinline__ void load_da(const DaSrc& s, unsigned pix, int w, int h, int c8, float* d) {
  unpack8(ldg_stream(s.a.p + static_cast<size_t>(pix) * s.a.pitch + c8), d);
  if (s.has_b) {
    float e[8];
    unpack8(*reinterpret_cast<const uint4*>(s.b.p + static_cast<size_t>(pix) * s.b.pitch + c8), e);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] += e[k];
  }
  if (s.has_up) {
    const PixXY q = decode_pix(pix, w, h);
    const __nv_bfloat16* u = s.up.p + ((static_cast<size_t>(q.b) * s.up.h + 2 * q.y) * s.up.w + 2 * q.x) * s.up.pitch + c8;
    float e[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const size_t off = static_cast<size_t>((j >> 1) * s.up.w + (j & 1)) * s.up.pitch;
      unpack8(*reinterpret_cast<const uint4*>(u + off), e);
#pragma unroll
      for (int k = 0; k < 8; ++k) d[k] += e[k];
    }
  }
}

constexpr int kBnRedIters = 32;  // pixels per thread in the reduction pass

__device__ __forceinline__ float silu_grad(float u, float d) {  // d * d/du [u * sigmoid(u)] = d * sg * (1 + u - u * sg)
  const float sg = sigmoid_fast(u);
  return (d * sg) * fmaf(u, 1.f - sg, 1.f);
}

// pass 1: per channel  S1 = sum du,  S2 = sum du * z   (dgamma = invstd * (S2 - mean * S1), dbeta = S1)
// Block reduction in a fixed order (warp shuffles, then one shared-memory row per warp summed sequentially): two runs on
// the same data produce the same fp32 block partials; only the final fp64 atomics are unordered.
template <int U, int MINB, bool SIMPLE>
__global__ void __launch_bounds__(kEwThreads, MINB)
bn_silu_bwd_reduce_kernel(View z, DaSrc da, const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ mean,
                          const float* __restrict__ invstd, double* __restrict__ dgamma_acc, double* __restrict__ dbeta_acc, unsigned npix,
                          int iters, int rev) {
  pdl_sync();
  extern __shared__ float sm[];  // [rows][2][c], rows = warps (c < 256) or blockDim.y (c >= 256)
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  const int nthreads = blockDim.x * blockDim.y;
  const int c8 = threadIdx.x * 8;
  float s[8], t[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { s[k] = scale[c8 + k]; t[k] = shift[c8 + k]; }
  float s1[8] = {0, 0, 0, 0, 0, 0, 0, 0}, s2[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // rev: start at the tail (written last by the data-gradient kernel, still in L2) and finish at the head, which the apply pass reads first
  const unsigned p0 = (rev ? gridDim.x - 1 - blockIdx.x : blockIdx.x) * (blockDim.y * iters) + threadIdx.y;
  constexpr bool simple = SIMPLE;  // one gradient source (the common case): leaner code, more resident blocks
#pragma unroll 1
  for (int it0 = 0; it0 < iters; it0 += U) {
    uint4 zq[U], dq[U];
    unsigned pixs[U];
    bool oks[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned pix_raw = p0 + (it0 + u) * blockDim.y;
      oks[u] = (it0 + u < iters) && pix_raw < npix;
      pixs[u] = oks[u] ? pix_raw : npix - 1;
      zq[u] = ldg_stream(z.p + static_cast<size_t>(pixs[u]) * z.pitch + c8);
      if (simple) {
        dq[u] = ldg_stream(da.a.p + static_cast<size_t>(pixs[u]) * da.a.pitch + c8);
        if (!oks[u]) dq[u] = make_uint4(0u, 0u, 0u, 0u);  // out-of-range pixel: zero gradient, no per-element select below
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float zf[8], d[8];
      unpack8_f16(zq[u], zf);
      if (simple) {
        unpack8(dq[u], d);
      } else {
        load_da(da, pixs[u], z.w, z.h, c8, d);
        if (!oks[u]) {
#pragma unroll
          for (int k = 0; k < 8; ++k) d[k] = 0.f;
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float du = silu_grad(fmaf(zf[k], s[k], t[k]), d[k]);
        s1[k] += du;
        s2[k] = fmaf(du, zf[k], s2[k]);
      }
    }
  }
  // blockDim.x a power of two below 32: lanes sharing a channel vector (same threadIdx.x) sit blockDim.x apart inside the warp and are folded
  // by shuffles first; otherwise (wide or non-power-of-two channel counts, e.g. 96 / 192 / 384 / 768 of the width-0.75 plans) every thread
  // row goes to shared memory
  const int cvx = blockDim.x;
  const bool shuf = cvx < 32 && (cvx & (cvx - 1)) == 0;
  if (shuf) {
    for (int off = 16; off >= cvx; off >>= 1) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        s1[k] += __shfl_xor_sync(0xffffffffu, s1[k], off);
        s2[k] += __shfl_xor_sync(0xffffffffu, s2[k], off);
      }
    }
  }
  const int rows = shuf ? nthreads / 32 : blockDim.y;
  const int row = shuf ? tid / 32 : threadIdx.y;
  if (!shuf || (tid & 31) < cvx) {
    float* dst = sm + static_cast<size_t>(row) * 2 * z.c;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      dst[c8 + k] = s2[k];
      dst[z.c + c8 + k] = s1[k];
    }
  }
  __syncthreads();
  for (int i = tid; i < z.c; i += nthreads) {
    float S1 = 0.f, S2 = 0.f;
    for (int r = 0; r < rows; ++r) {
      S2 += sm[static_cast<size_t>(r) * 2 * z.c + i];
      S1 += sm[static_cast<size_t>(r) * 2 * z.c + z.c + i];
    }
    atomicAdd(dgamma_acc + i, static_cast<double>(invstd[i]) * (static_cast<double>(S2) - static_cast<double>(mean[i]) * S1));
    atomicAdd(dbeta_acc + i, static_cast<double>(S1));
  }
}

// pass 2: dz = gamma*invstd * (du - dbeta/M - zhat*dgamma/M) = s*du + A*z + B  with per-channel A, B
template <bool SIMPLE>
__global__ void __launch_bounds__(kEwThreads, 3)
bn_silu_bwd_apply_kernel(View z, DaSrc da, View dz, const float* __restrict__ scale, const float* __restrict__ shift,
                         const float* __restrict__ mean, const float* __restrict__ invstd, const double* __restrict__ dgamma_acc,
                         const double* __restrict__ dbeta_acc, double inv_count, unsigned npix) {
  pdl_sync();
  const int c8 = threadIdx.x * 8;
  float s[8], t[8], A[8], B[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    s[k] = scale[c8 + k]; t[k] = shift[c8 + k];
    const float is = invstd[c8 + k], mu = mean[c8 + k];
    const float mg = static_cast<float>(dgamma_acc[c8 + k] * inv_count);
    const float mb = static_cast<float>(dbeta_acc[c8 + k] * inv_count);
    A[k] = -s[k] * is * mg;
    B[k] = -s[k] * mb - A[k] * mu;
  }
  const unsigned p0 = blockIdx.x * (blockDim.y * kEwIters) + threadIdx.y;
  constexpr bool simple = SIMPLE;
  constexpr int U = 2;
#pragma unroll 1
  for (int it0 = 0; it0 < kEwIters; it0 += U) {
    uint4 zq[U], dq[U];
    unsigned pixs[U];
    bool oks[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned pix_raw = p0 + (it0 + u) * blockDim.y;
      oks[u] = pix_raw < npix;
      pixs[u] = oks[u] ? pix_raw : npix - 1;
      zq[u] = ldg_stream(z.p + static_cast<size_t>(pixs[u]) * z.pitch + c8);
      if (simple) dq[u] = ldg_stream(da.a.p + static_cast<size_t>(pixs[u]) * da.a.pitch + c8);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float zf[8], d[8], o[8];
      unpack8_f16(zq[u], zf);
      if (simple) unpack8(dq[u], d); else load_da(da, pixs[u], z.w, z.h, c8, d);
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] = fmaf(s[k], silu_grad(fmaf(zf[k], s[k], t[k]), d[k]), fmaf(A[k], zf[k], B[k]));
      if (oks[u]) *reinterpret_cast<uint4*>(dz.p + static_cast<size_t>(pixs[u]) * dz.pitch + c8) = pack8(o);
    }
  }
}

// parameter gradients out of the fp64 accumulators, then re-zero them
__global__ void bn_param_grad_kernel(double* __restrict__ dgamma_acc, double* __restrict__ dbeta_acc, int c, float* __restrict__ dgamma,
                                     float* __restrict__ dbeta, int accumulate) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c) return;
  const float g = static_cast<float>(dgamma_acc[i]), b = static_cast<float>(dbeta_acc[i]);
  dgamma[i] = accumulate ? dgamma[i] + g : g;
  dbeta[i] = accumulate ? dbeta[i] + b : b;
  dgamma_acc[i] = 0.0;
  dbeta_acc[i] = 0.0;
}

// ------------------------------------------------------------------------------------------------
// SPP: max-pool k = 5, 9, 13 (stride 1, pad k/2, -inf padding) of x into three channel slices; argmax offsets kept
// for the backward (first maximum in row-major window order, as ATen max_pool2d_with_indices).
// ------------------------------------------------------------------------------------------------
__global__ void spp_pool_kernel(View x, View o5, View o9, View o13, uint8_t* __restrict__ arg) {
  pdl_sync();
  const int cv = x.c / 8;
  const long long total = 1LL * x.n * x.h * x.w * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = static_cast<int>(i % cv) * 8;
    const long long pix = i / cv;
    const int px = static_cast<int>(pix % x.w);
    const int py = static_cast<int>((pix / x.w) % x.h);
    const long long b = pix / (1LL * x.w * x.h);
    float m[3][8];
    int am[3][8];
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int k = 0; k < 8; ++k) { m[j][k] = -INFINITY; am[j][k] = 0; }
    for (int dy = -6; dy <= 6; ++dy) {
      const int yy = py + dy;
      if (yy < 0 || yy >= x.h) continue;
      for (int dx = -6; dx <= 6; ++dx) {
        const int xx = px + dx;
        if (xx < 0 || xx >= x.w) continue;
        float v[8];
        unpack8(*reinterpret_cast<const uint4*>(x.p + ((b * x.h + yy) * x.w + xx) * x.pitch + c8), v);
        const int ady = dy < 0 ? -dy : dy, adx = dx < 0 ? -dx : dx;
        const int r = ady > adx ? ady : adx;  // Chebyshev radius: window k covers r <= k/2
        const int code = (dy + 6) * 13 + (dx + 6);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          if (v[k] > m[2][k]) { m[2][k] = v[k]; am[2][k] = code; }
          if (r <= 4 && v[k] > m[1][k]) { m[1][k] = v[k]; am[1][k] = code; }
          if (r <= 2 && v[k] > m[0][k]) { m[0][k] = v[k]; am[0][k] = code; }
        }
      }
    }
    *reinterpret_cast<uint4*>(o5.p + pix * o5.pitch + c8) = pack8(m[0]);
    *reinterpret_cast<uint4*>(o9.p + pix * o9.pitch + c8) = pack8(m[1]);
    *reinterpret_cast<uint4*>(o13.p + pix * o13.pitch + c8) = pack8(m[2]);
    if (arg) {
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        uint8_t* a = arg + ((1LL * j * x.n * x.h * x.w + pix) * x.c + c8);
        uint2 pk;
        pk.x = am[j][0] | (am[j][1] << 8) | (am[j][2] << 16) | (am[j][3] << 24);
        pk.y = am[j][4] | (am[j][5] << 8) | (am[j][6] << 16) | (am[j][7] << 24);
        *reinterpret_cast<uint2*>(a) = pk;
      }
    }
  }
}

// Shared-memory version for maps that fit in one SM (the usual case: 20x20 at 640 px): one block per (CG channels, image).
// Every element becomes a 32-bit KEY = (order-preserving code of the bf16 value) << 16 | (0xFFFF - pixel index): the unsigned maximum of keys is
// the maximum value and, among equal values, the SMALLEST pixel index = the first maximum of the window in row-major order (ATen's rule), whatever
// the order in which the candidates are combined.  Max-pooling of keys is therefore separable (row pass, column pass: 5 + 5 reads) and cascades:
// pool9 = pool5(pool5), pool13 = pool5(pool9), exactly, borders included (windows clipped to the map = -inf padding).  30 shared-memory reads and
// 30 integer maxima per element for the three sizes instead of 54 compare / select chains.
__device__ __forceinline__ uint32_t spp_key(unsigned short bits, int pix) {
  if (bits == 0x8000u) bits = 0;  // -0 == +0
  const uint32_t ord = (bits & 0x8000u) ? (~static_cast<uint32_t>(bits) & 0xFFFFu) : (static_cast<uint32_t>(bits) | 0x8000u);
  return (ord << 16) | static_cast<uint32_t>(0xFFFF - pix);
}
__device__ __forceinline__ unsigned short spp_key_bits(uint32_t key) {
  const uint32_t ord = key >> 16;
  return static_cast<unsigned short>((ord & 0x8000u) ? (ord & 0x7FFFu) : (~ord & 0xFFFFu));
}

template <int CG>
__global__ void __launch_bounds__(256)
spp_pool_tiled_kernel(View x, View o5, View o9, View o13, uint8_t* __restrict__ arg) {
  pdl_sync();
  extern __shared__ uint32_t sp[];  // two [hw][CG] key planes
  const int hw = x.h * x.w;
  uint32_t* ka = sp;
  uint32_t* kb = sp + hw * CG;
  const int cg = blockIdx.x * CG;
  const int b = blockIdx.y;
  const int total = hw * CG;
  const __nv_bfloat16* src = x.p + static_cast<size_t>(b) * hw * x.pitch + cg;
  for (int e = threadIdx.x; e < total; e += blockDim.x) {
    const int ch = e % CG, p = e / CG;
    ka[e] = spp_key(__bfloat16_as_ushort(src[static_cast<size_t>(p) * x.pitch + ch]), p);
  }
  __syncthreads();
#pragma unroll 1
  for (int j = 0; j < 3; ++j) {
    // ka holds the keys pooled with window 4j + 1 (j = 0: the input): one more 5x5 pass -> window 4j + 5
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
      const int p = e / CG;
      const int px = p % x.w;
      const int lo = max(px - 2, 0) - px, hi = min(px + 2, x.w - 1) - px;
      uint32_t m = 0;
      for (int d = lo; d <= hi; ++d) m = max(m, ka[e + d * CG]);
      kb[e] = m;
    }
    __syncthreads();
    const View& o = j == 0 ? o5 : (j == 1 ? o9 : o13);
    __nv_bfloat16* dst = o.p + static_cast<size_t>(b) * hw * o.pitch + cg;
    uint8_t* adst = arg ? arg + (static_cast<size_t>(j) * x.n + b) * hw * x.c + cg : nullptr;
    const int rowstride = x.w * CG;
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
      const int ch = e % CG, p = e / CG;
      const int py = p / x.w, px = p - py * x.w;
      const int lo = max(py - 2, 0) - py, hi = min(py + 2, x.h - 1) - py;
      uint32_t m = 0;
      for (int d = lo; d <= hi; ++d) m = max(m, kb[e + d * rowstride]);
      ka[e] = m;  // each thread rewrites only its own elements of ka; the row pass of the next round starts after the barrier below
      dst[static_cast<size_t>(p) * o.pitch + ch] = __ushort_as_bfloat16(spp_key_bits(m));
      if (adst) {
        const int q = 0xFFFF - static_cast<int>(m & 0xFFFFu);  // pixel index of the first maximum
        const int qy = q / x.w, qx = q - qy * x.w;
        adst[static_cast<size_t>(p) * x.c + ch] = static_cast<uint8_t>((qy - py + 6) * 13 + (qx - px + 6));
      }
    }
    __syncthreads();
  }
}

// backward for the same maps: one block per (CG channels, image) routes the three pooled gradients to their argmax positions in a SHARED
// [hw][CG] fp32 plane that starts as the identity-branch gradient -- no scratch plane in HBM, no atomics.  One thread owns each (row, channel) of
// the plane and adds the gradients that land there in a fixed order (branch 5, 9, 13, then source pixel): the sums, and so the bf16 results, are
// the same in every run (shared-memory atomics added them in an order that depended on warp scheduling).
template <int CG>
__global__ void __launch_bounds__(256)
spp_pool_bwd_tiled_kernel(View d0, View d5, View d9, View d13, const uint8_t* __restrict__ arg, View dx) {
  pdl_sync();
  extern __shared__ float sacc[];  // [hw][CG] fp32 gradient plane, then the [hw][CG] bf16 gradients and argmax codes of one branch
  const int hw = dx.h * dx.w;
  const int cg = blockIdx.x * CG;
  const int b = blockIdx.y;
  const int total = hw * CG;
  __nv_bfloat16* const sgrad = reinterpret_cast<__nv_bfloat16*>(sacc + total);
  uint8_t* const scode = reinterpret_cast<uint8_t*>(sgrad + total);
  for (int e = threadIdx.x; e < total; e += blockDim.x) {
    const int ch = e % CG, p = e / CG;
    sacc[e] = __bfloat162float(d0.p[(static_cast<size_t>(b) * hw + p) * d0.pitch + cg + ch]);
  }
#pragma unroll 1
  for (int j = 0; j < 3; ++j) {
    const View& d = j == 0 ? d5 : (j == 1 ? d9 : d13);
    const uint8_t* a = arg + (static_cast<size_t>(j) * dx.n + b) * hw * dx.c + cg;
    __syncthreads();  // the previous branch is done with sgrad / scode
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
      const int ch = e % CG, p = e / CG;
      sgrad[e] = d.p[(static_cast<size_t>(b) * hw + p) * d.pitch + cg + ch];
      scode[e] = a[static_cast<size_t>(p) * dx.c + ch];
    }
    __syncthreads();
    // thread (y, ch) scans the source rows whose windows reach row y (pool 5 / 9 / 13: the argmax lies within 2 / 4 / 6 rows) and adds the
    // gradients whose argmax lies in row y
    const int r = 2 + 2 * j;
    for (int t = threadIdx.x; t < dx.h * CG; t += blockDim.x) {
      const int ch = t % CG, y = t / CG;
      const int y0 = max(y - r, 0), y1 = min(y + r, dx.h - 1);
      for (int py = y0; py <= y1; ++py) {
        for (int px = 0; px < dx.w; ++px) {
          const int p = py * dx.w + px;
          const int code = scode[p * CG + ch];
          const int dy = code / 13 - 6;
          if (py + dy != y) continue;
          sacc[(p + dy * dx.w + (code % 13 - 6)) * CG + ch] += __bfloat162float(sgrad[p * CG + ch]);
        }
      }
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < total; e += blockDim.x) {
    const int ch = e % CG, p = e / CG;
    dx.p[(static_cast<size_t>(b) * hw + p) * dx.pitch + cg + ch] = __float2bfloat16_rn(sacc[e]);
  }
}

// backward: scatter the three pooled gradients to their argmax positions (fp32 atomics into a zeroed scratch), ...
__global__ void spp_pool_bwd_scatter_kernel(View d5, View d9, View d13, const uint8_t* __restrict__ arg, float* __restrict__ scratch, int n,
                                            int h, int w, int c) {
  pdl_sync();
  const long long total = 3LL * n * h * w * c;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ch = static_cast<int>(i % c);
    const long long pix = (i / c) % (1LL * n * h * w);
    const int j = static_cast<int>(i / (1LL * c * n * h * w));
    const View& d = j == 0 ? d5 : (j == 1 ? d9 : d13);
    const float g = __bfloat162float(d.p[pix * d.pitch + ch]);
    const int code = arg[i];
    const int dy = code / 13 - 6, dx = code % 13 - 6;
    const int px = static_cast<int>(pix % w), py = static_cast<int>((pix / w) % h);
    const long long b = pix / (1LL * w * h);
    atomicAdd(scratch + ((b * h + py + dy) * w + px + dx) * c + ch, g);
  }
}
// ... then dx = identity-branch gradient + scattered sums
__global__ void spp_pool_bwd_finish_kernel(View d0, const float* __restrict__ scratch, View dx) {
  pdl_sync();
  const int cv = dx.c / 8;
  const long long total = 1LL * dx.n * dx.h * dx.w * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = static_cast<int>(i % cv) * 8;
    const long long pix = i / cv;
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(d0.p + pix * d0.pitch + c8), f);
    const float* s = scratch + pix * dx.c + c8;
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] += s[k];
    *reinterpret_cast<uint4*>(dx.p + pix * dx.pitch + c8) = pack8(f);
  }
}

// plain copy between views (used to place an activation into a concat slice when it cannot be produced there)
__global__ void copy_view_kernel(View s, View d) {
  pdl_sync();
  const int cv = s.c / 8;
  const long long total = 1LL * s.n * s.h * s.w * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = static_cast<int>(i % cv) * 8;
    const long long pix = i / cv;
    *reinterpret_cast<uint4*>(d.p + pix * d.pitch + c8) = *reinterpret_cast<const uint4*>(s.p + pix * s.pitch + c8);
  }
}

}  // namespace

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" int yb200_preprocess_focus(const uint8_t* images_nchw, int n, int h, int w, const int32_t* hw_valid, float pad_value,
                                      const yb200_act* out, void* stream) {
  YB_REQUIRE(images_nchw && out && out->ptr, YB200_ERR_INVALID, "preprocess_focus: null pointer");
  YB_REQUIRE(n > 0 && h > 0 && w > 0 && h % 2 == 0 && w % 2 == 0, YB200_ERR_INVALID, "preprocess_focus: image %dx%dx%d", n, h, w);
  YB_REQUIRE(out->n == n && out->h == h / 2 && out->w == w / 2 && out->c == 16 && out->c_pitch >= 16 && out->c_pitch % 8 == 0 && out->c_off == 0,
             YB200_ERR_INVALID, "preprocess_focus: output must be the first 16 channels of a [n,h/2,w/2,pitch] buffer");
  const long long total = 1LL * n * (h / 2) * (w / 2);
  launch_k(preprocess_focus_kernel, grid_for(total, 256), 256, 0, as_stream(stream), images_nchw, n, h, w, hw_valid, pad_value,
                                                                              static_cast<__nv_bfloat16*>(out->ptr), out->c_pitch);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_bn_finalize(double* stat_sum, double* stat_sqsum, int c, int64_t count, const float* gamma, const float* beta, float eps,
                                 float momentum, float* running_mean, float* running_var, int64_t* num_batches_tracked, float* scale,
                                 float* shift, float* save_mean, float* save_invstd, void* stream) {
  YB_REQUIRE(stat_sum && stat_sqsum && gamma && beta && scale && shift && save_mean && save_invstd, YB200_ERR_INVALID, "bn_finalize: null pointer");
  YB_REQUIRE(c > 0 && count > 0, YB200_ERR_INVALID, "bn_finalize: c=%d count=%lld", c, (long long)count);
  YB_REQUIRE((running_mean == nullptr) == (running_var == nullptr), YB200_ERR_INVALID, "bn_finalize: running stats must come in pairs");
  launch_k(bn_finalize_kernel, ceil_div(c, 128), 128, 0, as_stream(stream), stat_sum, stat_sqsum, c, static_cast<double>(count), gamma, beta, eps,
                                                                      momentum, running_mean, running_var,
                                                                      reinterpret_cast<long long*>(num_batches_tracked), scale, shift,
                                                                      save_mean, save_invstd);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_bn_eval_affine(int c, const float* gamma, const float* beta, const float* running_mean, const float* running_var, float eps,
                                    float* scale, float* shift, void* stream) {
  YB_REQUIRE(gamma && beta && running_mean && running_var && scale && shift && c > 0, YB200_ERR_INVALID, "bn_eval_affine: bad arguments");
  launch_k(bn_eval_affine_kernel, ceil_div(c, 128), 128, 0, as_stream(stream), c, gamma, beta, running_mean, running_var, eps, scale, shift);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int bn_apply_impl(const yb200_act* z, const float* scale, const float* shift, const yb200_act* residual, const yb200_act* out,
                         const yb200_act* out_up2x, const BnFinalize& fin, void* stream) {
  int rc;
  if ((rc = check_act(z, "bn_apply_silu z")) || (rc = check_act(out, "bn_apply_silu out"))) return rc;
  if (residual && (rc = check_act(residual, "bn_apply_silu residual"))) return rc;
  if (out_up2x && (rc = check_act(out_up2x, "bn_apply_silu out_up2x"))) return rc;
  YB_REQUIRE((scale && shift) || fin.ssum, YB200_ERR_INVALID, "bn_apply_silu: null scale/shift");
  YB_REQUIRE(same_shape(z, out) && (!residual || same_shape(z, residual)), YB200_ERR_INVALID, "bn_apply_silu: shape mismatch");
  YB_REQUIRE(!out_up2x || (out_up2x->n == z->n && out_up2x->h == 2 * z->h && out_up2x->w == 2 * z->w && out_up2x->c == z->c), YB200_ERR_INVALID,
             "bn_apply_silu: upsampled view must be [n,2h,2w,c]");
  View vz = mk(z), vo = mk(out), vr = residual ? mk(residual) : vz, vu = out_up2x ? mk(out_up2x) : vz;
  const long long npix = 1LL * z->n * z->h * z->w;
  const int cv = z->c / 8;
  YB_REQUIRE(cv <= kEwThreads && npix < (1LL << 31), YB200_ERR_UNSUPPORTED, "bn_apply_silu: %d channels / %lld pixels", z->c, npix);
  dim3 block(cv, kEwThreads / cv);
  const unsigned grid = static_cast<unsigned>((npix + block.y * kEwIters - 1) / (block.y * kEwIters));
  launch_k(bn_apply_silu_kernel, grid, block, 0, as_stream(stream), vz, vo, vr, vu, scale, shift, residual != nullptr, out_up2x != nullptr,
                                                             static_cast<unsigned>(npix), l2_order(), fin);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_bn_apply_silu(const yb200_act* z, const float* scale, const float* shift, const yb200_act* residual, const yb200_act* out,
                                   const yb200_act* out_up2x, void* stream) {
  BnFinalize fin;
  memset(&fin, 0, sizeof(fin));
  return bn_apply_impl(z, scale, shift, residual, out, out_up2x, fin, stream);
}

extern "C" int yb200_bn_train_apply_silu(const yb200_act* z, const double* stat_sum, const double* stat_sqsum, int64_t count, const float* gamma,
                                         const float* beta, float eps, float momentum, float* running_mean, float* running_var, float* scale,
                                         float* shift, float* save_mean, float* save_invstd, const yb200_act* residual, const yb200_act* out,
                                         const yb200_act* out_up2x, void* stream) {
  YB_REQUIRE(stat_sum && stat_sqsum && gamma && beta && scale && shift && save_mean && save_invstd && count > 0, YB200_ERR_INVALID,
             "bn_train_apply_silu: null pointer / empty batch");
  YB_REQUIRE((running_mean == nullptr) == (running_var == nullptr), YB200_ERR_INVALID, "bn_train_apply_silu: running stats must come in pairs");
  BnFinalize fin;
  fin.ssum = stat_sum; fin.ssq = stat_sqsum; fin.inv_count = 1.0 / static_cast<double>(count);
  fin.unbias = count > 1 ? static_cast<float>(static_cast<double>(count) / static_cast<double>(count - 1)) : 1.f; fin.gamma = gamma; fin.beta = beta; fin.eps = eps;
  fin.momentum = momentum; fin.running_mean = running_mean; fin.running_var = running_var; fin.scale_out = scale; fin.shift_out = shift;
  fin.mean_out = save_mean; fin.invstd_out = save_invstd;
  return bn_apply_impl(z, nullptr, nullptr, residual, out, out_up2x, fin, stream);
}

extern "C" int yb200_bn_silu_bwd(const yb200_act* z, const yb200_act* da, const yb200_act* da2, const yb200_act* da_up2x, const float* scale,
                                 const float* shift, const float* save_mean, const float* save_invstd, double* acc_dgamma, double* acc_dbeta,
                                 const yb200_act* dz, float* dgamma, float* dbeta, int accumulate, void* stream) {
  int rc;
  if ((rc = check_act(z, "bn_silu_bwd z")) || (rc = check_act(da, "bn_silu_bwd da")) || (rc = check_act(dz, "bn_silu_bwd dz"))) return rc;
  if (da2 && (rc = check_act(da2, "bn_silu_bwd da2"))) return rc;
  if (da_up2x && (rc = check_act(da_up2x, "bn_silu_bwd da_up2x"))) return rc;
  YB_REQUIRE(scale && shift && save_mean && save_invstd && acc_dgamma && acc_dbeta && (dgamma != nullptr) == (dbeta != nullptr), YB200_ERR_INVALID,
             "bn_silu_bwd: null pointer");
  YB_REQUIRE(same_shape(z, da) && same_shape(z, dz) && (!da2 || same_shape(z, da2)), YB200_ERR_INVALID, "bn_silu_bwd: shape mismatch");
  YB_REQUIRE(!da_up2x || (da_up2x->n == z->n && da_up2x->h == 2 * z->h && da_up2x->w == 2 * z->w && da_up2x->c == z->c), YB200_ERR_INVALID,
             "bn_silu_bwd: upsampled gradient view must be [n,2h,2w,c]");
  const long long npix = 1LL * z->n * z->h * z->w;
  const int cv = z->c / 8;
  YB_REQUIRE(cv <= kEwThreads && npix < (1LL << 31), YB200_ERR_UNSUPPORTED, "bn_silu_bwd: %d channels (at most 2048) / %lld pixels", z->c, npix);
  cudaStream_t st = as_stream(stream);
  DaSrc src;
  src.a = mk(da);
  src.b = da2 ? mk(da2) : src.a;
  src.up = da_up2x ? mk(da_up2x) : src.a;
  src.has_b = da2 != nullptr;
  src.has_up = da_up2x != nullptr;
  View vz = mk(z), vdz = mk(dz);
  dim3 block(cv, kEwThreads / cv);
  // pixels per thread in the reduction pass: up to 32, fewer for small tensors so that >= ~6 blocks per SM exist
  int red_iters = static_cast<int>(npix / (static_cast<long long>(block.y) * 6 * sm_count()));
  red_iters = red_iters < 4 ? 4 : (red_iters > kBnRedIters ? kBnRedIters : red_iters);
  const bool red_shuffle = cv < 32 && (cv & (cv - 1)) == 0;
  const int red_rows = red_shuffle ? static_cast<int>(block.x * block.y) / 32 : static_cast<int>(block.y);
  const size_t red_smem = static_cast<size_t>(red_rows) * 2 * z->c * sizeof(float);
  const unsigned grid_r = static_cast<unsigned>((npix + block.y * red_iters - 1) / (block.y * red_iters));
  static PerDevice<int> red_limit(48 * 1024);
  YB_CHECK_CUDA(raise_smem_limit(red_limit, static_cast<int>(red_smem), bn_silu_bwd_reduce_kernel<2, 3, false>, bn_silu_bwd_reduce_kernel<2, 3, true>));
  if (src.has_b || src.has_up)  // fan-out / upsampled gradient sources: the general kernel
    launch_k(bn_silu_bwd_reduce_kernel<2, 3, false>, grid_r, block, red_smem, st, vz, src, scale, shift, save_mean, save_invstd, acc_dgamma, acc_dbeta,
                                                                             static_cast<unsigned>(npix), red_iters, l2_order());
  else
    launch_k(bn_silu_bwd_reduce_kernel<2, 3, true>, grid_r, block, red_smem, st, vz, src, scale, shift, save_mean, save_invstd, acc_dgamma, acc_dbeta,
                                                                            static_cast<unsigned>(npix), red_iters, l2_order());
  YB_CHECK_CUDA(cudaGetLastError());
  const unsigned grid_a = static_cast<unsigned>((npix + block.y * kEwIters - 1) / (block.y * kEwIters));
  if (!src.has_b && !src.has_up)
    launch_k(bn_silu_bwd_apply_kernel<true>, grid_a, block, 0, st, vz, src, vdz, scale, shift, save_mean, save_invstd, acc_dgamma, acc_dbeta,
                                                              1.0 / static_cast<double>(npix), static_cast<unsigned>(npix));
  else
    launch_k(bn_silu_bwd_apply_kernel<false>, grid_a, block, 0, st, vz, src, vdz, scale, shift, save_mean, save_invstd, acc_dgamma, acc_dbeta,
                                                               1.0 / static_cast<double>(npix), static_cast<unsigned>(npix));
  YB_CHECK_CUDA(cudaGetLastError());
  if (dgamma == nullptr) return 0;  // deferred: yb200_bn_param_grads turns the accumulators of many layers into parameter gradients in one launch
  launch_k(bn_param_grad_kernel, ceil_div(z->c, 128), 128, 0, st, acc_dgamma, acc_dbeta, z->c, dgamma, dbeta, accumulate);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// the same for a run of layers: channel i of the run writes grad_base[gamma_off[i]] / grad_base[beta_off[i]]
__global__ void bn_param_grads_table_kernel(double* __restrict__ dgamma_acc, double* __restrict__ dbeta_acc, int c, const int* __restrict__ gamma_off,
                                            const int* __restrict__ beta_off, float* __restrict__ grad_base, int accumulate) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c) return;
  const float g = static_cast<float>(dgamma_acc[i]), b = static_cast<float>(dbeta_acc[i]);
  float* pg = grad_base + gamma_off[i];
  float* pb = grad_base + beta_off[i];
  *pg = accumulate ? *pg + g : g;
  *pb = accumulate ? *pb + b : b;
  dgamma_acc[i] = 0.0;
  dbeta_acc[i] = 0.0;
}

extern "C" int yb200_bn_param_grads(double* acc_dgamma, double* acc_dbeta, int c, const int32_t* gamma_off, const int32_t* beta_off, float* grad_base,
                                    int accumulate, void* stream) {
  YB_REQUIRE(acc_dgamma && acc_dbeta && gamma_off && beta_off && grad_base && c > 0, YB200_ERR_INVALID, "bn_param_grads: bad arguments");
  launch_k(bn_param_grads_table_kernel, ceil_div(c, 128), 128, 0, as_stream(stream), acc_dgamma, acc_dbeta, c, gamma_off, beta_off, grad_base, accumulate);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_spp_pool(const yb200_act* x, const yb200_act* o5, const yb200_act* o9, const yb200_act* o13, uint8_t* argmax, void* stream) {
  int rc;
  if ((rc = check_act(x, "spp_pool x")) || (rc = check_act(o5, "spp_pool o5")) || (rc = check_act(o9, "spp_pool o9")) ||
      (rc = check_act(o13, "spp_pool o13")))
    return rc;
  YB_REQUIRE(same_shape(x, o5) && same_shape(x, o9) && same_shape(x, o13), YB200_ERR_INVALID, "spp_pool: shape mismatch");
  constexpr int kCg = 16;
  const size_t tiled_smem = static_cast<size_t>(x->h) * x->w * kCg * 2 * sizeof(uint32_t);
  if (x->c % kCg == 0 && tiled_smem <= 200 * 1024) {
    static PerDevice<int> smem_limit(48 * 1024);
    YB_CHECK_CUDA(raise_smem_limit(smem_limit, static_cast<int>(tiled_smem), spp_pool_tiled_kernel<kCg>));
    launch_k(spp_pool_tiled_kernel<kCg>, dim3(x->c / kCg, x->n), 256, tiled_smem, as_stream(stream), mk(x), mk(o5), mk(o9), mk(o13), argmax);
    YB_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  const long long total = 1LL * x->n * x->h * x->w * (x->c / 8);
  launch_k(spp_pool_kernel, grid_for(total, 128), 128, 0, as_stream(stream), mk(x), mk(o5), mk(o9), mk(o13), argmax);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_spp_pool_bwd(const yb200_act* d0, const yb200_act* d5, const yb200_act* d9, const yb200_act* d13, const uint8_t* argmax,
                                  float* scratch, const yb200_act* dx, void* stream) {
  int rc;
  if ((rc = check_act(d0, "spp_pool_bwd d0")) || (rc = check_act(d5, "spp_pool_bwd d5")) || (rc = check_act(d9, "spp_pool_bwd d9")) ||
      (rc = check_act(d13, "spp_pool_bwd d13")) || (rc = check_act(dx, "spp_pool_bwd dx")))
    return rc;
  YB_REQUIRE(argmax && scratch, YB200_ERR_INVALID, "spp_pool_bwd: null pointer");
  YB_REQUIRE(same_shape(dx, d0) && same_shape(dx, d5) && same_shape(dx, d9) && same_shape(dx, d13), YB200_ERR_INVALID, "spp_pool_bwd: shape mismatch");
  cudaStream_t st = as_stream(stream);
  const long long elems = 1LL * dx->n * dx->h * dx->w * dx->c;
  constexpr int kCg = 16;
  // fp32 gradient plane + one branch's bf16 gradients and argmax codes
  const size_t tiled_smem = static_cast<size_t>(dx->h) * dx->w * kCg * (sizeof(float) + sizeof(__nv_bfloat16) + 1);
  if (dx->c % kCg == 0 && tiled_smem <= 200 * 1024) {  // every map the forward pools in shared memory (8 B per element) fits here
    static PerDevice<int> smem_limit(48 * 1024);
    YB_CHECK_CUDA(raise_smem_limit(smem_limit, static_cast<int>(tiled_smem), spp_pool_bwd_tiled_kernel<kCg>));
    launch_k(spp_pool_bwd_tiled_kernel<kCg>, dim3(dx->c / kCg, dx->n), 256, tiled_smem, st, mk(d0), mk(d5), mk(d9), mk(d13), argmax, mk(dx));
    YB_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  YB_CHECK_CUDA(cudaMemsetAsync(scratch, 0, elems * sizeof(float), st));
  launch_k(spp_pool_bwd_scatter_kernel, grid_for(3 * elems, 256), 256, 0, st, mk(d5), mk(d9), mk(d13), argmax, scratch, dx->n, dx->h, dx->w, dx->c);
  YB_CHECK_CUDA(cudaGetLastError());
  launch_k(spp_pool_bwd_finish_kernel, grid_for(elems / 8, 256), 256, 0, st, mk(d0), scratch, mk(dx));
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_copy_view(const yb200_act* src, const yb200_act* dst, void* stream) {
  int rc;
  if ((rc = check_act(src, "copy_view src")) || (rc = check_act(dst, "copy_view dst"))) return rc;
  YB_REQUIRE(same_shape(src, dst), YB200_ERR_INVALID, "copy_view: shape mismatch");
  const long long total = 1LL * src->n * src->h * src->w * (src->c / 8);
  launch_k(copy_view_kernel, grid_for(total, 256), 256, 0, as_stream(stream), mk(src), mk(dst));
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False) on fp32 planes [planes][h][w] -> [planes][2h][2w]
// (SparseInst mask logits, decoder_sparseinst.py:148-153).  Source coordinate (dst + 0.5) / 2 - 0.5, negative values clamped to 0, the upper
// neighbour clamped to the last row / column; the four products are combined in ATen's order.  One thread per INPUT pixel writes its 2 x 2 outputs.
// ------------------------------------------------------------------------------------------------
namespace {
__global__ void upsample_bilinear2x_kernel(const float* __restrict__ in, float* __restrict__ out, long long planes, int h, int w) {
  pdl_sync();
  const long long total = planes * h * w;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = static_cast<int>(i % w);
    const int y = static_cast<int>((i / w) % h);
    const long long pl = i / (1LL * w * h);
    const float* src = in + pl * h * w;
    float* dst = out + pl * 4LL * h * w;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      // output row 2y + dy: source y - 0.25 (dy = 0) or y + 0.25 (dy = 1)
      const int y0 = dy == 0 ? max(y - 1, 0) : y;
      const int y1 = min(y0 + 1, h - 1);
      const float ly = dy == 0 ? (y == 0 ? 0.f : 0.75f) : 0.25f;
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int x0 = dx == 0 ? max(x - 1, 0) : x;
        const int x1 = min(x0 + 1, w - 1);
        const float lx = dx == 0 ? (x == 0 ? 0.f : 0.75f) : 0.25f;
        const float v = (1.f - ly) * ((1.f - lx) * src[y0 * w + x0] + lx * src[y0 * w + x1]) + ly * ((1.f - lx) * src[y1 * w + x0] + lx * src[y1 * w + x1]);
        dst[(2LL * y + dy) * (2 * w) + 2 * x + dx] = v;
      }
    }
  }
}
}  // namespace

extern "C" int yb200_upsample_bilinear2x_f32(const float* in, float* out, int64_t planes, int h, int w, void* stream) {
  YB_REQUIRE(in && out && planes > 0 && h > 0 && w > 0, YB200_ERR_INVALID, "upsample_bilinear2x_f32: bad arguments");
  const long long total = planes * h * w;
  launch_k(upsample_bilinear2x_kernel, grid_for(total, 256), 256, 0, as_stream(stream), in, out, static_cast<long long>(planes), h, w);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
