// ConvNeXt block kernels that are not GEMMs (SURVEY.md par.8a row C1): 7x7 depthwise convolution (forward, data gradient, weight
// gradient), LayerNorm over the channel dimension (forward / backward), column sums for bias gradients, the layer-scale gradient and
// the 4x4 patch gather of the stem.  All activations are NHWC bf16 views (yb200_act); parameters and their gradients are fp32.
//   Block.forward        yolov7/modeling/backbone/convnext.py:47-60
//   LayerNorm.forward    convnext.py:196-206  (channels_last = F.layer_norm; channels_first = the same per-pixel statistics)
//   stem / downsample    convnext.py:80-91
// These are HBM / CUDA-core bound streaming kernels: 16-byte or 8-byte accesses along the channel dimension, shared-memory halo
// tiles for the 7x7 window, fixed-order reductions (bit-reproducible gradients).
#include "host_common.cuh"
#include "sm90.cuh"
#include <algorithm>
#include <type_traits>

using namespace yb;

namespace {

struct ActV {  // device-side view
  const __nv_bfloat16* p;
  int n, h, w, c, pitch;
};
inline ActV viewc(const yb200_act* a) {
  return ActV{static_cast<const __nv_bfloat16*>(a->ptr) + a->c_off, a->n, a->h, a->w, a->c, a->c_pitch};
}

// ------------------------------------------------------------------------------------------------------------------------------
// depthwise 7x7, stride 1, zero padding 3
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int kDwTW = 32, kDwTH = 8, kDwC = 32;           // output tile (pixels) x channel slice per CTA
constexpr int kDwHW = kDwTW + 6, kDwHH = kDwTH + 6;       // halo tile
constexpr int kDwRow = kDwHW + 1;                         // padded row length (pixels): consecutive rows land in different bank halves
constexpr int kDwPixWords = kDwC / 2;                     // 32-bit words per pixel of the slice

__device__ __forceinline__ void dw_load_halo(uint32_t* s_x, const ActV& x, int n, int h0, int w0, int c0) {
  // 16-byte chunks: 4 per pixel
  for (int i = threadIdx.x; i < kDwHH * kDwHW * 4; i += blockDim.x) {
    const int ch = i & 3, pix = i >> 2;
    const int r = pix / kDwHW, col = pix - r * kDwHW;
    const int y = h0 + r - 3, xx = w0 + col - 3;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (y >= 0 && y < x.h && xx >= 0 && xx < x.w)
      v = *reinterpret_cast<const uint4*>(x.p + (static_cast<size_t>(n) * x.h + y) * x.w * x.pitch + static_cast<size_t>(xx) * x.pitch + c0 + ch * 8);
    *reinterpret_cast<uint4*>(s_x + (r * kDwRow + col) * kDwPixWords + ch * 4) = v;
  }
}

// out = dwconv7(x; w) [+ bias] [+ addend];  FLIP: use w[c][48 - t] (the data gradient is a correlation with the flipped kernel)
template <bool FLIP>
__global__ void __launch_bounds__(256) dwconv7_kernel(ActV x, const float* __restrict__ w, const float* __restrict__ bias, ActV addend, ActV out_v,
                                                      __nv_bfloat16* __restrict__ out, int tiles_w, int tiles_h) {
  pdl_sync();
  __shared__ __align__(16) uint32_t s_x[kDwHH * kDwRow * kDwPixWords];
  __shared__ float2 s_w[49][kDwC / 2];
  int t = blockIdx.x;
  const int tw = t % tiles_w;
  t /= tiles_w;
  const int th = t % tiles_h;
  const int n = t / tiles_h;
  const int c0 = blockIdx.y * kDwC;
  const int h0 = th * kDwTH, w0 = tw * kDwTW;
  for (int i = threadIdx.x; i < 49 * (kDwC / 2); i += blockDim.x) {
    const int tap = i / (kDwC / 2), cp = i - tap * (kDwC / 2);
    const int src = FLIP ? 48 - tap : tap;
    s_w[tap][cp] = make_float2(w[(c0 + 2 * cp) * 49 + src], w[(c0 + 2 * cp + 1) * 49 + src]);
  }
  dw_load_halo(s_x, x, n, h0, w0, c0);
  __syncthreads();

  const int cp = threadIdx.x & 15;
  const int g = threadIdx.x >> 4;       // 16 groups: rows g & 7, column half g >> 3 (a warp holds two consecutive rows)
  const int row = g & 7, half = g >> 3;
  float acc0[16], acc1[16];
  const float b0 = bias ? bias[c0 + 2 * cp] : 0.f, b1 = bias ? bias[c0 + 2 * cp + 1] : 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) { acc0[i] = b0; acc1[i] = b1; }
#pragma unroll 1
  for (int ky = 0; ky < 7; ++ky) {
    float2 wk[7];
#pragma unroll
    for (int kx = 0; kx < 7; ++kx) wk[kx] = s_w[ky * 7 + kx][cp];
    const uint32_t* xr = s_x + ((row + ky) * kDwRow + half * 16) * kDwPixWords + cp;
#pragma unroll
    for (int j = 0; j < 22; ++j) {  // input column j feeds outputs j-6 .. j
      const uint32_t u = xr[j * kDwPixWords];
      const float x0 = bf16_lo(u), x1 = bf16_hi(u);
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const int o = j - kx;
        if (o >= 0 && o < 16) {
          acc0[o] = fmaf(wk[kx].x, x0, acc0[o]);
          acc1[o] = fmaf(wk[kx].y, x1, acc1[o]);
        }
      }
    }
  }
  const int y = h0 + row;
  if (y >= out_v.h) return;
  const size_t rowbase = (static_cast<size_t>(n) * out_v.h + y) * out_v.w;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int xx = w0 + half * 16 + i;
    if (xx < out_v.w) {
      float v0 = acc0[i], v1 = acc1[i];
      if (addend.p != nullptr) {
        const uint32_t a = *reinterpret_cast<const uint32_t*>(addend.p + (rowbase + xx) * addend.pitch + c0 + 2 * cp);
        v0 += bf16_lo(a);
        v1 += bf16_hi(a);
      }
      *reinterpret_cast<uint32_t*>(out + (rowbase + xx) * out_v.pitch + c0 + 2 * cp) = pack_bf16x2(v0, v1);
    }
  }
}

// weight gradient: dw[c][ky][kx] = sum_px dy[px][c] * x[px + (ky-3, kx-3)][c],  db[c] = sum_px dy[px][c].
// Persistent CTAs walk tiles of one 32-channel slice; thread = (channel pair, ky) keeps 7 kx accumulators per channel (ky == 7: bias).
constexpr int kDwgThreads = 128;
__global__ void __launch_bounds__(kDwgThreads) dwconv7_wgrad_kernel(ActV x, ActV dy, float* __restrict__ partial, int tiles_w, int tiles_h, int tiles_total,
                                                                     int ctas_per_slice) {
  pdl_sync();
  extern __shared__ __align__(16) uint32_t s_dyn[];
  uint32_t* s_x = s_dyn;                                  // halo tile of x
  uint32_t* s_d = s_dyn + kDwHH * kDwRow * kDwPixWords;   // dy tile
  const int slice = blockIdx.x / ctas_per_slice, member = blockIdx.x - slice * ctas_per_slice;
  const int c0 = slice * kDwC;
  const int cp = threadIdx.x & 15, ky = threadIdx.x >> 4;  // ky 0..6 taps rows, 7 = bias
  float a0[7], a1[7];
#pragma unroll
  for (int i = 0; i < 7; ++i) { a0[i] = 0.f; a1[i] = 0.f; }
  for (int tile = member; tile < tiles_total; tile += ctas_per_slice) {
    int t = tile;
    const int tw = t % tiles_w;
    t /= tiles_w;
    const int th = t % tiles_h;
    const int n = t / tiles_h;
    const int h0 = th * kDwTH, w0 = tw * kDwTW;
    __syncthreads();  // previous tile fully consumed
    dw_load_halo(s_x, x, n, h0, w0, c0);
    for (int i = threadIdx.x; i < kDwTH * kDwTW * 4; i += blockDim.x) {
      const int ch = i & 3, pix = i >> 2;
      const int r = pix / kDwTW, col = pix - r * kDwTW;
      const int y = h0 + r, xx = w0 + col;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (y < dy.h && xx < dy.w)
        v = *reinterpret_cast<const uint4*>(dy.p + ((static_cast<size_t>(n) * dy.h + y) * dy.w + xx) * dy.pitch + c0 + ch * 8);
      *reinterpret_cast<uint4*>(s_d + pix * kDwPixWords + ch * 4) = v;
    }
    __syncthreads();
    if (ky < 7) {
#pragma unroll 1
      for (int r = 0; r < kDwTH; ++r) {
        const uint32_t* xr = s_x + ((r + ky) * kDwRow) * kDwPixWords + cp;
        const uint32_t* dr = s_d + (r * kDwTW) * kDwPixWords + cp;
        float w0v[7], w1v[7];  // sliding window of x over columns c .. c+6
#pragma unroll
        for (int i = 0; i < 6; ++i) {
          const uint32_t u = xr[i * kDwPixWords];
          w0v[i + 1] = bf16_lo(u);
          w1v[i + 1] = bf16_hi(u);
        }
#pragma unroll 4
        for (int c = 0; c < kDwTW; ++c) {
#pragma unroll
          for (int i = 0; i < 6; ++i) { w0v[i] = w0v[i + 1]; w1v[i] = w1v[i + 1]; }
          const uint32_t u = xr[(c + 6) * kDwPixWords];
          w0v[6] = bf16_lo(u);
          w1v[6] = bf16_hi(u);
          const uint32_t d = dr[c * kDwPixWords];
          const float d0 = bf16_lo(d), d1 = bf16_hi(d);
#pragma unroll
          for (int kx = 0; kx < 7; ++kx) {
            a0[kx] = fmaf(d0, w0v[kx], a0[kx]);
            a1[kx] = fmaf(d1, w1v[kx], a1[kx]);
          }
        }
      }
    } else {
      for (int px = 0; px < kDwTH * kDwTW; ++px) {
        const uint32_t d = s_d[px * kDwPixWords + cp];
        a0[0] += bf16_lo(d);
        a1[0] += bf16_hi(d);
      }
    }
  }
  // partial[cta][50][32]: taps 0..48, 49 = bias
  float* dst = partial + static_cast<size_t>(blockIdx.x) * 50 * kDwC;
  if (ky < 7) {
#pragma unroll
    for (int kx = 0; kx < 7; ++kx) {
      dst[(ky * 7 + kx) * kDwC + 2 * cp] = a0[kx];
      dst[(ky * 7 + kx) * kDwC + 2 * cp + 1] = a1[kx];
    }
  } else {
    dst[49 * kDwC + 2 * cp] = a0[0];
    dst[49 * kDwC + 2 * cp + 1] = a1[0];
  }
}
__global__ void dwconv7_wgrad_reduce_kernel(const float* __restrict__ partial, int ctas_per_slice, int channels, float* __restrict__ dw,
                                            float* __restrict__ db, int accumulate) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over channels * 50
  if (i >= channels * 50) return;
  const int c = i / 50, tap = i - c * 50;
  const int slice = c / kDwC, cl = c - slice * kDwC;
  float acc = 0.f;
  for (int m = 0; m < ctas_per_slice; ++m) acc += partial[(static_cast<size_t>(slice) * ctas_per_slice + m) * 50 * kDwC + tap * kDwC + cl];
  float* dst = tap < 49 ? dw + c * 49 + tap : (db ? db + c : nullptr);
  if (dst) *dst = accumulate ? *dst + acc : acc;
}

// ------------------------------------------------------------------------------------------------------------------------------
// LayerNorm over channels, one warp per pixel, 8-byte accesses (4 channels per lane and step)
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int kLnMaxSteps = 8;  // channels <= 8 * 128 = 1024
constexpr int kLnWarps = 8;

__device__ __forceinline__ void unpack4(uint2 u, float* f) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <int STEPS>
__global__ void __launch_bounds__(kLnWarps * 32) layernorm_fwd_kernel(ActV x, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                                       __nv_bfloat16* __restrict__ y, int y_pitch, float2* __restrict__ stats,
                                                                       long long npix) {
  pdl_sync();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c4 = x.c >> 2;  // 4-channel groups
  float g[STEPS][4], b[STEPS][4];
#pragma unroll
  for (int s = 0; s < STEPS; ++s) {
    const int q = lane + 32 * s;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      g[s][k] = q < c4 ? gamma[4 * q + k] : 0.f;
      b[s][k] = q < c4 ? beta[4 * q + k] : 0.f;
    }
  }
  const float inv_c = 1.f / static_cast<float>(x.c);
  for (long long pix = static_cast<long long>(blockIdx.x) * kLnWarps + warp; pix < npix; pix += static_cast<long long>(gridDim.x) * kLnWarps) {
    const __nv_bfloat16* src = x.p + pix * x.pitch;
    float v[STEPS][4];
    float sum = 0.f;
#pragma unroll
    for (int s = 0; s < STEPS; ++s) {
      const int q = lane + 32 * s;
      if (q < c4) {
        unpack4(*reinterpret_cast<const uint2*>(src + 4 * q), v[s]);
        sum += (v[s][0] + v[s][1]) + (v[s][2] + v[s][3]);
      } else {
        v[s][0] = v[s][1] = v[s][2] = v[s][3] = 0.f;
      }
    }
    const float mean = warp_sum(sum) * inv_c;
    float sq = 0.f;
#pragma unroll
    for (int s = 0; s < STEPS; ++s) {
      if (lane + 32 * s < c4) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float d = v[s][k] - mean;
          sq = fmaf(d, d, sq);
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(sq) * inv_c + eps);
    __nv_bfloat16* dst = y + pix * y_pitch;
#pragma unroll
    for (int s = 0; s < STEPS; ++s) {
      const int q = lane + 32 * s;
      if (q < c4) {
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) o[k] = fmaf((v[s][k] - mean) * rstd, g[s][k], b[s][k]);
        *reinterpret_cast<uint2*>(dst + 4 * q) = make_uint2(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]));
      }
    }
    if (stats != nullptr && lane == 0) stats[pix] = make_float2(mean, rstd);
  }
}

// dx = rstd * (g*gamma - mean_c(g*gamma) - xhat * mean_c(g*gamma*xhat)) [+ addend];  dgamma = sum_px g*xhat, dbeta = sum_px g.
// partial[block][2][C]: per-block sums in a fixed order (warps 0..7), reduced by layernorm_param_grad_kernel.
template <int STEPS>
__global__ void __launch_bounds__(kLnWarps * 32) layernorm_bwd_kernel(ActV dy, ActV x, const float2* __restrict__ stats, const float* __restrict__ gamma,
                                                                       ActV addend, __nv_bfloat16* __restrict__ dx, int dx_pitch,
                                                                       float* __restrict__ partial, long long npix) {
  pdl_sync();
  extern __shared__ float s_red[];  // [kLnWarps][2][C]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c4 = x.c >> 2;
  float g[STEPS][4], ag[STEPS][4], ab[STEPS][4];
#pragma unroll
  for (int s = 0; s < STEPS; ++s) {
    const int q = lane + 32 * s;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      g[s][k] = q < c4 ? gamma[4 * q + k] : 0.f;
      ag[s][k] = 0.f;
      ab[s][k] = 0.f;
    }
  }
  const float inv_c = 1.f / static_cast<float>(x.c);
  for (long long pix = static_cast<long long>(blockIdx.x) * kLnWarps + warp; pix < npix; pix += static_cast<long long>(gridDim.x) * kLnWarps) {
    const float2 st = stats[pix];
    float xh[STEPS][4], gy[STEPS][4];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int s = 0; s < STEPS; ++s) {
      const int q = lane + 32 * s;
      if (q < c4) {
        float xv[4];
        unpack4(*reinterpret_cast<const uint2*>(x.p + pix * x.pitch + 4 * q), xv);
        unpack4(*reinterpret_cast<const uint2*>(dy.p + pix * dy.pitch + 4 * q), gy[s]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          xh[s][k] = (xv[k] - st.x) * st.y;
          ag[s][k] = fmaf(gy[s][k], xh[s][k], ag[s][k]);
          ab[s][k] += gy[s][k];
          const float t = gy[s][k] * g[s][k];
          gy[s][k] = t;
          s1 += t;
          s2 = fmaf(t, xh[s][k], s2);
        }
      }
    }
    const float m1 = warp_sum(s1) * inv_c, m2 = warp_sum(s2) * inv_c;
#pragma unroll
    for (int s = 0; s < STEPS; ++s) {
      const int q = lane + 32 * s;
      if (q < c4) {
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) o[k] = st.y * (gy[s][k] - m1 - xh[s][k] * m2);
        if (addend.p != nullptr) {
          float a[4];
          unpack4(*reinterpret_cast<const uint2*>(addend.p + pix * addend.pitch + 4 * q), a);
#pragma unroll
          for (int k = 0; k < 4; ++k) o[k] += a[k];
        }
        *reinterpret_cast<uint2*>(dx + pix * dx_pitch + 4 * q) = make_uint2(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]));
      }
    }
  }
  const int C = x.c;
#pragma unroll
  for (int s = 0; s < STEPS; ++s) {
    const int q = lane + 32 * s;
    if (q < c4) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        s_red[(warp * 2 + 0) * C + 4 * q + k] = ag[s][k];
        s_red[(warp * 2 + 1) * C + 4 * q + k] = ab[s][k];
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
    const int which = i / C, c = i - which * C;
    float acc = 0.f;
#pragma unroll
    for (int w = 0; w < kLnWarps; ++w) acc += s_red[(w * 2 + which) * C + c];
    partial[static_cast<size_t>(blockIdx.x) * 2 * C + i] = acc;
  }
}
__global__ void layernorm_param_grad_kernel(const float* __restrict__ partial, int blocks, int C, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                            int accumulate) {
  pdl_sync();
  // one warp per output element (2C of them): lanes stride over blocks, then a fixed-order shuffle tree
  const int lane = threadIdx.x & 31;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= 2 * C) return;
  float acc = 0.f;
  for (int b = lane; b < blocks; b += 32) acc += partial[static_cast<size_t>(b) * 2 * C + i];
  acc = warp_sum(acc);
  if (lane == 0) {
    float* dst = i < C ? dgamma + i : dbeta + (i - C);
    *dst = accumulate ? *dst + acc : acc;
  }
}

// ------------------------------------------------------------------------------------------------------------------------------
// column sums of a bf16 view (bias gradients), deterministic two-stage
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int kCsBlocks = 592;
__global__ void __launch_bounds__(256) colsum_partial_kernel(ActV x, long long npix, float* __restrict__ partial) {
  pdl_sync();
  // thread = (8-channel group, pixel lane); block covers all channel groups when c/8 <= 256
  extern __shared__ float s_cs[];  // [rows][c]
  const int groups = x.c >> 3;
  const int rows = blockDim.x / groups;
  const int gq = threadIdx.x % groups, r = threadIdx.x / groups;
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.f;
  if (r < rows) {
    for (long long pix = static_cast<long long>(blockIdx.x) * rows + r; pix < npix; pix += static_cast<long long>(gridDim.x) * rows) {
      const uint4 u = *reinterpret_cast<const uint4*>(x.p + pix * x.pitch + 8 * gq);
      acc[0] += bf16_lo(u.x); acc[1] += bf16_hi(u.x); acc[2] += bf16_lo(u.y); acc[3] += bf16_hi(u.y);
      acc[4] += bf16_lo(u.z); acc[5] += bf16_hi(u.z); acc[6] += bf16_lo(u.w); acc[7] += bf16_hi(u.w);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) s_cs[r * x.c + 8 * gq + k] = acc[k];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < x.c; c += blockDim.x) {
    float t = 0.f;
    for (int rr = 0; rr < rows; ++rr) t += s_cs[rr * x.c + c];
    partial[static_cast<size_t>(blockIdx.x) * x.c + c] = t;
  }
}
__global__ void colsum_final_kernel(const float* __restrict__ partial, int blocks, int C, float scale, float* __restrict__ out, int accumulate) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (c >= C) return;
  float acc = 0.f;
  for (int b = lane; b < blocks; b += 32) acc += partial[static_cast<size_t>(b) * C + c];
  acc = warp_sum(acc) * scale;
  if (lane == 0) out[c] = accumulate ? out[c] + acc : acc;
}

// ------------------------------------------------------------------------------------------------------------------------------
// layer scale (convnext.py:55-56): out = gamma * (h W2^T + b2).  With G = g_out^T h (the weight gradient w.r.t. the unscaled output
// gradient) and s = colsum(g_out):   dW2[c][k] = gamma[c] G[c][k],  dgamma[c] = sum_k W2[c][k] G[c][k] + b2[c] s[c],  db2[c] = gamma[c] s[c].
// One warp per output channel; G is overwritten by / accumulated into dW2.
// ------------------------------------------------------------------------------------------------------------------------------
__global__ void layer_scale_grad_kernel(const float* __restrict__ G, const float* __restrict__ W2, const float* __restrict__ b2,
                                        const float* __restrict__ gamma, const float* __restrict__ s, int C, int K, float* __restrict__ dW2,
                                        float* __restrict__ dgamma, float* __restrict__ db2, int accumulate) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (c >= C) return;
  const float gm = gamma[c];
  float dot = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float gv = G[static_cast<size_t>(c) * K + k];
    dot = fmaf(W2[static_cast<size_t>(c) * K + k], gv, dot);
    float* d = dW2 + static_cast<size_t>(c) * K + k;
    *d = accumulate ? *d + gm * gv : gm * gv;
  }
  dot = warp_sum(dot);
  if (lane == 0) {
    const float dg = dot + b2[c] * s[c], db = gm * s[c];
    dgamma[c] = accumulate ? dgamma[c] + dg : dg;
    db2[c] = accumulate ? db2[c] + db : db;
  }
}

// ------------------------------------------------------------------------------------------------------------------------------
// stem: gather 4x4 patches of the uint8 image into [N][H/4][W/4][48] bf16, channel index = c*16 + kh*4 + kw (the flattening of the
// OIHW stem weight, convnext.py:82), so the stem convolution becomes a K = 48 GEMM.
// ------------------------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) patchify4_kernel(const T* __restrict__ img, int n, int h, int w, __nv_bfloat16* __restrict__ out, int out_pitch,
                                                        int out_coff) {
  pdl_sync();
  const int ow = w >> 2, oh = h >> 2;
  const long long total = static_cast<long long>(n) * oh * ow * 12;  // one thread per (patch, c, kh): 4 pixels in, 4 bf16 out
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    // consecutive threads walk along the image row (ox fastest) so that the reads coalesce
    const int ox = static_cast<int>(i % ow);
    long long r = i / ow;
    const int kh = static_cast<int>(r % 4);
    r /= 4;
    const int oy = static_cast<int>(r % oh);
    r /= oh;
    const int c = static_cast<int>(r % 3);
    const int b = static_cast<int>(r / 3);
    const T* src = img + ((static_cast<size_t>(b) * 3 + c) * h + oy * 4 + kh) * w + ox * 4;
    float v[4];
    if constexpr (sizeof(T) == 1) {
      const uchar4 px = *reinterpret_cast<const uchar4*>(src);
      v[0] = px.x; v[1] = px.y; v[2] = px.z; v[3] = px.w;
    } else {
      const float4 px = *reinterpret_cast<const float4*>(src);
      v[0] = px.x; v[1] = px.y; v[2] = px.z; v[3] = px.w;
    }
    __nv_bfloat16* dst = out + ((static_cast<size_t>(b) * oh + oy) * ow + ox) * out_pitch + out_coff + c * 16 + kh * 4;
    *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]));
  }
}

__global__ void f64_to_f32_kernel(double* __restrict__ src, int n, float* __restrict__ dst, int accumulate, int zero_src) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = static_cast<float>(src[i]);
  dst[i] = accumulate ? dst[i] + v : v;
  if (zero_src) src[i] = 0.0;
}

// out = a + b on bf16 views of equal shape (tensor + positional embedding, detr_backbone.py:154-155)
__global__ void __launch_bounds__(256) add_bf16_kernel(ActV a, ActV b, __nv_bfloat16* __restrict__ out, int out_pitch, long long npix) {
  pdl_sync();
  const int groups = a.c >> 3;
  const long long total = npix * groups;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long pix = i / groups;
    const int c8 = static_cast<int>(i - pix * groups) * 8;
    const uint4 x = *reinterpret_cast<const uint4*>(a.p + pix * a.pitch + c8), y = *reinterpret_cast<const uint4*>(b.p + pix * b.pitch + c8);
    uint4 o;
    o.x = pack_bf16x2(bf16_lo(x.x) + bf16_lo(y.x), bf16_hi(x.x) + bf16_hi(y.x));
    o.y = pack_bf16x2(bf16_lo(x.y) + bf16_lo(y.y), bf16_hi(x.y) + bf16_hi(y.y));
    o.z = pack_bf16x2(bf16_lo(x.z) + bf16_lo(y.z), bf16_hi(x.z) + bf16_hi(y.z));
    o.w = pack_bf16x2(bf16_lo(x.w) + bf16_lo(y.w), bf16_hi(x.w) + bf16_hi(y.w));
    *reinterpret_cast<uint4*>(out + pix * out_pitch + c8) = o;
  }
}

// out = sigmoid(x) on bf16 views (instance activation maps, decoder_sparseinst.py:67)
__global__ void __launch_bounds__(256) sigmoid_bf16_kernel(ActV a, __nv_bfloat16* __restrict__ out, int out_pitch, long long npix) {
  pdl_sync();
  const int groups = a.c >> 3;
  const long long total = npix * groups;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long pix = i / groups;
    const int c8 = static_cast<int>(i - pix * groups) * 8;
    const uint4 x = *reinterpret_cast<const uint4*>(a.p + pix * a.pitch + c8);
    auto sg = [](float v) { return __fdividef(1.f, 1.f + __expf(-v)); };
    uint4 o;
    o.x = pack_bf16x2(sg(bf16_lo(x.x)), sg(bf16_hi(x.x)));
    o.y = pack_bf16x2(sg(bf16_lo(x.y)), sg(bf16_hi(x.y)));
    o.z = pack_bf16x2(sg(bf16_lo(x.z)), sg(bf16_hi(x.z)));
    o.w = pack_bf16x2(sg(bf16_lo(x.w)), sg(bf16_hi(x.w)));
    *reinterpret_cast<uint4*>(out + pix * out_pitch + c8) = o;
  }
}
// inst[r][c] = raw[r][c] / max(norm[r], 1e-6) -> bf16 (decoder_sparseinst.py:75-76)
__global__ void iam_normalize_kernel(const float* __restrict__ raw, const float* __restrict__ norm, int rows, int cols, __nv_bfloat16* __restrict__ out, int out_pitch) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int r = i / cols, c = i - r * cols;
  out[static_cast<size_t>(r) * out_pitch + c] = __float2bfloat16_rn(raw[i] / fmaxf(norm[r], 1e-6f));
}

template <typename F>
int dispatch_steps(int c, F&& f) {
  const int steps = (c / 4 + 31) / 32;
  switch (steps) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 3: return f(std::integral_constant<int, 3>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 5: case 6: return f(std::integral_constant<int, 6>{});
    case 7: case 8: return f(std::integral_constant<int, 8>{});
    default: return fail(YB200_ERR_UNSUPPORTED, "layernorm: %d channels (max %d)", c, kLnMaxSteps * 128);
  }
}

int ln_grid(long long npix) {
  const long long want = (npix + kLnWarps - 1) / kLnWarps;
  const long long cap = 8LL * sm_count();
  return static_cast<int>(want < cap ? want : cap);
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------------------------------------
extern "C" int yb200_dwconv7(const yb200_act* x, const float* w_c49, const float* bias, const yb200_act* addend, const yb200_act* out, int flip,
                             void* stream) {
  int rc;
  if ((rc = check_act(x, "dwconv7 x", 32))) return rc;
  if ((rc = check_act(out, "dwconv7 out", 32))) return rc;
  if (addend && (rc = check_act(addend, "dwconv7 addend"))) return rc;
  YB_REQUIRE(w_c49 != nullptr, YB200_ERR_INVALID, "dwconv7: null weights");
  YB_REQUIRE(same_shape(x, out) && (!addend || same_shape(addend, out)), YB200_ERR_INVALID, "dwconv7: shapes differ");
  const int tiles_w = ceil_div(x->w, kDwTW), tiles_h = ceil_div(x->h, kDwTH);
  dim3 grid(tiles_w * tiles_h * x->n, x->c / kDwC);
  ActV av = addend ? viewc(addend) : ActV{nullptr, 0, 0, 0, 0, 0};
  ActV ov = viewc(out);
  __nv_bfloat16* op = static_cast<__nv_bfloat16*>(out->ptr) + out->c_off;
  if (flip)
    launch_k(dwconv7_kernel<true>, grid, 256, 0, as_stream(stream), viewc(x), w_c49, bias, av, ov, op, tiles_w, tiles_h);
  else
    launch_k(dwconv7_kernel<false>, grid, 256, 0, as_stream(stream), viewc(x), w_c49, bias, av, ov, op, tiles_w, tiles_h);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int dwg_ctas_per_slice(const yb200_act* x) {
  const int slices = x->c / kDwC;
  const int tiles = ceil_div(x->w, kDwTW) * ceil_div(x->h, kDwTH) * x->n;
  int per = (4 * sm_count()) / slices;
  if (per < 1) per = 1;
  if (per > tiles) per = tiles;
  return per;
}

extern "C" int64_t yb200_dwconv7_wgrad_workspace(const yb200_act* x) {
  if (!x || x->c <= 0 || x->c % kDwC != 0) return YB200_ERR_INVALID;
  return 4LL * (x->c / kDwC) * dwg_ctas_per_slice(x) * 50 * kDwC;
}

extern "C" int yb200_dwconv7_wgrad(const yb200_act* x, const yb200_act* dy, float* grad_w_c49, float* grad_bias, int accumulate, void* workspace,
                                   void* stream) {
  int rc;
  if ((rc = check_act(x, "dwconv7_wgrad x", 32))) return rc;
  if ((rc = check_act(dy, "dwconv7_wgrad dy", 32))) return rc;
  YB_REQUIRE(same_shape(x, dy) && grad_w_c49 && workspace, YB200_ERR_INVALID, "dwconv7_wgrad: bad arguments");
  const int tiles_w = ceil_div(x->w, kDwTW), tiles_h = ceil_div(x->h, kDwTH);
  const int per = dwg_ctas_per_slice(x);
  const int slices = x->c / kDwC;
  cudaStream_t st = as_stream(stream);
  constexpr int kSmem = (kDwHH * kDwRow + kDwTH * kDwTW) * kDwPixWords * 4;
  static PerDevice<int> smem_limit(0);
  YB_CHECK_CUDA(raise_smem_limit(smem_limit, kSmem, dwconv7_wgrad_kernel));
  launch_k(dwconv7_wgrad_kernel, slices * per, kDwgThreads, kSmem, st, viewc(x), viewc(dy), static_cast<float*>(workspace), tiles_w, tiles_h,
                                                             tiles_w * tiles_h * x->n, per);
  launch_k(dwconv7_wgrad_reduce_kernel, ceil_div(x->c * 50, 256), 256, 0, st, static_cast<const float*>(workspace), per, x->c, grad_w_c49, grad_bias, accumulate);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_layernorm_fwd(const yb200_act* x, const float* gamma, const float* beta, float eps, const yb200_act* y, float* stats_mean_rstd,
                                   void* stream) {
  int rc;
  if ((rc = check_act(x, "layernorm_fwd x", 4))) return rc;
  if ((rc = check_act(y, "layernorm_fwd y", 4))) return rc;
  YB_REQUIRE(gamma && beta && same_shape(x, y), YB200_ERR_INVALID, "layernorm_fwd: bad arguments");
  const long long npix = 1LL * x->n * x->h * x->w;
  cudaStream_t st = as_stream(stream);
  __nv_bfloat16* yp = static_cast<__nv_bfloat16*>(y->ptr) + y->c_off;
  rc = dispatch_steps(x->c, [&](auto steps) {
    launch_k(layernorm_fwd_kernel<decltype(steps)::value>, ln_grid(npix), kLnWarps * 32, 0, st, viewc(x), gamma, beta, eps, yp, y->c_pitch,
             reinterpret_cast<float2*>(stats_mean_rstd), npix);
    return 0;
  });
  if (rc) return rc;
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int64_t yb200_layernorm_bwd_workspace(const yb200_act* x) {
  if (!x || x->c <= 0) return YB200_ERR_INVALID;
  return 4LL * 2 * x->c * ln_grid(1LL * x->n * x->h * x->w);
}

extern "C" int yb200_layernorm_bwd(const yb200_act* dy, const yb200_act* x, const float* stats_mean_rstd, const float* gamma, const yb200_act* addend,
                                   const yb200_act* dx, float* grad_gamma, float* grad_beta, int accumulate, void* workspace, void* stream) {
  int rc;
  if ((rc = check_act(dy, "layernorm_bwd dy", 4))) return rc;
  if ((rc = check_act(x, "layernorm_bwd x", 4))) return rc;
  if ((rc = check_act(dx, "layernorm_bwd dx", 4))) return rc;
  if (addend && (rc = check_act(addend, "layernorm_bwd addend", 4))) return rc;
  YB_REQUIRE(stats_mean_rstd && gamma && grad_gamma && grad_beta && workspace, YB200_ERR_INVALID, "layernorm_bwd: null pointer");
  YB_REQUIRE(same_shape(dy, x) && same_shape(dx, x) && (!addend || same_shape(addend, x)), YB200_ERR_INVALID, "layernorm_bwd: shapes differ");
  const long long npix = 1LL * x->n * x->h * x->w;
  const int blocks = ln_grid(npix);
  const int smem = kLnWarps * 2 * x->c * 4;
  cudaStream_t st = as_stream(stream);
  ActV av = addend ? viewc(addend) : ActV{nullptr, 0, 0, 0, 0, 0};
  __nv_bfloat16* dxp = static_cast<__nv_bfloat16*>(dx->ptr) + dx->c_off;
  rc = dispatch_steps(x->c, [&](auto steps) {
    constexpr int S = decltype(steps)::value;
    static PerDevice<int> smem_limit(0);  // per instantiation
    const cudaError_t e = raise_smem_limit(smem_limit, kLnWarps * 2 * S * 128 * 4, layernorm_bwd_kernel<S>);
    if (e != cudaSuccess) return fail(YB200_ERR_CUDA, "layernorm_bwd: %s", cudaGetErrorString(e));
    launch_k(layernorm_bwd_kernel<S>, blocks, kLnWarps * 32, smem, st, viewc(dy), viewc(x), reinterpret_cast<const float2*>(stats_mean_rstd), gamma, av, dxp,
                                                                 dx->c_pitch, static_cast<float*>(workspace), npix);
    return 0;
  });
  if (rc) return rc;
  launch_k(layernorm_param_grad_kernel, ceil_div(2 * x->c * 32, 256), 256, 0, st, static_cast<const float*>(workspace), blocks, x->c, grad_gamma, grad_beta,
                                                                            accumulate);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int64_t yb200_colsum_workspace(const yb200_act* x) {
  if (!x || x->c <= 0) return YB200_ERR_INVALID;
  return 4LL * kCsBlocks * x->c;
}

extern "C" int yb200_colsum(const yb200_act* x, float scale, float* out, int accumulate, void* workspace, void* stream) {
  int rc;
  if ((rc = check_act(x, "colsum x"))) return rc;
  YB_REQUIRE(out && workspace, YB200_ERR_INVALID, "colsum: null pointer");
  YB_REQUIRE(x->c / 8 <= 256, YB200_ERR_UNSUPPORTED, "colsum: %d channels (max 2048)", x->c);
  const long long npix = 1LL * x->n * x->h * x->w;
  const int groups = x->c / 8, rows = 256 / groups;
  const int smem = rows * x->c * 4;
  cudaStream_t st = as_stream(stream);
  launch_k(colsum_partial_kernel, kCsBlocks, 256, smem, st, viewc(x), npix, static_cast<float*>(workspace));
  launch_k(colsum_final_kernel, ceil_div(x->c * 32, 256), 256, 0, st, static_cast<const float*>(workspace), kCsBlocks, x->c, scale, out, accumulate);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_layer_scale_grad(const float* raw_wgrad, const float* w2, const float* b2, const float* gamma, const float* gout_colsum, int channels,
                                      int hidden, float* grad_w2, float* grad_gamma, float* grad_b2, int accumulate, void* stream) {
  YB_REQUIRE(raw_wgrad && w2 && b2 && gamma && gout_colsum && grad_w2 && grad_gamma && grad_b2 && channels > 0 && hidden > 0, YB200_ERR_INVALID,
             "layer_scale_grad: bad arguments");
  launch_k(layer_scale_grad_kernel, ceil_div(channels * 32, 256), 256, 0, as_stream(stream), raw_wgrad, w2, b2, gamma, gout_colsum, channels, hidden, grad_w2,
                                                                                       grad_gamma, grad_b2, accumulate);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_patchify4(const void* images_nchw, int is_f32, int n, int h, int w, const yb200_act* out, void* stream) {
  int rc;
  if ((rc = check_act(out, "patchify4 out"))) return rc;
  YB_REQUIRE(images_nchw && n > 0 && h % 4 == 0 && w % 4 == 0, YB200_ERR_INVALID, "patchify4: image %dx%dx%d (H, W must be multiples of 4)", n, h, w);
  YB_REQUIRE(out->n == n && out->h == h / 4 && out->w == w / 4 && out->c == 48, YB200_ERR_INVALID, "patchify4: output must be [%d][%d][%d][48]", n, h / 4,
             w / 4);
  const long long total = 1LL * n * (h / 4) * (w / 4) * 12;
  const int blocks = static_cast<int>(std::min<long long>((total + 255) / 256, 16LL * sm_count()));
  __nv_bfloat16* op = static_cast<__nv_bfloat16*>(out->ptr);
  if (is_f32)
    launch_k(patchify4_kernel<float>, blocks, 256, 0, as_stream(stream), static_cast<const float*>(images_nchw), n, h, w, op, out->c_pitch, out->c_off);
  else
    launch_k(patchify4_kernel<uint8_t>, blocks, 256, 0, as_stream(stream), static_cast<const uint8_t*>(images_nchw), n, h, w, op, out->c_pitch, out->c_off);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_f64_to_f32(double* src, int n, float* dst, int accumulate, int zero_src, void* stream) {
  YB_REQUIRE(src && dst && n >= 0, YB200_ERR_INVALID, "f64_to_f32: null pointer");
  if (n == 0) return 0;
  launch_k(f64_to_f32_kernel, ceil_div(n, 256), 256, 0, as_stream(stream), src, n, dst, accumulate, zero_src);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_add(const yb200_act* a, const yb200_act* b, const yb200_act* out, void* stream) {
  int rc;
  if ((rc = check_act(a, "add a"))) return rc;
  if ((rc = check_act(b, "add b"))) return rc;
  if ((rc = check_act(out, "add out"))) return rc;
  YB_REQUIRE(same_shape(a, b) && same_shape(a, out), YB200_ERR_INVALID, "add: shapes differ");
  const long long npix = 1LL * a->n * a->h * a->w;
  const long long total = npix * (a->c / 8);
  const int blocks = static_cast<int>(std::min<long long>((total + 255) / 256, 16LL * sm_count()));
  launch_k(add_bf16_kernel, blocks, 256, 0, as_stream(stream), viewc(a), viewc(b), static_cast<__nv_bfloat16*>(out->ptr) + out->c_off, out->c_pitch, npix);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_sigmoid(const yb200_act* x, const yb200_act* out, void* stream) {
  int rc;
  if ((rc = check_act(x, "sigmoid x"))) return rc;
  if ((rc = check_act(out, "sigmoid out"))) return rc;
  YB_REQUIRE(same_shape(x, out), YB200_ERR_INVALID, "sigmoid: shapes differ");
  const long long npix = 1LL * x->n * x->h * x->w;
  const long long total = npix * (x->c / 8);
  const int blocks = static_cast<int>(std::min<long long>((total + 255) / 256, 16LL * sm_count()));
  launch_k(sigmoid_bf16_kernel, blocks, 256, 0, as_stream(stream), viewc(x), static_cast<__nv_bfloat16*>(out->ptr) + out->c_off, out->c_pitch, npix);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_iam_normalize(const float* raw, const float* normalizer, int rows, int cols, const yb200_act* out, void* stream) {
  int rc;
  if ((rc = check_act(out, "iam_normalize out"))) return rc;
  YB_REQUIRE(raw && normalizer && rows > 0 && cols > 0, YB200_ERR_INVALID, "iam_normalize: bad arguments");
  YB_REQUIRE(out->n == 1 && out->h == 1 && out->w == rows && out->c == cols, YB200_ERR_INVALID, "iam_normalize: output must be a [1][1][%d][%d] view", rows, cols);
  launch_k(iam_normalize_kernel, ceil_div(rows * cols, 256), 256, 0, as_stream(stream), raw, normalizer, rows, cols, static_cast<__nv_bfloat16*>(out->ptr) + out->c_off,
                                                                                  out->c_pitch);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
