// Kernels of the SparseInst InstanceContextEncoder (yolov7/modeling/transcoders/encoder_sparseinst.py:18-127) that are not GEMMs: the
// pyramid pooling's average pool and its adjoint, the bilinear resize to an arbitrary size and its adjoint, and the nearest x2 top-down
// path and its adjoint.  The 1x1 / 3x3 convolutions of the encoder, their data / weight gradients and the bias column sums are the
// implicit-GEMM entry points of conv_api.cu and convnext.cu.  Every operand is an NHWC bf16 view (channel slices of concat buffers), every
// sum runs in fp32 in a fixed order and there are no atomics: the results are bit-reproducible.
#include "host_common.cuh"
#include "sm90.cuh"

#include <algorithm>

using namespace yb;

namespace {

// a view with its channel offset applied: element (n, y, x, c) at p[((n * h + y) * w + x) * pitch + c]
struct V {
  const __nv_bfloat16* p;
  int n, h, w, c, pitch;
};
struct VO {
  __nv_bfloat16* p;
  int n, h, w, c, pitch;
};

V in_view(const yb200_act* a) {
  return V{a ? static_cast<const __nv_bfloat16*>(a->ptr) + a->c_off : nullptr, a ? a->n : 0, a ? a->h : 0, a ? a->w : 0, a ? a->c : 0,
           a ? a->c_pitch : 0};
}
VO out_view(const yb200_act* a) {
  return VO{static_cast<__nv_bfloat16*>(a->ptr) + a->c_off, a->n, a->h, a->w, a->c, a->c_pitch};
}

__device__ __forceinline__ const uint4* at(const V& v, int n, int y, int x, int c) {
  return reinterpret_cast<const uint4*>(v.p + ((static_cast<long long>(n) * v.h + y) * v.w + x) * v.pitch + c);
}
__device__ __forceinline__ uint4* at(const VO& v, int n, int y, int x, int c) {
  return reinterpret_cast<uint4*>(v.p + ((static_cast<long long>(n) * v.h + y) * v.w + x) * v.pitch + c);
}

__device__ __forceinline__ void unpack8(uint4 u, float* f) {
  f[0] = bf16_lo(u.x), f[1] = bf16_hi(u.x), f[2] = bf16_lo(u.y), f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z), f[5] = bf16_hi(u.z), f[6] = bf16_lo(u.w), f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

// thread index t -> (image, row, column, first channel) of an 8-channel chunk of `o`'s pixels
struct Chunk {
  int n, y, x, c;
};
template <typename T>
__device__ __forceinline__ Chunk chunk_of(long long t, const T& o) {
  const int chunks = o.c >> 3;
  const long long pix = t / chunks;
  Chunk k;
  k.c = static_cast<int>(t - pix * chunks) * 8;
  k.x = static_cast<int>(pix % o.w);
  const long long r = pix / o.w;
  k.y = static_cast<int>(r % o.h);
  k.n = static_cast<int>(r / o.h);
  return k;
}

// MyAdaptiveAvgPool2d (encoder_sparseinst.py:18-39): F.avg_pool2d with kernel = stride = (kh, kw), floor mode, no padding.  The window is
// summed row by row, left to right, then divided by kh * kw (count_include_pad makes the divisor the window size).
__global__ void __launch_bounds__(256) avg_pool_kernel(V x, VO o, int kh, int kw, long long total) {
  pdl_sync();
  const float div = static_cast<float>(kh * kw);
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const Chunk k = chunk_of(t, o);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, v[8];
    for (int dy = 0; dy < kh; ++dy)
      for (int dx = 0; dx < kw; ++dx) {
        unpack8(*at(x, k.n, k.y * kh + dy, k.x * kw + dx, k.c), v);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += v[j];
      }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] /= div;
    *at(o, k.n, k.y, k.x, k.c) = pack8(acc);
  }
}

constexpr int kMaxStages = 8;
struct Stage {
  const __nv_bfloat16* p;
  int h, w, pitch, kh, kw;
};
struct Stages {
  Stage s[kMaxStages];
  int count;
};

// The gradient of the PPM's input (encoder_sparseinst.py:56-68: feats feeds every stage's pool and the concat): d x = d cat + sum over the
// stages, in order, of avg_pool2d's adjoint, d pooled / (kh * kw) at every pixel of the window that covers it.  Pixels beyond the last full
// window (floor mode) receive only d cat.  One fp32 sum, rounded to bf16 once.
__global__ void __launch_bounds__(256) ppm_input_grad_kernel(V dcat, Stages st, VO dx, long long total) {
  pdl_sync();
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const Chunk k = chunk_of(t, dx);
    float acc[8], v[8];
    unpack8(*at(dcat, k.n, k.y, k.x, k.c), acc);
    for (int i = 0; i < st.count; ++i) {
      const Stage& s = st.s[i];
      const int py = k.y / s.kh, px = k.x / s.kw;
      if (py >= s.h || px >= s.w) continue;
      const float div = static_cast<float>(s.kh * s.kw);
      unpack8(*reinterpret_cast<const uint4*>(s.p + ((static_cast<long long>(k.n) * s.h + py) * s.w + px) * s.pitch + k.c), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j] / div;
    }
    *at(dx, k.n, k.y, k.x, k.c) = pack8(acc);
  }
}

// ATen's upsample_bilinear2d index arithmetic (align_corners=False, no scale factor given): scale = in / out,
// src = max(scale * (dst + 0.5) - 0.5, 0), i0 = (int)src, i1 = i0 + (i0 < in - 1), weights (1 - l, l) with l = src - i0, all in fp32
struct Tap {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ Tap bilinear_tap(float scale, int dst, int in) {
  float s = scale * (static_cast<float>(dst) + 0.5f) - 0.5f;
  s = s < 0.f ? 0.f : s;
  Tap t;
  t.i0 = static_cast<int>(s);
  t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
  t.l1 = s - static_cast<float>(t.i0);
  t.l0 = 1.f - t.l1;
  return t;
}
__device__ __forceinline__ float tap_weight(const Tap& t, int i) { return (t.i0 == i ? t.l0 : 0.f) + (t.i1 == i ? t.l1 : 0.f); }

// F.interpolate(x, size=(ho, wo), mode="bilinear", align_corners=False) (encoder_sparseinst.py:58-66 the PPM priors, :121-125 the fusion's
// x2 / x4): h0 (w0 x00 + w1 x01) + h1 (w0 x10 + w1 x11), the order of ATen's CUDA kernel
__global__ void __launch_bounds__(256) resize_bilinear_kernel(V x, VO o, float sh, float sw, long long total) {
  pdl_sync();
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const Chunk k = chunk_of(t, o);
    const Tap ty = bilinear_tap(sh, k.y, x.h), tx = bilinear_tap(sw, k.x, x.w);
    float a[8], b[8], c[8], d[8], r[8];
    unpack8(*at(x, k.n, ty.i0, tx.i0, k.c), a);
    unpack8(*at(x, k.n, ty.i0, tx.i1, k.c), b);
    unpack8(*at(x, k.n, ty.i1, tx.i0, k.c), c);
    unpack8(*at(x, k.n, ty.i1, tx.i1, k.c), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = ty.l0 * (tx.l0 * a[j] + tx.l1 * b[j]) + ty.l1 * (tx.l0 * c[j] + tx.l1 * d[j]);
    *at(o, k.n, k.y, k.x, k.c) = pack8(r);
  }
}

// output rows [lo, hi] that may tap input row i (src in [i - 1, i + 1)), widened by one row each side against rounding; rows outside
// the taps get weight 0 from tap_weight
__device__ __forceinline__ void tap_range(float scale, int i, int out, int* lo, int* hi) {
  *lo = max(0, static_cast<int>(floorf((static_cast<float>(i) - 0.5f) / scale - 0.5f)) - 1);
  *hi = min(out - 1, static_cast<int>(ceilf((static_cast<float>(i) + 1.5f) / scale - 0.5f)) + 1);
}

// The adjoint of resize_bilinear_kernel in gather form: input pixel (iy, ix) sums weight * d out over the output pixels whose taps reach it,
// output rows ascending, within a row the columns ascending (row sums first, then weighted by the row weight).  With h given (the ReLU output
// that was resized, same shape as dx), dx = h > 0 ? sum : 0: the gradient of the pre-activation of interpolate(relu(z)).
__global__ void __launch_bounds__(256) resize_bilinear_bwd_kernel(V dout, V h, VO dx, float sh, float sw, long long total) {
  pdl_sync();
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const Chunk k = chunk_of(t, dx);
    int y0, y1, x0, x1;
    tap_range(sh, k.y, dout.h, &y0, &y1);
    tap_range(sw, k.x, dout.w, &x0, &x1);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, row[8], v[8];
    for (int oy = y0; oy <= y1; ++oy) {
      const float wy = tap_weight(bilinear_tap(sh, oy, dx.h), k.y);
      if (wy == 0.f) continue;
#pragma unroll
      for (int j = 0; j < 8; ++j) row[j] = 0.f;
      for (int ox = x0; ox <= x1; ++ox) {
        const float wx = tap_weight(bilinear_tap(sw, ox, dx.w), k.x);
        if (wx == 0.f) continue;
        unpack8(*at(dout, k.n, oy, ox, k.c), v);
#pragma unroll
        for (int j = 0; j < 8; ++j) row[j] += wx * v[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += wy * row[j];
    }
    if (h.p) {
      unpack8(*at(h, k.n, k.y, k.x, k.c), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = v[j] > 0.f ? acc[j] : 0.f;
    }
    *at(dx, k.n, k.y, k.x, k.c) = pack8(acc);
  }
}

// The top-down path (encoder_sparseinst.py:114-118): out = lat + F.interpolate(coarse, scale_factor=2, mode="nearest"), one fp32 add rounded
// to bf16.  out may be lat itself (each element is read before it is written by the same thread).
__global__ void __launch_bounds__(256) nearest2x_add_kernel(V lat, V coarse, VO o, long long total) {
  pdl_sync();
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const Chunk k = chunk_of(t, o);
    float a[8], b[8];
    unpack8(*at(lat, k.n, k.y, k.x, k.c), a);
    unpack8(*at(coarse, k.n, k.y >> 1, k.x >> 1, k.c), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    *at(o, k.n, k.y, k.x, k.c) = pack8(a);
  }
}

// The adjoint of the nearest x2 up-sampling: dx = sum of the 2 x 2 block of dy, order (0,0) (0,1) (1,0) (1,1); with h given (the coarse
// level's ReLU output, same shape as dx), dx = h > 0 ? sum : 0
__global__ void __launch_bounds__(256) nearest2x_bwd_kernel(V dy, V h, VO dx, long long total) {
  pdl_sync();
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const Chunk k = chunk_of(t, dx);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, v[8];
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        unpack8(*at(dy, k.n, 2 * k.y + a, 2 * k.x + b, k.c), v);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += v[j];
      }
    if (h.p) {
      unpack8(*at(h, k.n, k.y, k.x, k.c), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = v[j] > 0.f ? acc[j] : 0.f;
    }
    *at(dx, k.n, k.y, k.x, k.c) = pack8(acc);
  }
}

long long chunks_of(const yb200_act* a) { return 1LL * a->n * a->h * a->w * (a->c / 8); }
int grid_of(long long total) { return static_cast<int>(std::max<long long>(1, std::min<long long>((total + 255) / 256, 16LL * sm_count()))); }

}  // namespace

extern "C" int yb200_avg_pool2d(const yb200_act* x, int kh, int kw, const yb200_act* out, void* stream) {
  int rc;
  if ((rc = check_act(x, "avg_pool2d x"))) return rc;
  if ((rc = check_act(out, "avg_pool2d out"))) return rc;
  YB_REQUIRE(kh > 0 && kw > 0 && x->h >= kh && x->w >= kw, YB200_ERR_INVALID, "avg_pool2d: %dx%d window on a %dx%d map", kh, kw, x->h, x->w);
  YB_REQUIRE(out->n == x->n && out->h == x->h / kh && out->w == x->w / kw && out->c == x->c, YB200_ERR_INVALID,
             "avg_pool2d: out %dx%dx%dx%d is not the %dx%d floor-mode pool of %dx%dx%dx%d", out->n, out->h, out->w, out->c, kh, kw, x->n, x->h, x->w,
             x->c);
  const long long total = chunks_of(out);
  launch_k(avg_pool_kernel, grid_of(total), 256, 0, as_stream(stream), in_view(x), out_view(out), kh, kw, total);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_ppm_input_grad(const yb200_act* dcat, const yb200_act* dpooled, const int32_t* kernel_hw, int nstages, const yb200_act* dx,
                                    void* stream) {
  int rc;
  if ((rc = check_act(dcat, "ppm_input_grad dcat"))) return rc;
  if ((rc = check_act(dx, "ppm_input_grad dx"))) return rc;
  YB_REQUIRE(same_shape(dcat, dx), YB200_ERR_INVALID, "ppm_input_grad: dcat and dx shapes differ");
  YB_REQUIRE(nstages >= 0 && nstages <= kMaxStages && (nstages == 0 || (dpooled && kernel_hw)), YB200_ERR_INVALID, "ppm_input_grad: %d stages",
             nstages);
  Stages st{};
  st.count = nstages;
  for (int i = 0; i < nstages; ++i) {
    const yb200_act* p = &dpooled[i];
    if ((rc = check_act(p, "ppm_input_grad dpooled"))) return rc;
    const int kh = kernel_hw[2 * i], kw = kernel_hw[2 * i + 1];
    YB_REQUIRE(kh > 0 && kw > 0 && p->n == dx->n && p->h == dx->h / kh && p->w == dx->w / kw && p->c == dx->c, YB200_ERR_INVALID,
               "ppm_input_grad: stage %d (%dx%dx%dx%d, window %dx%d) is not the pool of %dx%dx%dx%d", i, p->n, p->h, p->w, p->c, kh, kw, dx->n,
               dx->h, dx->w, dx->c);
    st.s[i] = Stage{static_cast<const __nv_bfloat16*>(p->ptr) + p->c_off, p->h, p->w, p->c_pitch, kh, kw};
  }
  const long long total = chunks_of(dx);
  launch_k(ppm_input_grad_kernel, grid_of(total), 256, 0, as_stream(stream), in_view(dcat), st, out_view(dx), total);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_resize_bilinear(const yb200_act* x, const yb200_act* out, void* stream) {
  int rc;
  if ((rc = check_act(x, "resize_bilinear x"))) return rc;
  if ((rc = check_act(out, "resize_bilinear out"))) return rc;
  YB_REQUIRE(out->n == x->n && out->c == x->c, YB200_ERR_INVALID, "resize_bilinear: %d images of %d channels -> %d of %d", x->n, x->c, out->n,
             out->c);
  const long long total = chunks_of(out);
  launch_k(resize_bilinear_kernel, grid_of(total), 256, 0, as_stream(stream), in_view(x), out_view(out),
           static_cast<float>(x->h) / static_cast<float>(out->h), static_cast<float>(x->w) / static_cast<float>(out->w), total);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_resize_bilinear_bwd(const yb200_act* dout, const yb200_act* h, const yb200_act* dx, void* stream) {
  int rc;
  if ((rc = check_act(dout, "resize_bilinear_bwd dout"))) return rc;
  if ((rc = check_act(dx, "resize_bilinear_bwd dx"))) return rc;
  if (h && (rc = check_act(h, "resize_bilinear_bwd h"))) return rc;
  YB_REQUIRE(dout->n == dx->n && dout->c == dx->c, YB200_ERR_INVALID, "resize_bilinear_bwd: %d images of %d channels -> %d of %d", dout->n,
             dout->c, dx->n, dx->c);
  YB_REQUIRE(!h || same_shape(h, dx), YB200_ERR_INVALID, "resize_bilinear_bwd: h and dx shapes differ");
  const long long total = chunks_of(dx);
  launch_k(resize_bilinear_bwd_kernel, grid_of(total), 256, 0, as_stream(stream), in_view(dout), in_view(h), out_view(dx),
           static_cast<float>(dx->h) / static_cast<float>(dout->h), static_cast<float>(dx->w) / static_cast<float>(dout->w), total);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_upsample_nearest2x_add(const yb200_act* lat, const yb200_act* coarse, const yb200_act* out, void* stream) {
  int rc;
  if ((rc = check_act(lat, "upsample_nearest2x_add lat"))) return rc;
  if ((rc = check_act(coarse, "upsample_nearest2x_add coarse"))) return rc;
  if ((rc = check_act(out, "upsample_nearest2x_add out"))) return rc;
  YB_REQUIRE(same_shape(lat, out), YB200_ERR_INVALID, "upsample_nearest2x_add: lat and out shapes differ");
  YB_REQUIRE(coarse->n == out->n && 2 * coarse->h == out->h && 2 * coarse->w == out->w && coarse->c == out->c, YB200_ERR_INVALID,
             "upsample_nearest2x_add: coarse %dx%dx%dx%d is not half of %dx%dx%dx%d", coarse->n, coarse->h, coarse->w, coarse->c, out->n, out->h,
             out->w, out->c);
  const long long total = chunks_of(out);
  launch_k(nearest2x_add_kernel, grid_of(total), 256, 0, as_stream(stream), in_view(lat), in_view(coarse), out_view(out), total);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_upsample_nearest2x_bwd(const yb200_act* dy, const yb200_act* h, const yb200_act* dx, void* stream) {
  int rc;
  if ((rc = check_act(dy, "upsample_nearest2x_bwd dy"))) return rc;
  if ((rc = check_act(dx, "upsample_nearest2x_bwd dx"))) return rc;
  if (h && (rc = check_act(h, "upsample_nearest2x_bwd h"))) return rc;
  YB_REQUIRE(dx->n == dy->n && 2 * dx->h == dy->h && 2 * dx->w == dy->w && dx->c == dy->c, YB200_ERR_INVALID,
             "upsample_nearest2x_bwd: dx %dx%dx%dx%d is not half of %dx%dx%dx%d", dx->n, dx->h, dx->w, dx->c, dy->n, dy->h, dy->w, dy->c);
  YB_REQUIRE(!h || same_shape(h, dx), YB200_ERR_INVALID, "upsample_nearest2x_bwd: h and dx shapes differ");
  const long long total = chunks_of(dx);
  launch_k(nearest2x_bwd_kernel, grid_of(total), 256, 0, as_stream(stream), in_view(dy), in_view(h), out_view(dx), total);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
